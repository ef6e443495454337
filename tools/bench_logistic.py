"""Time binary LogisticRegression on resident rows: the label scan, the Newton pass (loss, gradient and fp64 Hessian)
next to the Poisson Newton pass of b2_glm_pass on the same rows, the line-search pass (all 21 candidate steps) next to
b2_glm_line_search, predict_proba, and whole fits; prints one JSON line.

    python tools/bench_logistic.py [--rows 10000000] [--d 128] [--sk-rows 1000000] [--out FILE]

Rows: fp32 X ~ N(0, 1) drawn on the device with torch; labels 0 / 1 drawn with torch from expit(X beta + 0.2) with
beta ~ N(0, 1 / sqrt(d)), and a Poisson target from exp(0.3 (X beta) + 0.5) for the GLM passes.  Pass times are CUDA
events on the context's stream around the whole call (uploads of the coefficients and the copy of the sums included),
best of 3 after a warm-up.  Fits are host wall clock around ``fit`` on the device rows with device labels (the label
scan included).  For context, scikit-learn's LogisticRegression(solver="newton-cholesky") on the first --sk-rows rows
as host float64, end to end.  The card's name and power limit are read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bodywork_mlops_demo_b200 as b2  # noqa: E402
from bodywork_mlops_demo_b200 import _native as native  # noqa: E402


def _best(ctx, fn, reps=3):
    fn()
    best = float("inf")
    for _ in range(reps):
        ctx.sync()
        ctx.timer_start()
        fn()
        best = min(best, ctx.timer_stop())
    return round(best, 3)


def _device_copy(ctx, t, kind, shape):
    out = ctx.empty(shape, kind)
    import torch
    torch.cuda.synchronize()
    assert native.load().b2_copy_d2d(ctx._h, out.ptr, t.data_ptr(), t.numel() * t.element_size()) == 0, \
        native.last_error()
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--sk-rows", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = b2.Context(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    n, d = a.rows, a.d
    res = {"bench": "logistic", "gpu": ctx.info()["name"], "power_limit": power, "rows": n, "d": d}
    g = torch.Generator(device="cuda").manual_seed(0)
    Xt = torch.randn(n, d, device="cuda", generator=g, dtype=torch.float32)
    beta = torch.randn(d, device="cuda", generator=g, dtype=torch.float64) / np.sqrt(d)
    xb = Xt.double() @ beta
    labels = (torch.rand(n, device="cuda", generator=g, dtype=torch.float64) < torch.sigmoid(xb + 0.2)).float()
    counts = torch.poisson(torch.exp(0.3 * xb + 0.5), generator=g).float()
    X = _device_copy(ctx, Xt, "f32", (n, d))
    y = _device_copy(ctx, labels.contiguous(), "f32", (n,))
    yc = _device_copy(ctx, counts.contiguous(), "f32", (n,))
    coef = beta.cpu().numpy() * 0.5
    step = beta.cpu().numpy() * 0.1
    res["label_scan_ms"] = _best(ctx, lambda: ctx.label_scan(y))
    res["newton_pass_ms"] = _best(ctx, lambda: ctx.logistic_pass(X, y, coef, 0.1, hessian=True))
    res["glm_newton_pass_ms"] = _best(ctx, lambda: ctx.glm_pass(X, yc, coef * 0.3, 0.5, power=1.0, hessian=True))
    res["gradient_pass_ms"] = _best(ctx, lambda: ctx.logistic_pass(X, y, coef, 0.1, hessian=False))
    res["line_search_pass_ms"] = _best(ctx, lambda: ctx.logistic_line_search(X, y, coef, 0.1, step, 0.01))
    res["glm_line_search_pass_ms"] = _best(ctx, lambda: ctx.glm_line_search(X, yc, coef * 0.3, 0.5, step * 0.3, 0.01,
                                                                            power=1.0))

    def proba():
        ctx.logistic_predict(X, coef, 0.1, proba=True)["proba"].free()
    res["predict_proba_ms"] = _best(ctx, proba)
    res["newton_over_glm"] = round(res["newton_pass_ms"] / res["glm_newton_pass_ms"], 3)
    res["line_search_over_glm"] = round(res["line_search_pass_ms"] / res["glm_line_search_pass_ms"], 3)
    est = b2.B200LogisticRegression(ctx=ctx)
    est.fit(X, y)
    fits = []
    for _ in range(3):
        ctx.sync()
        t0 = time.perf_counter()
        est.fit(X, y)
        ctx.sync()
        fits.append((time.perf_counter() - t0) * 1e3)
    res["n_iter"] = int(est.n_iter_[0])
    res["fit_ms"] = round(min(fits), 2)
    res["two_passes_ms"] = round(res["newton_pass_ms"] + res["line_search_pass_ms"], 3)
    if a.sk_rows > 0:
        from sklearn import linear_model
        m = min(a.sk_rows, n)
        Xh = Xt[:m].double().cpu().numpy()
        yh = labels[:m].double().cpu().numpy()
        sk = linear_model.LogisticRegression(solver="newton-cholesky")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            t0 = time.perf_counter()
            sk.fit(Xh, yh)
            res["sklearn_rows"] = m
            res["sklearn_fit_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            res["sklearn_n_iter"] = int(sk.n_iter_[0])
    for buf in (X, y, yc):
        buf.free()
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
