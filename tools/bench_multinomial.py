"""Time multinomial LogisticRegression on resident rows: the label discovery, the gradient, Newton (loss, gradient and
every class-pair fp64 Hessian block) and line-search passes next to the binary b2_logistic_pass /
b2_logistic_line_search on the same rows, the host solve of the K (D + 1) Newton system, predict_proba and whole fits,
at K = 3, 10 and 32; prints one JSON line.

    python tools/bench_multinomial.py [--rows 10000000] [--d 128] [--classes 3,10,32] [--sk-rows 100000]
                                      [--sk-max-classes 10] [--out FILE]

Rows: fp32 X ~ N(0, 1) drawn on the device with torch; labels drawn with torch as argmax(X B + Gumbel noise) with
B ~ N(0, 1 / d), so every class is present.  Pass times are CUDA events on the context's stream around the whole call
(uploads of the coefficients and the copy of the sums included), best of --reps after a warm-up.  The host solve is
scipy.linalg.solve(assume_a="sym") of the Newton system the estimator forms from one Newton pass, wall clock.  Fits are
host wall clock around one ``fit`` on the device rows with device labels (the label discovery included), after a warm
fit at K = 3.  For context, scikit-learn's LogisticRegression(solver="newton-cholesky") on the first --sk-rows rows as
host float64, end to end, up to --sk-max-classes classes.  The card's name and power limit are read in the same run.
Writes nothing to the tree."""
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


def _best(ctx, fn, reps):
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


def _wall(ctx, fn):
    ctx.sync()
    t0 = time.perf_counter()
    out = fn()
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    import scipy.linalg
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--classes", default="3,10,32")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sk-rows", type=int, default=100_000)
    ap.add_argument("--sk-max-classes", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = b2.Context(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    n, d = a.rows, a.d
    res = {"bench": "multinomial", "gpu": ctx.info()["name"], "power_limit": power, "rows": n, "d": d}
    g = torch.Generator(device="cuda").manual_seed(0)
    Xt = torch.randn(n, d, device="cuda", generator=g, dtype=torch.float32)
    X = _device_copy(ctx, Xt, "f32", (n, d))
    rng = np.random.default_rng(0)
    # the binary passes on the same rows
    beta = torch.randn(d, device="cuda", generator=g, dtype=torch.float64) / np.sqrt(d)
    yb = (torch.rand(n, device="cuda", generator=g, dtype=torch.float64) < torch.sigmoid(Xt.double() @ beta)).float()
    ybd = _device_copy(ctx, yb.contiguous(), "f32", (n,))
    coef_b, step_b = beta.cpu().numpy() * 0.5, beta.cpu().numpy() * 0.1
    res["binary_gradient_pass_ms"] = _best(ctx, lambda: ctx.logistic_pass(X, ybd, coef_b, 0.1, hessian=False), a.reps)
    res["binary_newton_pass_ms"] = _best(ctx, lambda: ctx.logistic_pass(X, ybd, coef_b, 0.1, hessian=True), a.reps)
    res["binary_line_search_ms"] = _best(ctx, lambda: ctx.logistic_line_search(X, ybd, coef_b, 0.1, step_b, 0.01),
                                         a.reps)
    ybd.free()
    per = {}
    warm = True
    for k in [int(v) for v in a.classes.split(",")]:
        r = {}
        B = torch.randn(d, k, device="cuda", generator=g, dtype=torch.float32) / np.sqrt(d)
        u = torch.rand(n, k, device="cuda", generator=g, dtype=torch.float32).clamp_min(1e-12)
        labels = torch.argmax(Xt @ B - torch.log(-torch.log(u)), dim=1).float()
        del u
        y = _device_copy(ctx, labels.contiguous(), "f32", (n,))
        classes = np.arange(k, dtype=np.float32)

        def discover():
            ctx.label_scan(y)
            ctx.label_values(y)
        r["label_discovery_ms"] = _best(ctx, discover, a.reps)
        coef = rng.normal(size=(k, d + 1)) * 0.3 / np.sqrt(d)
        step = rng.normal(size=(k, d + 1)) * 0.1 / np.sqrt(d)
        reps = a.reps if k <= 10 else 1
        r["gradient_pass_ms"] = _best(ctx, lambda: ctx.multinomial_pass(X, y, classes, coef, hessian=False), reps)
        r["newton_pass_ms"] = _best(ctx, lambda: ctx.multinomial_pass(X, y, classes, coef, hessian=True), reps)
        r["line_search_ms"] = _best(ctx, lambda: ctx.multinomial_line_search(X, y, classes, coef, step), reps)
        s = ctx.multinomial_pass(X, y, classes, coef, hessian=True)
        m = k * (d + 1)
        H = s["hessian"].transpose(2, 0, 3, 1).reshape(m, m) / n
        H[np.arange(k * d), np.arange(k * d)] += 1.0 / n
        grad = (s["grad"] / n).ravel(order="F")
        t0 = time.perf_counter()
        scipy.linalg.solve(H[:-1, :-1], -grad[:-1], check_finite=False, assume_a="sym")
        r["host_solve_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
        est = b2.B200MultinomialLogisticRegression(ctx=ctx)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            if warm:
                est.fit(X, y)
                warm = False
            ms, _ = _wall(ctx, lambda: est.fit(X, y))
        r["fit_ms"] = round(ms, 1)
        r["n_iter"] = int(est.n_iter_[0])

        def proba():
            est.predict_proba(X).free()
        r["predict_proba_ms"] = _best(ctx, proba, reps)
        pairs = k * (k + 1) / 2
        r["newton_over_pairs_x_binary"] = round(r["newton_pass_ms"] / (pairs * res["binary_newton_pass_ms"]), 3)
        r["gradient_over_binary"] = round(r["gradient_pass_ms"] / res["binary_gradient_pass_ms"], 3)
        r["line_search_over_k_half_binary"] = round(r["line_search_ms"] / (k / 2 * res["binary_line_search_ms"]), 3)
        r["fit_model_ms"] = round(r["n_iter"] * (r["newton_pass_ms"] + r["line_search_ms"]) +
                                  r["n_iter"] * r["host_solve_ms"], 1)
        if a.sk_rows > 0 and k <= a.sk_max_classes:
            from sklearn import linear_model
            mrows = min(a.sk_rows, n)
            Xh = Xt[:mrows].double().cpu().numpy()
            yh = labels[:mrows].double().cpu().numpy()
            sk = linear_model.LogisticRegression(solver="newton-cholesky")
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                t0 = time.perf_counter()
                sk.fit(Xh, yh)
                r["sklearn_rows"] = mrows
                r["sklearn_fit_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                r["sklearn_n_iter"] = int(sk.n_iter_[0])
        y.free()
        per[str(k)] = r
    res["classes"] = per
    X.free()
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
