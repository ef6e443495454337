"""Time the GLM regressors on resident rows: the Newton pass (loss, gradient and fp64 Hessian), the line-search pass
(all 21 candidate steps) against one b2_score pass, and whole PoissonRegressor / GammaRegressor fits; prints one JSON
line.

    python tools/bench_glm.py [--rows 10000000] [--d 128] [--sk-rows 1000000] [--out FILE]

Rows: fp32 X ~ N(0, 1) drawn on the device with torch, targets drawn with torch from eta = X beta + 0.5 with
beta ~ N(0, 0.3 / sqrt(d)): Poisson(exp(eta)) and Gamma(shape 2, mean exp(eta)).  Pass times are CUDA events on the
context's stream around the whole call (uploads of the coefficients and the copy of the sums included), best of 3 after
a warm-up; the Newton pass's fp64 rate counts (d + 1)(d + 2) flops per row.  Fits are host wall clock around
``fit`` on the device rows.  For context, scikit-learn's solver="newton-cholesky" on the first --sk-rows rows as host
float64, end to end.  The card's name and power limit are read in the same run.  Writes nothing to the tree."""
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
    res = {"bench": "glm", "gpu": ctx.info()["name"], "power_limit": power, "rows": n, "d": d, "targets": []}
    torch.manual_seed(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    Xt = torch.randn(n, d, device="cuda", generator=g, dtype=torch.float32)
    beta = torch.randn(d, device="cuda", generator=g, dtype=torch.float64) * (0.3 / np.sqrt(d))
    eta = Xt.double() @ beta + 0.5
    X = ctx.empty((n, d), "f32")
    torch.cuda.synchronize()
    assert native.load().b2_copy_d2d(ctx._h, X.ptr, Xt.data_ptr(), n * d * 4) == 0, native.last_error()
    mu = torch.exp(eta)
    targets = {"poisson": torch.poisson(mu, generator=g),
               "gamma": torch.distributions.Gamma(torch.full_like(mu, 2.0), 2.0 / mu).sample()}
    coef = beta.cpu().numpy() * 0.5
    step = beta.cpu().numpy() * 0.1
    score_ms = None
    for name, yt in targets.items():
        yt = yt.float().contiguous()
        y = ctx.empty((n,), "f32")
        torch.cuda.synchronize()
        assert native.load().b2_copy_d2d(ctx._h, y.ptr, yt.data_ptr(), n * 4) == 0, native.last_error()
        p = 1.0 if name == "poisson" else 2.0
        t_newton = _best(ctx, lambda: ctx.glm_pass(X, y, coef, 0.3, power=p, hessian=True))
        t_grad = _best(ctx, lambda: ctx.glm_pass(X, y, coef, 0.3, power=p, hessian=False))
        t_ladder = _best(ctx, lambda: ctx.glm_line_search(X, y, coef, 0.3, step, 0.01, power=p))
        if score_ms is None:
            score_ms = _best(ctx, lambda: ctx.score(X, coef, 0.3, y=y, want_yhat=False))
        cls = b2.B200PoissonRegressor if name == "poisson" else b2.B200GammaRegressor
        est = cls(ctx=ctx, alpha=1e-4)
        est.fit(X, y)
        fits = []
        for _ in range(3):
            ctx.sync()
            t0 = time.perf_counter()
            est.fit(X, y)
            ctx.sync()
            fits.append((time.perf_counter() - t0) * 1e3)
        row = {"target": name, "newton_pass_ms": t_newton,
               "newton_pass_fp64_tflops": round(n * (d + 1) * (d + 2) / (t_newton * 1e-3) / 1e12, 2),
               "gradient_pass_ms": t_grad, "line_search_pass_ms": t_ladder, "score_pass_ms": score_ms,
               "line_search_over_score": round(t_ladder / score_ms, 3), "n_iter": int(est.n_iter_),
               "fit_ms": round(min(fits), 2),
               "fit_ms_per_iteration": round(min(fits) / max(est.n_iter_, 1), 2),
               "two_passes_ms": round(t_newton + t_ladder, 3)}
        if a.sk_rows > 0:
            from sklearn import linear_model
            m = min(a.sk_rows, n)
            Xh = Xt[:m].double().cpu().numpy()
            yh = yt[:m].double().cpu().numpy()
            sk = getattr(linear_model, "PoissonRegressor" if name == "poisson" else "GammaRegressor")(
                solver="newton-cholesky", alpha=1e-4)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                t0 = time.perf_counter()
                sk.fit(Xh, yh)
                row["sklearn_rows"] = m
                row["sklearn_fit_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                row["sklearn_n_iter"] = int(sk.n_iter_)
        res["targets"].append(row)
        y.free()
    X.free()
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
