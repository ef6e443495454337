"""Time BayesianRidge / ARDRegression on resident rows: the Gram pass, the anchor pass, the solves and the
predict(return_std=True) pass; prints one JSON line.

    python tools/bench_bayes.py [--rows 10000000] [--d 128] [--sk-rows 200000] [--out FILE]

Tables: b2_synth fp32 rows and the correlated table of tools/bench_enet.py.  Per table, with CUDA events on the context's
stream (best of 3 after a warm-up): the Gram pass with w0 (b2_fit), the anchor pass (b2_residual_moments), one b2_score
pass for comparison, the eigendecomposition (b2_solve_eigh), b2_solve_bayes_ridge (eigh + the BayesianRidge kernel),
b2_solve_ard with its iterations and time per iteration, and b2_score_std with its fp64 rate at 2 D^2 flops per row.
For context, scikit-learn's BayesianRidge / ARDRegression(max_iter=3) on the first --sk-rows rows in float64, end to end,
against the estimators on the same host rows.  The card's name and power limit are read in the same run.  Writes nothing
to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bodywork_mlops_demo_b200 as b2  # noqa: E402
from bench_enet import _correlated, _timed  # noqa: E402


def _best(ctx, fn, reps=3):
    fn()
    out, best = None, float("inf")
    for _ in range(reps):
        out, ms = _timed(ctx, fn)
        best = min(best, ms)
    return out, round(best, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--sk-rows", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = b2.Context(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    res = {"bench": "bayes", "gpu": ctx.info()["name"], "power_limit": power, "rows": a.rows, "d": a.d, "tables": []}
    n, d = a.rows, a.d
    for table in ("synth", "correlated"):
        keep = None
        if table == "synth":
            X, y = ctx.synth(n, d)
        else:
            X, y, Xt, yt = _correlated(ctx, n, d)
            keep = (Xt, yt)
        tab = {"table": table}
        (w0, b0), tab["gram_fit_ms"] = _best(ctx, lambda: ctx.fit(X, y))
        moments, tab["anchor_pass_ms"] = _best(ctx, lambda: ctx.residual_moments(X, y, w0, b0))
        _, tab["score_pass_ms"] = _best(ctx, lambda: ctx.score(X, w0, b0, y=y, want_yhat=False))
        anchor = np.concatenate([w0, moments])
        _, tab["eigh_ms"] = _best(ctx, lambda: ctx.solve_eigh())
        br, tab["bayes_ridge_solve_ms"] = _best(ctx, lambda: ctx.solve_bayes_ridge(anchor=anchor))
        tab["bayes_ridge_kernel_ms"] = round(tab["bayes_ridge_solve_ms"] - tab["eigh_ms"], 3)
        tab["bayes_ridge_n_iter"] = br["n_iter"]
        ard, tab["ard_ms"] = _best(ctx, lambda: ctx.solve_ard(anchor=anchor))
        tab["ard_n_iter"] = ard["n_iter"]
        tab["ard_ms_per_iter"] = round(tab["ard_ms"] / (ard["n_iter"] + 1), 4)
        tab["ard_kept"] = int(np.sum(ard["lambda"] < 1e4))
        mean = ctx.gram_export()[:d, d] / n
        (yh, ys), tab["score_std_ms"] = _best(
            ctx, lambda: ctx.score_std(X, mean, br["sigma"], 1.0 / br["alpha"], br["coef"], br["intercept"]))
        yh.free(); ys.free()
        tab["score_std_fp64_tflops"] = round(2.0 * d * d * n / (tab["score_std_ms"] * 1e-3) / 1e12, 2)
        if a.sk_rows > 0:
            from sklearn.linear_model import ARDRegression, BayesianRidge
            if keep is None:
                Xs, ysyn = ctx.synth(a.sk_rows, d)
                Xh, yh_ = Xs.to_host().astype(np.float64), ysyn.to_host().astype(np.float64)
                Xs.free(); ysyn.free()
            else:
                Xh = keep[0][: a.sk_rows].cpu().numpy().astype(np.float64)
                yh_ = keep[1][: a.sk_rows].cpu().numpy().astype(np.float64)
            for name, sk, ours in (("BayesianRidge", BayesianRidge(), b2.B200BayesianRidge(ctx=ctx)),
                                   ("ARDRegression max_iter=3", ARDRegression(max_iter=3),
                                    b2.B200ARDRegression(ctx=ctx, max_iter=3))):
                t0 = time.perf_counter()
                sk.fit(Xh, yh_)
                sk_s = time.perf_counter() - t0
                ours.fit(Xh, yh_)
                t0 = time.perf_counter()
                ours.fit(Xh, yh_)
                tab[name] = {"rows": a.sk_rows, "sklearn_s": round(sk_s, 3), "b2_s": round(time.perf_counter() - t0, 4),
                             "alpha_rel_diff": float(abs(ours.alpha_ - sk.alpha_) / sk.alpha_),
                             "n_iter": [int(ours.n_iter_), int(sk.n_iter_)]}
        res["tables"].append(tab)
        X.free(); y.free()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
