"""Time LinearDiscriminantAnalysis on resident rows: the class-sum pass, the within-class scatter pass with and without
weights next to the logistic Newton pass on the same rows, the host solvers, whole fits for each solver, predict,
predict_proba and transform, for several class counts; prints one JSON line.

    python tools/bench_lda.py [--rows 10000000] [--d 128] [--classes 2,10,32] [--sk-rows 1000000] [--out FILE]

Rows: fp32 b2_synth rows (seed 1234), labelled 3 k - 7 by the K quantile bins of their synthetic y.  Pass times are CUDA
events on the context's stream around the whole call (uploads and the copy of the sums included), best of 3 after a
warm-up.  Host solvers are host wall clock on the statistics of the run.  Fits are host wall clock around ``fit`` on the
device rows with device labels (label scan and label discovery included), median of 3 after a warm-up; predictions are
host wall clock on device rows with the device outputs, best of 3.  For context, scikit-learn's LDA on the first
--sk-rows rows as host float64 at K = 10, end to end.  The card's name and power limit are read in the same run.
Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bodywork_mlops_demo_b200 as b2  # noqa: E402
from bodywork_mlops_demo_b200 import estimator as est_mod  # noqa: E402


def _best(ctx, fn, reps=3):
    fn()
    best = float("inf")
    for _ in range(reps):
        ctx.sync()
        ctx.timer_start()
        fn()
        best = min(best, ctx.timer_stop())
    return round(best, 3)


def _wall(ctx, fn, reps=3, median=False):
    """host wall clock of fn() to a device synchronise, after a warm-up: best (or median) of reps; frees what fn
    returns on the device"""
    def run():
        out = fn()
        ctx.sync()
        for v in (out.values() if isinstance(out, dict) else [out]):
            if isinstance(v, b2.DeviceArray):
                v.free()
    run()
    ts = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        run()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(ts) if median else min(ts)), 2)


def _host_ms(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(min(ts), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--classes", default="2,10,32")
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
    res = {"bench": "lda", "gpu": ctx.info()["name"], "power_limit": power, "rows": n, "d": d, "per_k": {}}
    X, ys = ctx.synth(n, d, seed=1234)
    yh = ys.to_host()
    ys.free()
    flops = n * d * (d + 1)                          # the scatter's rate at n D (D + 1) flops: its upper triangle
    for k in [int(v) for v in a.classes.split(",")]:
        cuts = np.quantile(yh, np.linspace(0, 1, k + 1)[1:-1])
        t = np.searchsorted(cuts, yh)
        labels = (3.0 * np.arange(k) - 7.0).astype(np.float32)
        y = ctx.to_device(labels[t].astype(np.float32))
        r = {}
        cs = ctx.class_sums(X, y, labels)
        nk = cs["sums"][:, d]
        means = cs["sums"][:, :d] / nk[:, None]
        priors = nk / nk.sum()
        r["label_discovery_ms"] = _best(ctx, lambda: (ctx.label_scan(y), ctx.label_values(y)))
        r["class_sums_ms"] = _best(ctx, lambda: ctx.class_sums(X, y, labels))
        r["scatter_ms"] = _best(ctx, lambda: ctx.class_scatter(X, y, labels, means))
        r["scatter_weighted_ms"] = _best(ctx, lambda: ctx.class_scatter(X, y, labels, means, priors / nk))
        r["scatter_fp64_tflops"] = round(flops / r["scatter_ms"] * 1e-9, 2)
        w = np.full(d, 0.01)
        r["logistic_newton_pass_ms"] = _best(ctx, lambda: ctx.logistic_pass(X, y, w, 0.1, float(labels[0]),
                                                                            float(labels[1]), hessian=True))
        r["scatter_over_logistic_newton"] = round(r["scatter_ms"] / r["logistic_newton_pass_ms"], 3)
        sw1 = ctx.class_scatter(X, y, labels, means)["scatter"]
        cov = ctx.class_scatter(X, y, labels, means, priors / nk)["scatter"]
        xbar = nk @ means / nk.sum()
        total = (sw1 + (nk[:, None] * (means - xbar)).T @ (means - xbar)) / nk.sum()
        mc = min(k - 1, d)
        r["host_solver_ms"] = {
            "svd": _host_ms(lambda: est_mod._lda_svd(sw1, means, nk, priors, 1e-4, mc)),
            "lsqr": _host_ms(lambda: est_mod._lda_lstsq(cov, means, priors)),
            "eigen": _host_ms(lambda: est_mod._lda_eigen(cov, total, means, priors, mc))}
        fits = {}
        for solver in ("svd", "lsqr", "eigen"):
            est = b2.B200LinearDiscriminantAnalysis(solver=solver, ctx=ctx)
            fits[solver] = _wall(ctx, lambda: est.fit(X, y), median=True)
        r["fit_ms"] = fits
        est = b2.B200LinearDiscriminantAnalysis(ctx=ctx).fit(X, y)
        W, bb = est._model()
        r["decision_pass_ms"] = _wall(ctx, lambda: ctx.classify(X, W, bb, est._fp32_classes(est.classes_),
                                                                decision=True))
        r["predict_ms"] = _wall(ctx, lambda: est.predict(X))
        r["predict_proba_ms"] = _wall(ctx, lambda: est.predict_proba(X))
        c = min(est.scalings_.shape[1], est._max_components)
        S = est.scalings_[:, :c]
        r["transform_pass_ms"] = _wall(ctx, lambda: ctx.classify(X, S.T, -(est.xbar_ @ S),
                                                                 np.arange(max(c, 2), dtype=np.float32), decision=True))
        r["transform_ms"] = _wall(ctx, lambda: est.transform(X))
        budget = r["label_discovery_ms"] + r["class_sums_ms"] + r["scatter_ms"] + r["host_solver_ms"]["svd"] + 2.0
        r["goals"] = {"scatter_le_newton": r["scatter_ms"] <= r["logistic_newton_pass_ms"],
                      "svd_fit_le_parts_plus_2ms": fits["svd"] <= budget, "svd_fit_budget_ms": round(budget, 2),
                      "transform_le_pass_plus_1ms": r["transform_ms"] <= r["transform_pass_ms"] + 1.0,
                      "proba_le_pass_plus_1ms": None if k == 2 else r["predict_proba_ms"] <= r["decision_pass_ms"] + 1.0}
        res["per_k"][str(k)] = r
        if k == 10 and a.sk_rows > 0:
            from sklearn.discriminant_analysis import LinearDiscriminantAnalysis
            sk = min(a.sk_rows, n)
            Xh = np.empty((sk, d), np.float32)        # the first sk rows only
            assert b2.native.load().b2_copy_d2h(ctx._h, Xh.ctypes.data, X.ptr, Xh.nbytes) == 0, b2.native.last_error()
            yk = labels[t[:sk]]
            Xh = Xh.astype(np.float64)
            t0 = time.perf_counter()
            LinearDiscriminantAnalysis().fit(Xh, yk)
            res["sklearn_fit_s"] = {"rows": sk, "classes": k, "s": round(time.perf_counter() - t0, 2)}
        y.free()
    X.free()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
