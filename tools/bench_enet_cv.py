"""Time LassoCV / ElasticNetCV on resident rows: b2_gram_folds against one Gram pass, b2_solve_enet_cv against the
slowest of its fold paths run alone, and the whole B200LassoCV.fit; prints one JSON line.

    python tools/bench_enet_cv.py [--rows 10000000] [--d 128] [--folds 5] [--sk-rows 1000000] [--out FILE]

Tables: b2_synth fp32 rows and the correlated table of tools/bench_enet.py, 5 contiguous folds, 100 alphas, tol 1e-4.
  * folds: b2_gram_folds over all rows against one pass (b2_gram_reset + b2_gram_accumulate) over the same rows, and the
    fixed cost of one dispatch (a pass over 2 048 rows); the goal is folds <= 1.1 x (pass + (folds - 1) x fixed);
  * paths: b2_solve_enet_cv at L = 1 (lasso) and L = 7 (l1_ratio .1 .5 .7 .9 .95 .99 1) against the slowest of its
    L x folds paths run alone through b2_solve_enet_path on the same training statistic and grid; the goal is 1.25 x;
  * B200LassoCV().fit end to end on the resident rows, and scikit-learn's LassoCV on the first --sk-rows rows (host).
Times are the best of 3 (CUDA events on the context's stream).  The card's name and power limit are read in the same
run.  Writes nothing to the tree."""
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

L7 = (0.1, 0.5, 0.7, 0.9, 0.95, 0.99, 1.0)


def _best(ctx, fn, reps=3):
    out, best = None, np.inf
    for _ in range(reps):
        out, ms = _timed(ctx, fn)
        best = min(best, ms)
    return out, round(best, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--folds", type=int, default=5)
    ap.add_argument("--sk-rows", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = b2.Context(0)
    info = ctx.info()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    K = a.folds
    res = {"bench": "enet_cv", "gpu": info["name"], "power_limit": power, "rows": a.rows, "d": a.d, "folds": K,
           "n_alphas": 100, "tol": 1e-4, "tables": []}
    ids, _ = b2.fold_ids(a.rows, cv=K)
    idd = ctx.to_device(ids)
    for table in ("synth", "correlated"):
        keep = None
        if table == "synth":
            X, y = ctx.synth(a.rows, a.d)
        else:
            X, y, Xt, yt = _correlated(ctx, a.rows, a.d)
            keep = (Xt, yt)
        _, gram_ms = _best(ctx, lambda: (ctx.gram_reset(a.d), ctx.gram_accumulate(X, y)))
        Xs, ys = ctx.synth(2048, a.d)
        fixed = [_timed(ctx, lambda: (ctx.gram_reset(a.d), ctx.gram_accumulate(Xs, ys)))[1] for _ in range(5)]
        Xs.free(); ys.free()
        fixed_ms = round(min(fixed), 4)
        fold_S, folds_ms = _best(ctx, lambda: ctx.gram_folds(X, y, idd, K))
        tab = {"table": table, "gram_pass_ms": gram_ms, "dispatch_fixed_ms": fixed_ms, "gram_folds_ms": folds_ms,
               "gram_folds_goal_ratio": round(folds_ms / (gram_ms + (K - 1) * fixed_ms), 3), "paths": []}
        for l1 in ((1.0,), L7):
            ctx.gram_folds(X, y, idd, K)
            ctx.solve_enet_cv(K, l1, tol=1e-4)                                   # warm-up
            r, cv_ms = _best(ctx, lambda: ctx.solve_enet_cv(K, l1, tol=1e-4))
            single, same = [], True
            for k in range(K):
                T = np.zeros_like(fold_S[0])
                for j in range(K):
                    if j != k:
                        T = T + fold_S[j]
                ctx.gram_import(T)
                for li, ratio in enumerate(l1):
                    p, ms = _best(ctx, lambda: ctx.solve_enet_path(l1_ratio=ratio, alphas=r["alphas"][li], tol=1e-4),
                                  reps=2)
                    same = same and np.array_equal(p["n_iter"], r["n_iter"][li, k])
                    single.append(ms)
            tab["paths"].append({"n_l1": len(l1), "paths": len(l1) * K, "solve_enet_cv_ms": cv_ms,
                                 "slowest_single_path_ms": max(single), "sum_single_paths_ms": round(sum(single), 3),
                                 "ratio_to_slowest": round(cv_ms / max(single), 3), "same_sweeps_alone": bool(same),
                                 "sweeps_max_path": int(np.max(np.sum(r["n_iter"], axis=2)))})
        est = b2.B200LassoCV(cv=K, ctx=ctx)
        est.fit(X, y)
        _, fit_ms = _best(ctx, lambda: est.fit(X, y))
        tab["lasso_cv_fit_ms"] = fit_ms
        tab["lasso_cv_alpha"] = est.alpha_
        if a.sk_rows > 0:
            from sklearn.linear_model import LassoCV
            if keep is None:
                Xs, ys = ctx.synth(a.sk_rows, a.d)
                Xh, yh = Xs.to_host().astype(np.float64), ys.to_host().astype(np.float64)
                Xs.free(); ys.free()
            else:
                Xh = keep[0][: a.sk_rows].cpu().numpy().astype(np.float64)
                yh = keep[1][: a.sk_rows].cpu().numpy().astype(np.float64)
            t0 = time.perf_counter()
            sk = LassoCV(cv=K).fit(Xh, yh)
            sk_s = time.perf_counter() - t0
            t0 = time.perf_counter()
            ours = b2.B200LassoCV(cv=K, ctx=ctx).fit(Xh, yh)
            tab["lasso_cv_host_rows"] = {"rows": a.sk_rows, "sklearn_s": round(sk_s, 3), "b2_s": round(time.perf_counter() - t0, 4),
                                         "same_alpha": bool(np.isclose(ours.alpha_, sk.alpha_, rtol=1e-6)),
                                         "coef_diff": float(np.max(np.abs(ours.coef_ - sk.coef_)))}
        res["tables"].append(tab)
        X.free(); y.free()
        keep = None
    idd.free()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
