"""Time the elastic-net path (b2_solve_enet_path) on resident rows against the Gram pass and scikit-learn; prints one
JSON line.

    python tools/bench_enet.py [--rows 10000000] [--d 128] [--sk-rows 1000000] [--out FILE]

Tables: b2_synth fp32 rows (independent U(0, 100) columns) and a correlated table (Gaussian columns sharing one common
factor, rho = 0.5, half of the true coefficients zero).  Per table: the Gram pass (b2_gram_reset + b2_gram_accumulate)
and each path call timed with CUDA events on the context's stream; for a 100-alpha lasso path and an l1_ratio = 0.5 path
at tol 1e-4 and 1e-10: the total sweeps, the time per sweep and per coordinate visit (sweeps x D, an upper bound on the
visits: screening shrinks the active set).  For context, scikit-learn's Gram coordinate descent
(enet_coordinate_descent_gram, the solver alone) on the same fp64 Q, q, ||yc||^2 on the host, and Lasso().fit on the
first --sk-rows rows (end to end).  The card's name and power limit are read in the same run.  Writes nothing to the
tree."""
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


def _correlated(ctx, n, d, seed=7):
    """(X, y) DeviceArrays of a correlated fp32 table built with torch on the device, and the host copy of its first rows
    (callers slice)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn(n, d, device="cuda", generator=g, dtype=torch.float32)
    X.mul_(0.5).add_(0.5 * X[:, :1])
    beta = torch.rand(d, device="cuda", generator=g, dtype=torch.float32) * 2 - 1
    beta[torch.rand(d, device="cuda", generator=g) < 0.5] = 0.0
    y = X @ beta + torch.randn(n, device="cuda", generator=g, dtype=torch.float32)
    torch.cuda.synchronize()
    Xd, yd = ctx.empty((n, d), "f32"), ctx.empty((n,), "f32")
    lib = b2.native.load()
    for dst, src in ((Xd, X), (yd, y)):
        assert lib.b2_copy_d2d(ctx._h, dst.ptr, src.data_ptr(), dst.nbytes) == 0
    ctx.sync()
    return Xd, yd, X, y


def _timed(ctx, fn):
    ctx.sync()
    ctx.timer_start()
    out = fn()
    return out, ctx.timer_stop()


def _sk_solver(S, l1_ratio, alphas, tol, max_iter=1000):
    """sklearn's Gram coordinate descent alone, over the same alphas and warm starts as enet_path."""
    from sklearn.linear_model._cd_fast import enet_coordinate_descent_gram
    d = S.shape[0] - 2
    n = S[d, d]
    m, ybar = S[:d, d] / n, S[d, d + 1] / n
    Q = np.ascontiguousarray(S[:d, :d] - n * np.outer(m, m))
    q = np.ascontiguousarray(S[:d, d + 1] - n * m * ybar)
    yv = np.array([np.sqrt(max(S[d + 1, d + 1] - n * ybar * ybar, 0.0))])   # only y.y enters: the gap tolerance
    w = np.zeros(d)
    rng = np.random.RandomState(0)
    sweeps = 0
    t0 = time.perf_counter()
    for a in alphas:
        w, _, _, it = enet_coordinate_descent_gram(w, a * l1_ratio * n, a * (1 - l1_ratio) * n, Q, q, yv, max_iter,
                                                   tol, rng, False, False, True)
        sweeps += int(it)
    return (time.perf_counter() - t0) * 1e3, sweeps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
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
    res = {"bench": "enet", "gpu": info["name"], "power_limit": power, "rows": a.rows, "d": a.d, "tables": []}
    for table in ("synth", "correlated"):
        if table == "synth":
            X, y = ctx.synth(a.rows, a.d)
            keep = None
        else:
            X, y, Xt, yt = _correlated(ctx, a.rows, a.d)
            keep = (Xt, yt)
        gram = []
        for _ in range(3):
            _, ms = _timed(ctx, lambda: (ctx.gram_reset(a.d), ctx.gram_accumulate(X, y)))
            gram.append(ms)
        S = ctx.gram_export()
        tab = {"table": table, "gram_ms": round(min(gram), 3), "paths": []}
        for name, l1_ratio in (("lasso_path", 1.0), ("enet_path l1_ratio 0.5", 0.5)):
            for tol in (1e-4, 1e-10):
                ctx.solve_enet_path(l1_ratio=l1_ratio, tol=tol)               # warm-up
                r, ms = _timed(ctx, lambda: ctx.solve_enet_path(l1_ratio=l1_ratio, tol=tol))
                sweeps = int(np.sum(r["n_iter"]))
                sk_ms, sk_sweeps = _sk_solver(S, l1_ratio, r["alphas"], tol)
                tab["paths"].append({"path": name, "tol": tol, "n_alphas": int(r["alphas"].size),
                                     "path_ms": round(ms, 3), "sweeps": sweeps,
                                     "us_per_sweep": round(1e3 * ms / max(sweeps, 1), 3),
                                     "ns_per_coordinate": round(1e6 * ms / max(sweeps * a.d, 1), 2),
                                     "unconverged_alphas": int(np.sum(r["gaps"] > r["tol"])),
                                     "sklearn_solver_ms": round(sk_ms, 2), "sklearn_sweeps": sk_sweeps})
        if a.sk_rows > 0:
            from sklearn.linear_model import Lasso
            if keep is None:
                Xs, ys = ctx.synth(a.sk_rows, a.d)
                Xh, yh = Xs.to_host().astype(np.float64), ys.to_host().astype(np.float64)
                Xs.free(); ys.free()
            else:
                Xh = keep[0][: a.sk_rows].cpu().numpy().astype(np.float64)
                yh = keep[1][: a.sk_rows].cpu().numpy().astype(np.float64)
            t0 = time.perf_counter()
            sk = Lasso().fit(Xh, yh)
            sk_s = time.perf_counter() - t0
            ours = b2.B200Lasso(ctx=ctx)
            t0 = time.perf_counter()
            ours.fit(Xh, yh)
            tab["lasso_fit_host_rows"] = {"rows": a.sk_rows, "sklearn_s": round(sk_s, 3), "sklearn_n_iter": int(sk.n_iter_),
                                          "b2_s": round(time.perf_counter() - t0, 4), "b2_n_iter": ours.n_iter_,
                                          "coef_diff": float(np.max(np.abs(ours.coef_ - sk.coef_)))}
        res["tables"].append(tab)
        X.free(); y.free()
        keep = None
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
