"""Time the refined fit (b2_fit_refined) against the plain fit, the exact SIMT fit and scoring on resident fp32 rows, and
measure its coefficient error against the SIMT fit; prints one JSON line.

    python tools/bench_refine.py [--rows 10000000] [--d 128] [--reps 5] [--rho 0.999]

Two tables: the benchmark's synthetic rows (b2_synth, independent columns, kappa ~ 1) and a seeded table of correlated
blocks (8 columns with pairwise correlation rho; kappa ~ 8e3 at rho = 0.999), built on the host in chunks.  Per table:
median wall time of each call (every call ends in a device synchronisation), the per-kernel device times of one refined
pass from torch.profiler (CUPTI), and the scale-free coefficient error max_j |coef_j - coef_simt_j| sigma_j.
Writes nothing to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bodywork_mlops_demo_b200 as b2  # noqa: E402
from oracle import ols_oracle as orc  # noqa: E402


def _median_ms(fn, reps):
    fn()
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def _correlated(ctx, n, d, rho, seed=2024, chunk=500_000):
    X = ctx.empty((n, d), "f32")
    y = ctx.empty((n,), "f32")
    rng = np.random.RandomState(seed)
    beta = rng.uniform(0.5, 2.0, size=d) * rng.choice([-1.0, 1.0], size=d)
    lib = b2.native.load()
    for r0 in range(0, n, chunk):
        rows = min(chunk, n - r0)
        Xc = np.empty((rows, d), dtype=np.float32)
        for b0 in range(0, d, 8):
            w = min(8, d - b0)
            common = rng.standard_normal((rows, 1)).astype(np.float32)
            Xc[:, b0:b0 + w] = np.sqrt(rho) * common + np.sqrt(1.0 - rho) * rng.standard_normal((rows, w)).astype(np.float32)
        yc = (3.0 + Xc.astype(np.float64) @ beta + rng.standard_normal(rows)).astype(np.float32)
        b2.native._check(lib.b2_copy_h2d(ctx._h, X.ptr + r0 * d * 4, Xc.ctypes.data, Xc.nbytes), "b2_copy_h2d")
        b2.native._check(lib.b2_copy_h2d(ctx._h, y.ptr + r0 * 4, yc.ctypes.data, yc.nbytes), "b2_copy_h2d")
    return X, y


def _pass_kernels(ctx, X, y):
    """device time per kernel name of one refined pass: the difference of a 2-pass and a 1-pass refined fit"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    def kernels(passes):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.fit_refined(X, y, max_passes=passes, tol=0.0)
        out = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                key = ev.name.replace("(anonymous namespace)::", "").split("(")[0].replace("void b2::", "")
                out[key] = out.get(key, 0.0) + ev.device_time_total / 1e3
        return out
    one, two = kernels(1), kernels(2)
    return {k: round(two.get(k, 0.0) - one.get(k, 0.0), 4) for k in two if two.get(k, 0.0) - one.get(k, 0.0) > 0.0}


def run_table(ctx, name, X, y, reps, profile):
    out = {"table": name}
    ctx.set_kernel(b2.KERNEL_SIMT)
    out["simt_fit_ms"] = round(_median_ms(lambda: ctx.fit(X, y), max(2, reps // 2)), 3)
    c_simt, b_simt = ctx.fit(X, y)
    S = ctx.gram_export()
    ctx.set_kernel(b2.KERNEL_AUTO)
    out["kappa"] = float(f"{orc.centred_condition(S):.4g}")
    out["fit_ms"] = round(_median_ms(lambda: ctx.fit(X, y), reps), 3)
    c0, b0 = ctx.fit(X, y)
    errs = [orc.coef_error(c0, c_simt, S)]
    for p in (1, 2, 3):
        out[f"refined_{p}_ms"] = round(_median_ms(lambda: ctx.fit_refined(X, y, max_passes=p, tol=0.0), reps), 3)
        c, b, kept, step = ctx.fit_refined(X, y, max_passes=p, tol=0.0)
        errs.append(orc.coef_error(c, c_simt, S))
        out[f"refined_{p}_kept_step"] = [kept, float(f"{step:.3g}")]
    out["coef_err_vs_simt_by_passes"] = [float(f"{e:.3g}") for e in errs]
    out["contraction_per_pass"] = [float(f"{b_ / a:.3g}") if a > 0 else None for a, b_ in zip(errs, errs[1:])]
    out["score_ms"] = round(_median_ms(lambda: ctx.score(X, c0, b0, y=y, want_yhat=False), reps), 3)
    if profile:
        out["one_pass_kernel_ms"] = _pass_kernels(ctx, X, y)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rho", type=float, default=0.999)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    ctx = b2.Context(0)
    info = ctx.info()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    res = {"bench": "refine", "gpu": info["name"], "power_limit": power, "rows": a.rows, "d": a.d}
    X, y = ctx.synth(a.rows, a.d, seed=1234)
    res["synth"] = run_table(ctx, "synth", X, y, a.reps, not a.no_profile)
    X.free(); y.free()
    X, y = _correlated(ctx, a.rows, a.d, a.rho)
    res["correlated"] = run_table(ctx, f"correlated rho={a.rho}", X, y, a.reps, not a.no_profile)
    X.free(); y.free()
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
