"""Time RidgeCV's leave-one-out search (b2_ridge_loo) against the plain fit (b2_fit) on resident rows; prints one JSON line.

    python tools/bench_ridge_cv.py [--rows 10000000] [--d 128] [--reps 5] [--sk-rows 1000000] [--out FILE]

Tables: b2_synth rows in fp32 and in bf16.  Per table and per number of alphas A in {1, 13, 64}: the median wall time of
b2_ridge_loo and of b2_fit on the same rows (every call ends in a device synchronisation), the per-kernel device times of
one b2_ridge_loo from torch.profiler (CUPTI), and the pass's achieved fp64 rate from its flop count n (2 D^2 + 4 A D)
over the device time of loo_kernel, beside NVIDIA's 67 TFLOP/s FP64 tensor-core figure for the H100 SXM.  For context,
scikit-learn's RidgeCV on a host subset of fp32 rows.  The card's name and power limit are read in the same run.
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

FP64_TC_TFLOPS = 67.0        # NVIDIA H100 SXM data sheet, dense FP64 tensor core


def _median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def _kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            key = ev.name.replace("(anonymous namespace)::", "").split("(")[0].replace("void b2::", "")
            key = key.split("<")[0]
            out[key] = round(out.get(key, 0.0) + ev.device_time_total / 1e3, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
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
    res = {"bench": "ridge_cv", "gpu": info["name"], "power_limit": power, "rows": a.rows, "d": a.d, "tables": []}
    for kind in ("f32", "bf16"):
        X, y = ctx.synth(a.rows, a.d, kind=kind)
        tab = {"rows": kind, "fit_ms": round(_median_ms(lambda: ctx.fit(X, y, alpha=1.0), a.reps), 3), "alphas": []}
        for n_al in (1, 13, 64):
            grid = list(np.logspace(-2, 4, n_al)) if n_al > 1 else [1.0]
            wall = _median_ms(lambda: ctx.ridge_loo(X, y, grid), a.reps)
            k = _kernels(lambda: ctx.ridge_loo(X, y, grid))
            t_pass = k.get("loo_kernel", 0.0)
            flops = a.rows * (2 * a.d * a.d + 4 * n_al * a.d)
            tflops = flops / (t_pass * 1e-3) / 1e12 if t_pass > 0 else 0.0
            tab["alphas"].append({"n_alphas": n_al, "ridge_loo_ms": round(wall, 3), "kernels_ms": k,
                                  "loo_pass_tflops": round(tflops, 2),
                                  "fraction_of_fp64_tc_datasheet": round(tflops / FP64_TC_TFLOPS, 3)})
        res["tables"].append(tab)
        X.free(); y.free()
    if a.sk_rows > 0:
        from sklearn.linear_model import RidgeCV
        Xs, ys = ctx.synth(a.sk_rows, a.d)
        Xh, yh = Xs.to_host().astype(np.float64), ys.to_host().astype(np.float64)
        Xs.free(); ys.free()
        grid = list(np.logspace(-2, 4, 13))
        t0 = time.perf_counter()
        sk = RidgeCV(alphas=grid).fit(Xh, yh)
        res["sklearn_ridgecv_13_alphas"] = {"rows": a.sk_rows, "s": round(time.perf_counter() - t0, 3),
                                            "alpha": float(sk.alpha_)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
