"""Time RidgeClassifierCV's leave-one-out search (b2_ridge_classifier_loo) on resident rows; prints one JSON line.

    python tools/bench_ridge_classifier_cv.py [--rows 10000000] [--d 128] [--reps 3] [--out FILE]

Rows: b2_synth fp32 rows, labelled by the quantiles of their synthetic y into K classes.  Per K in {2, 10, 32} and number
of alphas A in {3, 13, 64}: the median wall time of b2_ridge_classifier_loo (every call ends in a device
synchronisation), the per-kernel device times of one more call from torch.profiler (CUPTI), the call's time outside the
Gram, class-sum, eigendecomposition and leave-one-out kernels (the median wall time minus those kernels' device times;
the profiler is not running while the wall time is taken, its own cost would dwarf what is measured), and the pass's
achieved fp64 rate from its flop count n (2 D^2 + 2 D A + 2 D T A), T = 1 for K = 2 else K, over the device time of
loo_classes_kernel.  Beside it, b2_ridge_loo's loo_kernel at the same A on the same rows.  The card's name and power
limit are read in the same run.  Writes nothing to the tree."""
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
# the kernels the whole call is compared against: the Gram (gram_*, its shift sample and finalize), the class sums, the
# eigendecomposition and the pass
PARTS = ("tc_shift_kernel", "tc_finalize_kernel", "class_sums_kernel", "solve_eigh_kernel", "loo_classes_kernel")


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
            # "void b2::(anonymous namespace)::f<...>(...)" for templates, "b2::(anonymous namespace)::f(...)" otherwise
            key = ev.name.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0]
            key = key.removeprefix("void ").removeprefix("b2::")
            out[key] = round(out.get(key, 0.0) + ev.device_time_total / 1e3, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = b2.Context(0)
    info = ctx.info()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    res = {"bench": "ridge_classifier_cv", "gpu": info["name"], "power_limit": power, "rows": a.rows, "d": a.d,
           "ridge_loo": [], "runs": []}
    X, y = ctx.synth(a.rows, a.d)
    yh = y.to_host()
    grids = {A: list(np.logspace(-2, 4, A)) for A in (3, 13, 64)}
    for A, grid in grids.items():
        k = _kernels(lambda: ctx.ridge_loo(X, y, grid))
        res["ridge_loo"].append({"n_alphas": A, "loo_kernel_ms": k.get("loo_kernel", 0.0)})
    ref = {r["n_alphas"]: r["loo_kernel_ms"] for r in res["ridge_loo"]}
    for K in (2, 10, 32):
        cuts = np.quantile(yh, np.arange(1, K) / K)
        labels = np.digitize(yh, cuts).astype(np.float32)
        classes = np.arange(K, dtype=np.float32)
        yk = ctx.to_device(labels)
        T = 1 if K == 2 else K
        for A, grid in grids.items():
            run = lambda: ctx.ridge_classifier_loo(X, yk, classes, grid)          # noqa: E731
            wall = _median_ms(run, a.reps)
            k = _kernels(run)
            t_pass = k.get("loo_classes_kernel", 0.0)
            parts = sum(v for name, v in k.items() if name in PARTS or name.startswith("gram"))
            flops = a.rows * (2 * a.d * a.d + 2 * a.d * A + 2 * a.d * T * A)
            tflops = flops / (t_pass * 1e-3) / 1e12 if t_pass > 0 else 0.0
            res["runs"].append({"K": K, "n_alphas": A, "call_ms": round(wall, 3), "kernels_ms": k,
                                "loo_pass_ms": t_pass, "pass_vs_ridge_loo": round(t_pass / ref[A], 3),
                                "outside_parts_ms": round(wall - parts, 3), "loo_pass_tflops": round(tflops, 2),
                                "fraction_of_fp64_tc_datasheet": round(tflops / FP64_TC_TFLOPS, 3)})
        yk.free()
    X.free()
    y.free()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
