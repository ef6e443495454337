"""Time what the single rank rule adds to a solve from a resident statistic (``partial_fit``, ``solve_resident``,
``fit(with_spectrum=False)`` with alpha = 0): the eigenvalue kernel (b2_solve_eigvals) after the LDL^T solve (b2_solve),
and the minimum-norm kernel (b2_solve_spectral) where the rank rule picks it; prints one JSON line.

    python tools/bench_rank_rule.py [--d 128] [--reps 200]

The statistic is a seeded full-rank one (well-conditioned fp32 rows), imported once; every call ends in a device
synchronisation, so each figure is the median wall time of one synchronous call.  Writes nothing to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bodywork_mlops_demo_b200 as b2  # noqa: E402
from oracle import ols_oracle as orc  # noqa: E402


def _median_us(fn, reps):
    for _ in range(5):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e6)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    ctx = b2.Context(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    X, y = orc.generate_dataset(20_000, a.d, seed=3)
    S = orc.gram_stats(X, y)
    ctx.gram_import(S)
    res = {"bench": "rank_rule", "gpu": ctx.info()["name"], "power_limit": power, "d": a.d, "reps": a.reps}
    res["solve_us"] = _median_us(lambda: ctx.solve(), a.reps)
    res["eigvals_us"] = _median_us(lambda: ctx.solve_eigvals(), a.reps)
    res["spectral_us"] = _median_us(lambda: ctx.solve_spectral(), a.reps)
    est = b2.B200LinearRegression(ctx=ctx)
    res["solve_resident_us"] = _median_us(lambda: est.solve_resident(a.d, S), a.reps)
    ridge = b2.B200LinearRegression(ctx=ctx, alpha=1e-3)
    res["solve_resident_ridge_us"] = _median_us(lambda: ridge.solve_resident(a.d, S), a.reps)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
