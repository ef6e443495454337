"""What the Gram kernel's chunk drains cost: its time with the default drain_rows against one drain per CTA.

    python tools/bench_drain.py [--rows 12500000] [--x-dtype f32|bf16] [--precision split|bf16] [--rounds 4]
                                [--fits 10] [--out FILE]

Fits the bench.py shard (b2_synth rows, seed 1234, D = 128) on the tensor-core path and reads the Gram kernel's device
time (`last_kernel_ms`, CUDA events around each launch) over `--fits` fits per setting and round, the two settings
alternating round by round: `drain_rows` = 8 192 (the default) and 1 << 30, which leaves one drain per CTA, at the end of
its range.  The second setting sums longer fp32 chains, so its results are less accurate; its time is the kernel without
the periodic drains, the most that cheaper drains can gain.  The card's name and power limit are read in the same run.
Prints one JSON line; writes nothing to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bodywork_mlops_demo_b200 as b2  # noqa: E402

DEFAULT_DRAIN_ROWS = 8192
NO_DRAIN_ROWS = 1 << 30


def _query(field):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=12_500_000)
    ap.add_argument("--x-dtype", default="f32", choices=["f32", "bf16"])
    ap.add_argument("--precision", default="split", choices=["split", "bf16"])
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--fits", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = b2.Context(0)
    X, y = ctx.synth(a.rows, 128, seed=1234, kind=a.x_dtype)
    ctx.set_kernel(b2.KERNEL_TCGEN05)
    ctx.set_precision(b2.PRECISION_BF16 if a.precision == "bf16" else b2.PRECISION_SPLIT)
    settings = {"default": DEFAULT_DRAIN_ROWS, "one_drain": NO_DRAIN_ROWS}
    per_round = {k: [] for k in settings}
    for _ in range(a.rounds):
        for key, rows in settings.items():
            ctx.set_drain_rows(rows)
            for _ in range(2):
                ctx.fit(X, y)
            ctx.sync()
            ctx.last_kernel_ms()                   # drops the warm-up launches
            for _ in range(a.fits):
                ctx.fit(X, y)
            ctx.sync()
            ms, n = ctx.last_kernel_ms()
            per_round[key].append(ms / max(n, 1))
    ctx.set_drain_rows(DEFAULT_DRAIN_ROWS)
    res = {"bench": "drain", "lib": os.environ.get("B2_LIB_PATH", "in-tree"), "gpu": ctx.info()["name"],
           "power_limit": _query("power.limit"), "sm_clock_max": _query("clocks.max.sm"), "rows": a.rows,
           "x_dtype": a.x_dtype, "precision": a.precision, "launches_per_setting": a.rounds * a.fits}
    for key in settings:
        v = per_round[key]
        res[f"gram_ms_{key}"] = {"median": round(statistics.median(v), 4), "min": round(min(v), 4),
                                 "max": round(max(v), 4), "rounds": [round(t, 4) for t in v]}
    res["drain_cost_ms"] = round(res["gram_ms_default"]["median"] - res["gram_ms_one_drain"]["median"], 4)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    X.free(); y.free()
    ctx.close()


if __name__ == "__main__":
    main()
