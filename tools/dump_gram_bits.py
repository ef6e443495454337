"""Dump the tensor-core Gram statistic and the fit of a fixed grid of cases, to compare two builds bit for bit.

    python tools/dump_gram_bits.py --out FILE.npz            # with the in-tree library, or B2_LIB_PATH=... for another
    python tools/dump_gram_bits.py --compare A.npz B.npz     # every array equal byte for byte?

Grid: fp32 and bf16 rows x hi + lo and single-operand precision x d = 128 (fixed-D kernel; bf16: the raw tile is the
B operand), 96 (runtime d), 64, 40 and 20 (2, 3 and 5 rows packed to a super-row; 24 for bf16 rows, whose rows
must be whole 16-byte vectors) x rows unmasked and masked (keep = 1 of
a seeded 0/1 mask) x drain_rows = 64, 8 192 and 1 << 30 x three row counts: 1 689 637 (200 tiles per CTA on 132 SMs: a
128-tile chunk and a partial one), 70 001 (one chunk per CTA at 8 192) and 5 000 on one CTA (set_sm_limit(1)).  Per
case: S = gram_export() after gram_reset + gram_accumulate, and coef / intercept of fit() on the same rows.  Rows are
device Philox rows (b2_synth, fixed seeds), so two builds on one GPU see the same input.  Prints one JSON line."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS = (128, 96, 64, 40, 20)
DRAINS = (64, 8192, 1 << 30)
ROWS = ((1_689_637, 0), (70_001, 0), (5_000, 1))        # (rows, sm_limit: 0 = every SM)


def dump(out):
    import bodywork_mlops_demo_b200 as b2
    ctx = b2.Context(0)
    res = {}
    for kind in ("f32", "bf16"):
        for d in (DS if kind == "f32" else DS[:-1] + (24,)):
            for n, sm_limit in ROWS:
                X, y = ctx.synth(n, d, seed=100 + d + n % 97, kind=kind)
                mask = (np.random.RandomState(d + n % 89).rand(n) < 0.7).astype(np.uint8)
                md = ctx.to_device(mask)
                for masked in (False, True):
                    for prec in ("split", "bf16"):
                        for drain in DRAINS:
                            ctx.set_kernel(b2.KERNEL_TCGEN05)
                            ctx.set_precision(b2.PRECISION_SPLIT if prec == "split" else b2.PRECISION_BF16)
                            ctx.set_drain_rows(drain)
                            ctx.set_sm_limit(sm_limit)
                            m = md if masked else None
                            ctx.gram_reset(d)
                            ctx.gram_accumulate(X, y, m, 1)
                            S = ctx.gram_export()
                            try:
                                coef, b0 = ctx.fit(X, y, row_mask=m, mask_keep=1)
                            except np.linalg.LinAlgError:        # a refused solve is compared as NaN
                                coef, b0 = np.full(d, np.nan), np.nan
                            key = f"{kind}-d{d}-n{n}-sm{sm_limit}-{'masked' if masked else 'all'}-{prec}-drain{drain}"
                            res[key + "-S"] = S
                            res[key + "-coef"] = np.asarray(coef, dtype=np.float64)
                            res[key + "-intercept"] = np.asarray([b0], dtype=np.float64)
                md.free(); X.free(); y.free()
    ctx.set_drain_rows(8192)
    ctx.set_precision(b2.PRECISION_SPLIT)
    info = ctx.info()
    ctx.close()
    np.savez(out, **res)
    print(json.dumps({"dump": out, "lib": os.environ.get("B2_LIB_PATH", "in-tree"), "gpu": info["name"],
                      "arrays": len(res), "cases": len(res) // 3}))


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    keys_a, keys_b = set(a.files), set(b.files)
    differ = sorted(k for k in keys_a & keys_b if a[k].dtype != b[k].dtype or a[k].shape != b[k].shape
                    or a[k].tobytes() != b[k].tobytes())
    res = {"a": a_path, "b": b_path, "arrays": len(keys_a & keys_b), "only_in_one": sorted(keys_a ^ keys_b),
           "differ": len(differ), "first_differences": differ[:10]}
    res["bit_identical"] = not differ and not res["only_in_one"]
    print(json.dumps(res))
    return 0 if res["bit_identical"] else 1


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("--out or --compare is required")
    dump(args.out)
