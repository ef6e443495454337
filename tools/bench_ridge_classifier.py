"""Time RidgeClassifier on resident rows: the Gram, the class-sum pass next to one b2_score pass over the same rows, the
multi-target solve, whole fits, predict and decision_function, for several class counts; prints one JSON line.

    python tools/bench_ridge_classifier.py [--rows 10000000] [--d 128] [--classes 2,10,32] [--sk-rows 1000000] [--out FILE]

Rows: fp32 X ~ N(0, 1) drawn on the device with torch; the K labels 3 k - 7 of argmax_k (X B + noise), B ~ N(0, 1).  Pass
times are CUDA events on the context's stream around the whole call (uploads and the copy of the sums included), best of
3 after a warm-up.  Fits are host wall clock around ``fit`` on the device rows with device labels (label scan and label
discovery included).  For context, scikit-learn's RidgeClassifier on the first --sk-rows rows as host float64 with the
middle class count, end to end.  The card's name and power limit are read in the same run.  Writes nothing to the
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
from bodywork_mlops_demo_b200 import _native as native  # noqa: E402


def _best(ctx, fn, reps=3):
    fn()
    best = float("inf")
    for _ in range(reps):
        ctx.sync()
        ctx.timer_start()
        fn()
        best = min(best, ctx.timer_stop())
    return round(best, 3)


def _wall(ctx, fn, reps=3):
    fn()
    best = float("inf")
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        fn()
        ctx.sync()
        best = min(best, (time.perf_counter() - t0) * 1e3)
    return round(best, 2)


def _device_copy(ctx, t, kind, shape):
    out = ctx.empty(shape, kind)
    import torch
    torch.cuda.synchronize()
    assert native.load().b2_copy_d2d(ctx._h, out.ptr, t.data_ptr(), t.numel() * t.element_size()) == 0, \
        native.last_error()
    return out


def main():
    import torch
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
    ks = [int(k) for k in a.classes.split(",")]
    res = {"bench": "ridge_classifier", "gpu": ctx.info()["name"], "power_limit": power, "rows": n, "d": d}
    g = torch.Generator(device="cuda").manual_seed(0)
    Xt = torch.randn(n, d, device="cuda", generator=g, dtype=torch.float32)
    X = _device_copy(ctx, Xt, "f32", (n, d))
    coef = np.random.default_rng(0).normal(size=d) / np.sqrt(d)
    per_k = {}
    for k in ks:
        B = torch.randn(d, k, device="cuda", generator=g, dtype=torch.float32)
        t = torch.argmax(Xt @ B + torch.randn(n, k, device="cuda", generator=g), dim=1)
        yk = _device_copy(ctx, (t.float() * 3 - 7).contiguous(), "f32", (n,))
        classes = np.arange(k, dtype=np.float32) * 3 - 7
        if "gram_ms" not in res:                    # the rows and their Gram do not depend on the labels
            res["gram_ms"] = _best(ctx, lambda: (ctx.gram_reset(d), ctx.gram_accumulate(X, yk)))
            res["score_pass_ms"] = _best(ctx, lambda: ctx.score(X, coef, 0.1, y=yk, want_yhat=False))
        ctx.gram_reset(d)
        ctx.gram_accumulate(X, yk)
        S = ctx.gram_export()
        center = S[:d, d] / S[d, d]
        r = {"class_sums_ms": _best(ctx, lambda: ctx.class_sums(X, yk, classes, center))}
        r["solve_ms"] = _best(ctx, lambda: ctx.solve_classes(None, 1.0, True, n_classes=k))
        est = b2.B200RidgeClassifier(alpha=1.0, ctx=ctx)
        r["fit_ms"] = _wall(ctx, lambda: est.fit(X, yk))
        r["predict_ms"] = _best(ctx, lambda: est.predict(X).free())
        r["decision_function_ms"] = _best(ctx, lambda: est.decision_function(X).free())
        r["class_sums_over_score"] = round(r["class_sums_ms"] / res["score_pass_ms"], 3)
        r["fit_minus_gram_and_class_sums_ms"] = round(r["fit_ms"] - res["gram_ms"] - r["class_sums_ms"], 2)
        r["predict_over_score"] = round(r["predict_ms"] / res["score_pass_ms"], 3)
        per_k[str(k)] = r
        yk.free()
    res["per_classes"] = per_k
    if a.sk_rows > 0:
        from sklearn import linear_model
        k = ks[len(ks) // 2]
        m = min(a.sk_rows, n)
        Xh = Xt[:m].double().cpu().numpy()
        B = np.random.default_rng(1).normal(size=(d, k))
        yh = np.argmax(Xh @ B + np.random.default_rng(2).normal(size=(m, k)), axis=1)
        t0 = time.perf_counter()
        linear_model.RidgeClassifier(alpha=1.0).fit(Xh, yh)
        res["sklearn_rows"], res["sklearn_classes"] = m, k
        res["sklearn_fit_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    X.free()
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
