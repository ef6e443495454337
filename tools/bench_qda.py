"""Time QuadraticDiscriminantAnalysis on resident rows: the per-class scatter pass (class-order step included) next to
the pooled within-class scatter pass on the same rows, with balanced and skewed labels; the K host eigendecompositions;
svd fits; the decision pass, predict and predict_proba, for several class counts; prints one JSON line.

    python tools/bench_qda.py [--rows 10000000] [--d 128] [--classes 2,10,32] [--sk-rows 1000000] [--out FILE]

Rows: fp32 b2_synth rows (seed 1234).  Balanced labels are the K quantile bins of their synthetic y, labelled 3 k - 7;
skewed labels put the lowest 95 % of y in class 0 and the rest in K - 1 quantile bins.  Pass times are CUDA events on
the context's stream around the whole call (uploads and the copy of the sums included), best of 3 after a warm-up.  The
host solver is host wall clock on the scatters of the run.  Fits are host wall clock around ``fit`` on the device rows
with device labels (label scan and label discovery included), median of 3 after a warm-up; predictions are host wall
clock on device rows with the device outputs, best of 3.  For context, scikit-learn's QDA on the first --sk-rows rows as
host float64 at K = 10, end to end.  The card's name and power limit are read in the same run.  Writes nothing to the
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
from bodywork_mlops_demo_b200 import estimator as est_mod  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_lda import _best, _host_ms, _wall  # noqa: E402


def _labels(yh, k, skewed):
    """class indices of the rows: K quantile bins of y, or 95 % in class 0 and K - 1 bins of the rest"""
    if not skewed:
        return np.searchsorted(np.quantile(yh, np.linspace(0, 1, k + 1)[1:-1]), yh)
    q = np.quantile(yh, 0.95)
    hi = yh > q
    t = np.zeros(yh.size, np.int64)
    t[hi] = 1 + np.searchsorted(np.quantile(yh[hi], np.linspace(0, 1, k)[1:-1]), yh[hi])
    return t


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
    res = {"bench": "qda", "gpu": ctx.info()["name"], "power_limit": power, "rows": n, "d": d, "per_k": {}}
    X, ys = ctx.synth(n, d, seed=1234)
    yh = ys.to_host()
    ys.free()
    for k in [int(v) for v in a.classes.split(",")]:
        labels = (3.0 * np.arange(k) - 7.0).astype(np.float32)
        r = {}
        for skewed in (False, True):
            t = _labels(yh, k, skewed)
            y = ctx.to_device(labels[t].astype(np.float32))
            cs = ctx.class_sums(X, y, labels)
            nk = cs["sums"][:, d]
            means = cs["sums"][:, :d] / nk[:, None]
            p = {"largest_class_share": round(float(nk.max() / nk.sum()), 3)}
            p["scatters_ms"] = _best(ctx, lambda: ctx.class_scatters(X, y, labels, means))
            p["pooled_scatter_ms"] = _best(ctx, lambda: ctx.class_scatter(X, y, labels, means))
            p["scatters_over_pooled"] = round(p["scatters_ms"] / p["pooled_scatter_ms"], 3)
            r["skewed" if skewed else "balanced"] = p
            if skewed:
                y.free()
                continue
            sc = ctx.class_scatters(X, y, labels, means)["scatters"]
            r["label_discovery_ms"] = _best(ctx, lambda: (ctx.label_scan(y), ctx.label_values(y)))
            r["class_sums_ms"] = _best(ctx, lambda: ctx.class_sums(X, y, labels))
            r["host_eigh_ms"] = _host_ms(lambda: [est_mod._qda_class(sc[j], nk[j], "svd", None, 0.0)
                                                  for j in range(k)])
            est = b2.B200QuadraticDiscriminantAnalysis(ctx=ctx)
            r["fit_svd_ms"] = _wall(ctx, lambda: est.fit(X, y), median=True)
            ops = est._operands()
            cl = est._fp32_classes(est.classes_)
            r["decision_pass_ms"] = _wall(ctx, lambda: ctx.qda_decision(X, *ops, cl, decision=True))
            r["decision_fp64_tflops"] = round(2.0 * k * d * d * n / r["decision_pass_ms"] * 1e-9, 2)
            r["predict_ms"] = _wall(ctx, lambda: est.predict(X))
            r["predict_proba_ms"] = _wall(ctx, lambda: est.predict_proba(X))
            budget = r["label_discovery_ms"] + r["class_sums_ms"] + p["scatters_ms"] + r["host_eigh_ms"] + 2.0
            r["goals"] = {"fit_le_parts_plus_2ms": r["fit_svd_ms"] <= budget, "fit_budget_ms": round(budget, 2),
                          "decision_ge_15_tflops": r["decision_fp64_tflops"] >= 15.0,
                          "predict_le_pass_plus_1ms": None if k > 10 else
                          r["predict_ms"] <= r["decision_pass_ms"] + 1.0}
            if k == 10 and a.sk_rows > 0:
                from sklearn.discriminant_analysis import QuadraticDiscriminantAnalysis
                sk = min(a.sk_rows, n)
                Xh = np.empty((sk, d), np.float32)        # the first sk rows only
                assert b2.native.load().b2_copy_d2h(ctx._h, Xh.ctypes.data, X.ptr, Xh.nbytes) == 0, \
                    b2.native.last_error()
                Xh = Xh.astype(np.float64)
                t0 = time.perf_counter()
                QuadraticDiscriminantAnalysis().fit(Xh, labels[t[:sk]]).predict(Xh)
                res["sklearn_fit_predict_s"] = {"rows": sk, "classes": k, "s": round(time.perf_counter() - t0, 2)}
            y.free()
        r["goals"]["scatters_within_1.2x_pooled"] = all(r[s]["scatters_over_pooled"] <= 1.2
                                                        for s in ("balanced", "skewed"))
        res["per_k"][str(k)] = r
    X.free()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
