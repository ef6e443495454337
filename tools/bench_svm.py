"""Time LinearSVC's trust-region Newton fit on resident rows: b2_svm_pass at changed fractions 0, about 1 %, about 10 %
and 1 next to the binary logistic gradient and Newton passes on the same rows, whole binary fits on a noisy and a nearly
separable label set with, per iteration, the active and changed fractions and the rejected steps, the same fits with a
full active Gram per pass (coef_from = NULL), and scikit-learn for context; prints one JSON line.

    python tools/bench_svm.py [--rows 10000000] [--d 128] [--sk-rows 1000000] [--out FILE]

Rows: fp32 X ~ N(0, 1) drawn on the device with torch; noisy labels 0 / 1 from expit(X beta + 0.2), beta ~ N(0, 1 /
sqrt(d)); nearly separable labels sign(X beta) with 0.1 % of them flipped.  Pass times are CUDA events on the context's
stream around the whole call, best of 3 after a warm-up.  Fits are host wall clock around ``fit`` on the device rows
with device labels, best of 2 after a warm-up.  The card's name and power limit are read in the same run.  Writes
nothing to the tree."""
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
from bench_logistic import _best, _device_copy  # noqa: E402


class _Recorder:
    """the context, with each svm_pass recorded; ``full``: every pass computes the whole active Gram at the trial point
    (coef_from = NULL) and the change is formed on the host from the Gram kept for the accepted point"""

    def __init__(self, ctx, full=False):
        self.ctx, self.full, self.log, self.grams = ctx, full, [], {}

    def __getattr__(self, name):
        return getattr(self.ctx, name)

    def svm_pass(self, X, y, coef, intercept, *, coef_from=None, intercept_from=0.0, hessian=True, **kw):
        if not (self.full and hessian and coef_from is not None):
            r = self.ctx.svm_pass(X, y, coef, intercept, coef_from=coef_from, intercept_from=intercept_from,
                                  hessian=hessian, **kw)
            if self.full and hessian:
                self.grams[(np.asarray(coef).tobytes(), float(intercept))] = r["dhessian"]
        else:
            r = self.ctx.svm_pass(X, y, coef, intercept, coef_from=None, hessian=True, **kw)
            full = r["dhessian"]
            self.grams[(np.asarray(coef).tobytes(), float(intercept))] = full
            r["dhessian"] = full - self.grams[(np.asarray(coef_from).tobytes(), float(intercept_from))]
            r["entering"] = r["leaving"] = float("nan")
        self.log.append({k: r[k] for k in ("kept", "active", "entering", "leaving")} | {"from": coef_from is not None})
        return r


def _fit(ctx, X, y, full=False):
    rec = _Recorder(ctx, full)
    est = b2.B200LinearSVC(ctx=rec, dual=False)
    est.fit(X, y)
    times = []
    for _ in range(2):
        rec.log = []
        ctx.sync()
        t0 = time.perf_counter()
        est.fit(X, y)
        ctx.sync()
        times.append((time.perf_counter() - t0) * 1e3)
    n = rec.log[0]["kept"]
    iters = [{"active": round(p["active"] / n, 4), "changed": round((p["entering"] + p["leaving"]) / n, 5)}
             for p in rec.log[1:]]
    return est, round(min(times), 2), iters


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
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
    res = {"bench": "svm", "gpu": ctx.info()["name"], "power_limit": power, "rows": n, "d": d}
    g = torch.Generator(device="cuda").manual_seed(0)
    Xt = torch.randn(n, d, device="cuda", generator=g, dtype=torch.float32)
    beta = torch.randn(d, device="cuda", generator=g, dtype=torch.float64) / np.sqrt(d)
    xb = Xt.double() @ beta
    noisy = (torch.rand(n, device="cuda", generator=g, dtype=torch.float64) < torch.sigmoid(xb + 0.2)).float()
    flip = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) < 1e-3
    separable = ((xb > 0) ^ flip).float()
    X = _device_copy(ctx, Xt, "f32", (n, d))
    y = _device_copy(ctx, noisy.contiguous(), "f32", (n,))
    ys = _device_copy(ctx, separable.contiguous(), "f32", (n,))
    del Xt, xb
    torch.cuda.empty_cache()
    w = beta.cpu().numpy() * 0.5
    rng = np.random.default_rng(0)
    direction = rng.normal(size=d) / np.sqrt(d)
    res["logistic_gradient_pass_ms"] = _best(ctx, lambda: ctx.logistic_pass(X, y, w, 0.1, hessian=False))
    res["logistic_newton_pass_ms"] = _best(ctx, lambda: ctx.logistic_pass(X, y, w, 0.1, hessian=True))
    kw = dict(loss=native.SVM_SQUARED_HINGE, param=1.0)
    res["svm_gradient_pass_ms"] = _best(ctx, lambda: ctx.svm_pass(X, y, w, 0.1, coef_from=w, intercept_from=0.1,
                                                                  hessian=False, **kw))
    passes = {}
    r = ctx.svm_pass(X, y, np.zeros(d), 0.0, **kw)
    passes["start (all rows)"] = (r["entering"] / n, _best(ctx, lambda: ctx.svm_pass(X, y, np.zeros(d), 0.0, **kw)))
    passes["0"] = (0.0, _best(ctx, lambda: ctx.svm_pass(X, y, w, 0.1, coef_from=w, intercept_from=0.1, **kw)))
    for target in (0.01, 0.1):                     # the step along `direction` whose changed fraction is nearest
        best = None
        for alpha in np.geomspace(1e-3, 3.0, 24):
            r = ctx.svm_pass(X, y, w + alpha * direction, 0.1, coef_from=w, intercept_from=0.1, hessian=False, **kw)
            f = (r["entering"] + r["leaving"]) / n
            if best is None or abs(np.log(f / target if f > 0 else 1e-9)) < abs(np.log(best[1] / target)):
                best = (alpha, max(f, 1e-12))
        wt = w + best[0] * direction
        passes[f"~{target}"] = (best[1], _best(ctx, lambda: ctx.svm_pass(X, y, wt, 0.1, coef_from=w, intercept_from=0.1,
                                                                         **kw)))
    res["svm_pass"] = {k: {"changed_fraction": round(f, 5), "ms": t} for k, (f, t) in passes.items()}
    res["start_over_logistic_newton"] = round(passes["start (all rows)"][1] / res["logistic_newton_pass_ms"], 3)
    res["no_change_over_logistic_gradient"] = round(passes["0"][1] / res["logistic_gradient_pass_ms"], 3)
    for name, labels in (("noisy", y), ("separable", ys)):
        est, t, iters = _fit(ctx, X, labels)
        _, t_full, _ = _fit(ctx, X, labels, full=True)
        res[f"fit_{name}"] = {"ms": t, "n_iter": est.n_iter_, "passes": len(iters) + 1,
                              "rejected_steps": len(iters) - est.n_iter_, "per_pass": iters,
                              "full_gram_per_pass_ms": t_full}
    sk = min(a.sk_rows, n)
    if sk > 0:
        from sklearn import svm
        Xh = X.to_host()[:sk].astype(np.float64)
        yh = y.to_host()[:sk]
        t0 = time.perf_counter()
        svm.LinearSVC(dual=False).fit(Xh, yh)
        res["sklearn_fit_s"] = {"rows": sk, "s": round(time.perf_counter() - t0, 2)}
    for arr in (X, y, ys):
        arr.free()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
