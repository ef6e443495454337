"""Dump what every public estimator leaves behind on a fixed grid of seeded cases, to compare two trees byte for byte.

    python tools/dump_estimator_state.py --out FILE.npz            # the estimators of the tree this file sits in
    python tools/dump_estimator_state.py --compare A.npz B.npz     # every entry equal byte for byte?

Cases: host fp32 rows (20 000 x 8), host float64 rows (70 000 x 16: converted and uploaded by upload_columns), device
fp32 and bf16 rows, masked host and device rows (keep = 1 of a seeded 0/1 mask), and for LogisticRegression host labels
beside device rows.  Targets follow each estimator's family (Gaussian, Poisson, gamma, compound Poisson-gamma, binary).
Per case: every fitted attribute (bytes, dtype, Python type), the outputs of predict / predict_proba /
decision_function / score / predict(return_std=True), vars(to_sklearn()) as types and bytes, and each warning's
category, message, file name and line; enet_path / lasso_path on the fp32 cases.  Prints one JSON line."""
import argparse
import json
import linecache
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, D = 20_000, 8
N64, D64 = 70_000, 16


def _estimators(b2, ctx):
    """(name, make, target family); the iteration limits make some fits warn, so warnings are compared too"""
    return [
        ("LinearRegression", lambda: b2.B200LinearRegression(ctx=ctx), "normal"),
        ("LinearRegression-refine", lambda: b2.B200LinearRegression(ctx=ctx, refine=1), "normal"),
        ("RidgeCV", lambda: b2.B200RidgeCV(alphas=(0.1, 1.0, 10.0), store_cv_results=True, ctx=ctx), "normal"),
        ("ElasticNet", lambda: b2.B200ElasticNet(alpha=0.01, max_iter=3, ctx=ctx), "normal"),
        ("Lasso", lambda: b2.B200Lasso(alpha=0.01, ctx=ctx), "normal"),
        ("ElasticNetCV", lambda: b2.B200ElasticNetCV(l1_ratio=(0.5, 0.9), cv=3, max_iter=4, ctx=ctx), "normal"),
        ("LassoCV", lambda: b2.B200LassoCV(cv=3, ctx=ctx), "normal"),
        ("BayesianRidge", lambda: b2.B200BayesianRidge(compute_score=True, ctx=ctx), "normal"),
        ("ARDRegression", lambda: b2.B200ARDRegression(ctx=ctx), "normal"),
        ("PoissonRegressor", lambda: b2.B200PoissonRegressor(alpha=1e-3, ctx=ctx), "poisson"),
        ("GammaRegressor", lambda: b2.B200GammaRegressor(alpha=1e-3, max_iter=2, ctx=ctx), "gamma"),
        ("TweedieRegressor", lambda: b2.B200TweedieRegressor(power=1.5, alpha=1e-3, ctx=ctx), "compound"),
        ("LogisticRegression", lambda: b2.B200LogisticRegression(C=1.0, ctx=ctx), "binary"),
    ]


def _data(n, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 0.5, size=(n, d)).astype(np.float32)
    eta = X.astype(np.float64) @ rng.uniform(-0.5, 0.5, size=d) + 0.2
    mu = np.exp(eta)
    y = {"normal": eta + rng.normal(0.0, 0.3, size=n), "poisson": rng.poisson(mu).astype(np.float64),
         "gamma": rng.gamma(2.0, mu / 2.0), "compound": rng.poisson(mu) * rng.gamma(2.0, 0.5, size=n),
         "binary": (rng.uniform(size=n) < 1.0 / (1.0 + np.exp(-eta))).astype(np.int64)}
    mask = (rng.uniform(size=n) < 0.7).astype(np.uint8)
    return X, y, mask


class _Dump:
    def __init__(self, b2):
        self.b2, self.res = b2, {}

    def put(self, key, v):
        """bytes, dtype and shape of arrays; repr of plain values; the type of everything"""
        if isinstance(v, self.b2.DeviceArray):
            self.res[key + ":type"] = np.array(f"DeviceArray/{v.kind}")
            h = v.to_host()
            v.free()
            self.res[key] = h
            return
        self.res[key + ":type"] = np.array(f"{type(v).__module__}.{type(v).__qualname__}")
        if isinstance(v, (list, tuple)):
            for i, e in enumerate(v):
                self.put(f"{key}[{i}]", e)
        elif isinstance(v, (np.ndarray, np.generic)) and v.dtype != object:
            self.res[key] = np.asarray(v)
        elif v is None or isinstance(v, (bool, int, float, str)):
            self.res[key] = np.array(repr(v))

    def warnings(self, key, caught):
        """a warning raised at a line of this file by its line number, one raised inside the package by the text of
        its line (the package's line numbers are what two trees may differ in)"""
        for i, w in enumerate(caught):
            here = os.path.basename(w.filename) == os.path.basename(__file__)
            where = w.lineno if here else linecache.getline(w.filename, w.lineno).strip()
            self.res[f"{key}:warning{i}"] = np.array(
                f"{w.category.__name__}|{w.message}|{os.path.basename(w.filename)}|{where}")


def _outcome(dmp, key, name, est, X, y, mask):
    est.fit(X, y, row_mask=mask)
    for attr in sorted(a for a in vars(est) if a.endswith("_") and not a.startswith("_")):
        dmp.put(f"{key}/attr/{attr}", getattr(est, attr))
    dmp.put(f"{key}/predict", est.predict(X))
    if hasattr(est, "score"):
        dmp.put(f"{key}/score", est.score(X, y, row_mask=mask))
    if hasattr(est, "predict_proba"):
        dmp.put(f"{key}/predict_proba", est.predict_proba(X))
        dmp.put(f"{key}/decision_function", est.decision_function(X))
    if name in ("BayesianRidge", "ARDRegression"):
        dmp.put(f"{key}/predict_std", est.predict(X, return_std=True))
    for attr, v in sorted(vars(est.to_sklearn()).items()):
        dmp.put(f"{key}/sklearn/{attr}", v)


def dump(out):
    import bodywork_mlops_demo_b200 as b2
    ctx = b2.Context(0)
    dmp = _Dump(b2)
    X, ys, mask = _data(N, D, 11)
    X64, ys64, _ = _data(N64, D64, 12)
    Xd, Xb, md = ctx.to_device(X), ctx.to_device(b2.native.to_bf16_bits(X), "bf16"), ctx.to_device(mask)
    for name, make, family in _estimators(b2, ctx):
        y, y64 = ys[family], ys64[family].astype(np.float64)
        yd = ctx.to_device(np.ascontiguousarray(y, dtype=np.float32))
        cases = {"host32": (X, y, None), "host64": (X64.astype(np.float64), y64, None), "dev32": (Xd, yd, None),
                 "devbf16": (Xb, yd, None), "masked-host": (X, y, mask), "masked-dev": (Xd, yd, md)}
        if family == "binary":
            cases["dev32-host-labels"] = (Xd, y, None)
        for case, (Xc, yc, mc) in cases.items():
            key = f"{name}/{case}"
            with warnings.catch_warnings(record=True) as caught:
                warnings.simplefilter("always")
                try:
                    _outcome(dmp, key, name, make(), Xc, yc, mc)
                except Exception as exc:            # a refusal is compared like any other outcome
                    dmp.put(f"{key}/refused", f"{type(exc).__name__}: {exc}")
            dmp.warnings(key, caught)
        yd.free()
    yd = ctx.to_device(np.ascontiguousarray(ys["normal"], dtype=np.float32))
    for fn in ("enet_path", "lasso_path"):
        for case, (Xc, yc) in {"host32": (X, ys["normal"]), "dev32": (Xd, yd)}.items():
            with warnings.catch_warnings(record=True) as caught:
                warnings.simplefilter("always")
                dmp.put(f"{fn}/{case}", getattr(b2, fn)(Xc, yc, alphas=8, max_iter=5, fit_intercept=True,
                                                         return_n_iter=True, ctx=ctx))
            dmp.warnings(f"{fn}/{case}", caught)
    yd.free(); Xd.free(); Xb.free(); md.free()
    info = ctx.info()
    ctx.close()
    np.savez(out, **{k.replace("/", "|"): v for k, v in dmp.res.items()})
    print(json.dumps({"dump": out, "root": ROOT, "gpu": info["name"], "entries": len(dmp.res),
                      "warnings": sum(":warning" in k for k in dmp.res)}))


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    keys_a, keys_b = set(a.files), set(b.files)
    differ = sorted(k for k in keys_a & keys_b if a[k].dtype != b[k].dtype or a[k].shape != b[k].shape
                    or a[k].tobytes() != b[k].tobytes())
    res = {"a": a_path, "b": b_path, "entries": len(keys_a & keys_b), "only_in_one": sorted(keys_a ^ keys_b)[:20],
           "differ": len(differ), "first_differences": differ[:20]}
    res["identical"] = not differ and not (keys_a ^ keys_b)
    print(json.dumps(res))
    return 0 if res["identical"] else 1


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
