"""Dump every output of the fp64 tile passes on a fixed grid of cases, to compare two builds bit for bit.

    python tools/dump_row_passes.py --out FILE.npz            # with the in-tree library, or B2_LIB_PATH=... for another
    python tools/dump_row_passes.py --compare A.npz B.npz     # every array equal byte for byte?

Calls: b2_glm_pass with and without the Hessian and b2_glm_line_search at identity / power 0 and log / powers 0, 1,
1.5, 2 and 3; b2_logistic_pass with and without the Hessian and b2_logistic_line_search (labels y > 1); b2_ridge_loo
at 1, 13 and 64 alphas with cv_out; b2_score_std with and without yhat.  Grid: d = 1, 8, 17, 64, 127 and 128 x fp32
and bf16 rows x device rows (4 133: ring tiles and a direct tail where the rows stream through the ring), device rows
of pitch d + 3 starting one element in, masked device rows (keep = 1 of a seeded 0/1 mask), and at d = 64 pinned and
pageable host rows over two staging blocks and a tail, masked.  Per call: every output and the launch count; an output
over 16 MB (the host cases' cv_out) as its SHA-256 digest, so a dump stays small.  Rows come from a fixed numpy seed.
The symmetric sums: b2_multinomial_pass with the Hessian at K = 3 and 7; b2_svm_pass with dhess_out for both losses,
with and without coef_from; b2_class_scatter with unit and per-class weights and b2_class_scatters at K = 7.  The
multiclass labels are floor(3 y) mod 7 (at K = 3 some rows have no class).  Prints one JSON line."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS = (1, 8, 17, 64, 127, 128)
N_DEV = 4_133
N_HOST = 2 * (1 << 18) + 4_321
BIG = 16 << 20                                          # bytes: larger outputs are dumped as their digest
GLM = (("identity", 0.0), ("log", 0.0), ("log", 1.0), ("log", 1.5), ("log", 2.0), ("log", 3.0))
CLASSES = np.arange(7, dtype=np.float32)               # the multiclass passes' labels
CLASS_WEIGHTS = np.linspace(0.5, 2.0, 7)


def _rows(n, d, seed):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) * 0.5).astype(np.float32)
    coef = rng.normal(size=d) * 0.4 / np.sqrt(d)
    y = rng.gamma(2.0, np.exp(X.astype(np.float64) @ coef + 0.2) / 2.0).astype(np.float32)
    mask = (rng.uniform(size=n) < 0.7).astype(np.uint8)
    A = rng.normal(size=(d, d)) / d
    return X, y, mask, coef, A @ A.T, rng.normal(size=d)


def dump(out):
    import bodywork_mlops_demo_b200 as b2
    from bodywork_mlops_demo_b200 import _native as native
    lib, ctx = native.load(), b2.Context(0)
    res, keep = {}, []

    def ok(rc):
        assert rc == 0, native.last_error()

    def run(key, mk, fn):
        """fn(outputs) fills the outputs it asks for through outputs(shape, dtype) -> pointer"""
        bufs = []

        def output(shape, dtype):
            if mk == native.MEM_HOST:
                a = np.empty(shape, dtype)
                bufs.append((a, None))
                return a.ctypes.data
            dv = ctx.empty(shape, "f32" if dtype == np.float32 else "f64")
            bufs.append((None, dv))
            return dv.ptr
        before = ctx.launch_count()
        host = fn(output)
        res[key + ":launches"] = np.array([ctx.launch_count() - before])
        for i, a in enumerate(host):
            res[f"{key}:{i}"] = np.asarray(a)
        for i, (a, dv) in enumerate(bufs):
            a = a if dv is None else dv.to_host()
            if a.nbytes > BIG:
                res[f"{key}:out{i}:sha256"] = np.frombuffer(hashlib.sha256(a.tobytes()).digest(), np.uint8)
            else:
                res[f"{key}:out{i}"] = a
            if dv is not None:
                dv.free()

    def calls(key, X, xdt, y, lab, mlab, mask, n, d, ldx, mk, coef, sigma, mean):
        base = (ctx._h, X, xdt)
        w, step = coef.ctypes.data, coef[::-1].copy()
        rng = np.random.default_rng(3000 + d)
        mn_coef = rng.normal(size=(7, d + 1)) * 0.5 / np.sqrt(d)
        means = rng.normal(size=(7, d)) * 0.1
        for link, power in GLM:
            lk = native.GLM_LOG if link == "log" else native.GLM_IDENTITY
            for hess in (True, False):
                def glm_pass(output, lk=lk, power=power, hess=hess):
                    sums, H = np.empty(d + 8), np.empty((d + 1, d + 1)) if hess else None
                    ok(lib.b2_glm_pass(*base, y, n, d, ldx, mk, mask, 1, lk, power, w, 0.2, 1, sums.ctypes.data,
                                       H.ctypes.data if hess else None))
                    return [sums] + ([H] if hess else [])
                run(f"{key}/glm_pass-{link}-{power}-{'hess' if hess else 'grad'}", mk, glm_pass)

            def glm_ladder(output, lk=lk, power=power):
                loss = np.empty(native.GLM_STEPS)
                ok(lib.b2_glm_line_search(*base, y, n, d, ldx, mk, mask, 1, lk, power, w, 0.2, step.ctypes.data, -0.1,
                                          native.GLM_STEPS, loss.ctypes.data))
                return [loss]
            run(f"{key}/glm_line_search-{link}-{power}", mk, glm_ladder)
        for hess in (True, False):
            def logistic_pass(output, hess=hess):
                sums, H = np.empty(d + 9), np.empty((d + 1, d + 1)) if hess else None
                ok(lib.b2_logistic_pass(*base, lab, n, d, ldx, mk, mask, 1, 0.0, 1.0, w, 0.2, 1, sums.ctypes.data,
                                        H.ctypes.data if hess else None))
                return [sums] + ([H] if hess else [])
            run(f"{key}/logistic_pass-{'hess' if hess else 'grad'}", mk, logistic_pass)

        def logistic_ladder(output):
            loss = np.empty(native.GLM_STEPS)
            ok(lib.b2_logistic_line_search(*base, lab, n, d, ldx, mk, mask, 1, 0.0, 1.0, w, 0.2, step.ctypes.data, -0.1,
                                           native.GLM_STEPS, loss.ctypes.data))
            return [loss]
        run(f"{key}/logistic_line_search", mk, logistic_ladder)
        for n_alphas in (1, 13, 64):
            def loo(output, n_alphas=n_alphas):
                alphas = np.geomspace(1e-3, 1e3, n_alphas)
                mse, c, b0, best = np.empty(n_alphas), np.empty(d), np.empty(1), np.zeros(1, np.int32)
                ok(lib.b2_ridge_loo(*base, y, n, d, ldx, mk, mask, 1, alphas.ctypes.data, n_alphas, 1, mse.ctypes.data,
                                    output((n, n_alphas), np.float64), best.ctypes.data_as(C.POINTER(C.c_int)),
                                    c.ctypes.data, b0.ctypes.data_as(C.POINTER(C.c_double))))
                return [mse, c, b0, best]
            run(f"{key}/ridge_loo-{n_alphas}", mk, loo)
        for want_yhat in (True, False):
            def score_std(output, want_yhat=want_yhat):
                ok(lib.b2_score_std(*base, n, d, ldx, mk, mean.ctypes.data, sigma.ctypes.data, 0.25, w, 0.2,
                                    output(n, np.float64) if want_yhat else None, output(n, np.float64)))
                return []
            run(f"{key}/score_std-{'yhat' if want_yhat else 'ystd'}", mk, score_std)
        for K in (3, 7):
            def multinomial_pass(output, K=K):
                W = np.ascontiguousarray(mn_coef[:K])
                sums, H = np.empty(5 + K * (d + 1)), np.empty((K, K, d + 1, d + 1))
                ok(lib.b2_multinomial_pass(*base, mlab, n, d, ldx, mk, mask, 1, CLASSES.ctypes.data, K, W.ctypes.data,
                                           1, sums.ctypes.data, H.ctypes.data))
                return [sums, H]
            run(f"{key}/multinomial_pass-{K}-hess", mk, multinomial_pass)
        for loss, yl, param in ((native.SVM_SQUARED_HINGE, lab, 1.0), (native.SVM_SQUARED_EPSILON, y, 0.1)):
            for from_step in (False, True):
                def svm_pass(output, loss=loss, yl=yl, param=param, from_step=from_step):
                    sums, dH = np.empty(d + 8), np.empty((d + 1, d + 1))
                    ok(lib.b2_svm_pass(*base, yl, n, d, ldx, mk, mask, 1, loss, param,
                                       step.ctypes.data if from_step else None, -0.1, w, 0.2, 1, sums.ctypes.data,
                                       dH.ctypes.data))
                    return [sums, dH]
                run(f"{key}/svm_pass-{loss}-{'from' if from_step else 'start'}", mk, svm_pass)
        for weighted in (False, True):
            def class_scatter(output, weighted=weighted):
                S, counts = np.empty((d, d)), np.empty(3)
                ok(lib.b2_class_scatter(*base, mlab, n, d, ldx, mk, mask, 1, CLASSES.ctypes.data, 7, means.ctypes.data,
                                        CLASS_WEIGHTS.ctypes.data if weighted else None, S.ctypes.data,
                                        counts.ctypes.data))
                return [S, counts]
            run(f"{key}/class_scatter-{'weighted' if weighted else 'unit'}", mk, class_scatter)

        def class_scatters(output):
            S, nk, counts = np.empty((7, d, d)), np.empty(7), np.empty(3)
            ok(lib.b2_class_scatters(*base, mlab, n, d, ldx, mk, mask, 1, CLASSES.ctypes.data, 7, means.ctypes.data,
                                     S.ctypes.data, nk.ctypes.data, counts.ctypes.data))
            return [S, nk, counts]
        run(f"{key}/class_scatters", mk, class_scatters)

    for kind in ("f32", "bf16"):
        xdt, es = (b2.F32, 4) if kind == "f32" else (b2.BF16, 2)
        conv = (lambda a: a) if kind == "f32" else native.to_bf16_bits
        for d in DS:
            X, y, mask, coef, sigma, mean = _rows(N_DEV, d, 1000 + d)
            lab = (y > 1.0).astype(np.float32)
            mlab = (np.floor(3 * y) % 7).astype(np.float32)
            yd, ld, mld, md = ctx.to_device(y), ctx.to_device(lab), ctx.to_device(mlab), ctx.to_device(mask)
            Xd = ctx.to_device(conv(X))
            Xs = np.zeros((N_DEV, d + 3), np.float32)           # pitch d + 3, the rows one element in
            Xs[:, 1:d + 1] = X
            Xsd = ctx.to_device(conv(Xs))
            for layout, Xp, ldx, mp in (("dev", Xd.ptr, d, None), ("strided", Xsd.ptr + es, d + 3, None),
                                        ("masked", Xd.ptr, d, md.ptr)):
                calls(f"{kind}-d{d}-{layout}", Xp, xdt, yd.ptr, ld.ptr, mld.ptr, mp, N_DEV, d, ldx, native.MEM_DEVICE,
                      coef, sigma, mean)
            for a in (yd, ld, mld, md, Xd, Xsd):
                a.free()
        d = 64
        X, y, mask, coef, sigma, mean = _rows(N_HOST, d, 2000)
        lab = (y > 1.0).astype(np.float32)
        mlab = (np.floor(3 * y) % 7).astype(np.float32)
        for host in ("pageable", "pinned"):
            arrs = [conv(X), y, lab, mlab, mask]
            if host == "pinned":
                pins = [ctx.pinned(a.shape, a.dtype) for a in arrs]
                for p, a in zip(pins, arrs):
                    p.array[:] = a
                arrs = [p.array for p in pins]
            Xh, yh, lh, mlh, mh = arrs
            calls(f"{kind}-d{d}-{host}", Xh.ctypes.data, xdt, yh.ctypes.data, lh.ctypes.data, mlh.ctypes.data,
                  mh.ctypes.data, N_HOST, d, d, native.MEM_HOST, coef, sigma, mean)
            if host == "pinned":
                for p in pins:
                    p.free()
    info = ctx.info()
    ctx.close()
    np.savez(out, **res)
    print(json.dumps({"dump": out, "lib": os.environ.get("B2_LIB_PATH", "in-tree"), "gpu": info["name"],
                      "arrays": len(res), "calls": sum(k.endswith(":launches") for k in res)}))


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
