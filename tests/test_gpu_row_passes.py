"""Every pass over a call's rows streams host rows through the staging ring the same way (DESIGN.md section 3): these
tests run each host-streamed entry point on masked host rows of three staging blocks plus a tail, at d = 8 (the narrow
ring) and d = 64 (the wide ring), and on one strided layout.

  * pinned and pageable rows give bit-identical outputs in the same number of launches;
  * every per-row output (yhat, ystd, mu, the logistic decision, proba and label) is bit-identical to the same call on
    each staging block's rows alone;
  * the outputs agree with the same call on device rows.  The Gram runs on the exact fp64 kernel, so every difference
    is the order of fp64 sums: relative ROW_TOL on fp64 results (LOO_TOL behind b2_ridge_loo's eigendecomposition),
    FP32_TOL on b2_score's fp32 predictions and test_gpu_glm.PASS_TOL on the GLM and logistic sums.
"""
import ctypes as C

import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from test_gpu_glm import PASS_TOL

pytestmark = pytest.mark.gpu

BLOCK = 1 << 18                    # rows per staging block
N = 2 * BLOCK + 4321               # three blocks, the last one partial
ROW_TOL = 1e-12
LOO_TOL = 1e-9
FP32_TOL = 1e-6
ALPHAS = np.array([0.1, 1.0, 10.0, 100.0])


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ok(rc):
    assert rc == 0, native.last_error()


class Rows:
    """One layout of the same rows: X (row pitch ldx), y, the mask and the labels y > 1 (0 / 1) as host (pageable or
    pinned) or device pointers."""

    def __init__(self, ctx, Xs, y, mask, kind, d, ld_off=0):
        self.ctx, self.kind, self.n, self.d = ctx, kind, y.size, d
        self.ldx, self.host = Xs.shape[1], kind != "device"
        self._keep = []
        self._labels = labels = (y > 1.0).astype(np.float32)    # pageable rows point into it
        if kind == "pageable":
            arrs = [Xs, y, mask, labels]
        elif kind == "pinned":
            arrs = []
            for a in (Xs, y, mask, labels):
                p = ctx.pinned(a.shape, a.dtype)
                p.array[:] = a
                self._keep.append(p)
                arrs.append(p.array)
        else:
            self._keep = [ctx.to_device(Xs), ctx.to_device(y), ctx.to_device(mask), ctx.to_device(labels)]
            arrs = self._keep
        ptr = [a.ctypes.data if isinstance(a, np.ndarray) else a.ptr for a in arrs]
        self.X, self.y, self.mask, self.labels = ptr[0] + 4 * ld_off, ptr[1], ptr[2], ptr[3]
        self.mk = native.MEM_HOST if self.host else native.MEM_DEVICE

    def out(self, shape, dtype):
        """(buffer, pointer, fetch) of a per-row output in this layout's memory"""
        if self.host:
            a = np.empty(shape, dtype)
            return a, a.ctypes.data, lambda: a
        dv = self.ctx.empty(shape, "f32" if dtype == np.float32 else "f64")
        self._keep.append(dv)
        return dv, dv.ptr, dv.to_host

    def free(self):
        for a in self._keep:
            a.free()


def _calls(ctx, r, coef, b0):
    """name -> (outputs, launches) of every row pass on the rows of r"""
    lib, d, n = native.load(), r.d, r.n
    base = (ctx._h, r.X, b2.F32)
    res = {}

    def run(name, fn):
        before = ctx.launch_count()
        res[name] = (fn(), ctx.launch_count() - before)

    def score():
        _, yp, yh = r.out(n, np.float32)
        st = np.empty(10)
        _ok(lib.b2_score(*base, n, d, r.ldx, r.mk, coef.ctypes.data, b0, r.y, r.mask, 1, yp, st.ctypes.data))
        return {"yhat": yh().copy(), "stats": st}

    def fit():
        c, i = np.empty(d), np.empty(1)
        _ok(lib.b2_fit(*base, r.y, n, d, r.ldx, r.mk, r.mask, 1, 0.0, 1, c.ctypes.data, _dp(i)))
        return {"coef": c, "intercept": i}

    def moments():             # at (coef, b0) with m from the resident S of fit()
        out = np.empty(d + 2)
        _ok(lib.b2_residual_moments(*base, r.y, n, d, r.ldx, r.mk, r.mask, 1, coef.ctypes.data, b0, 1,
                                    out.ctypes.data))
        return {"moments": out}

    def loo():
        _, cp, cv = r.out((n, ALPHAS.size), np.float64)
        mse, c, i, best = np.empty(ALPHAS.size), np.empty(d), np.empty(1), np.zeros(1, np.int32)
        _ok(lib.b2_ridge_loo(*base, r.y, n, d, r.ldx, r.mk, r.mask, 1, ALPHAS.ctypes.data, ALPHAS.size, 1,
                             mse.ctypes.data, cp, best.ctypes.data_as(C.POINTER(C.c_int)), c.ctypes.data, _dp(i)))
        return {"mse": mse, "cv": cv().copy(), "best": best, "coef": c}

    def score_std():
        rng = np.random.default_rng(d)
        A = rng.normal(size=(d, d)) / d
        sigma, mean = A @ A.T, rng.normal(size=d)
        _, sp, ys = r.out(n, np.float64)
        _, hp, yh = r.out(n, np.float64)
        _ok(lib.b2_score_std(*base, n, d, r.ldx, r.mk, mean.ctypes.data, sigma.ctypes.data, 0.25, coef.ctypes.data, b0,
                             hp, sp))
        return {"ystd": ys().copy(), "yhat": yh().copy()}

    def glm_pass():
        sums, H = np.empty(d + 8), np.empty((d + 1, d + 1))
        _ok(lib.b2_glm_pass(*base, r.y, n, d, r.ldx, r.mk, r.mask, 1, native.GLM_LOG, 1.5, coef.ctypes.data, b0, 1,
                            sums.ctypes.data, H.ctypes.data))
        return {"sums": sums, "hessian": H}

    def line_search():
        step, out = coef[::-1].copy(), np.empty(native.GLM_STEPS)
        _ok(lib.b2_glm_line_search(*base, r.y, n, d, r.ldx, r.mk, r.mask, 1, native.GLM_LOG, 1.5, coef.ctypes.data,
                                   b0, step.ctypes.data, -0.1, native.GLM_STEPS, out.ctypes.data))
        return {"ladder": out}

    def glm_predict():
        _, mp, mu = r.out(n, np.float64)
        _ok(lib.b2_glm_predict(*base, n, d, r.ldx, r.mk, native.GLM_LOG, coef.ctypes.data, b0, mp))
        return {"mu": mu().copy()}

    def logistic_pass(hessian):
        sums, H = np.empty(d + 9), np.empty((d + 1, d + 1)) if hessian else None
        _ok(lib.b2_logistic_pass(*base, r.labels, n, d, r.ldx, r.mk, r.mask, 1, 0.0, 1.0, coef.ctypes.data, b0, 1,
                                 sums.ctypes.data, H.ctypes.data if hessian else None))
        return {"sums": sums, "hessian": H} if hessian else {"sums": sums}

    def logistic_line_search():
        step, out = coef[::-1].copy(), np.empty(native.GLM_STEPS)
        _ok(lib.b2_logistic_line_search(*base, r.labels, n, d, r.ldx, r.mk, r.mask, 1, 0.0, 1.0, coef.ctypes.data, b0,
                                        step.ctypes.data, -0.1, native.GLM_STEPS, out.ctypes.data))
        return {"ladder": out}

    def logistic_predict():
        _, dp_, dec = r.out(n, np.float64)
        _, pp, proba = r.out((n, 2), np.float64)
        _, lp, lab = r.out(n, np.float32)
        _ok(lib.b2_logistic_predict(*base, n, d, r.ldx, r.mk, coef.ctypes.data, b0, 0.0, 1.0, dp_, pp, lp))
        return {"decision": dec().copy(), "proba": proba().copy(), "label": lab().copy()}

    for name, fn in (("score", score), ("fit", fit), ("moments", moments), ("loo", loo), ("score_std", score_std),
                     ("glm_pass", glm_pass), ("line_search", line_search), ("glm_predict", glm_predict),
                     ("logistic_pass", lambda: logistic_pass(True)), ("logistic_grad", lambda: logistic_pass(False)),
                     ("logistic_line_search", logistic_line_search), ("logistic_predict", logistic_predict)):
        run(name, fn)
    return res


def _table(d, seed, spare=0):
    rng = np.random.default_rng(seed)
    Xs = (rng.normal(size=(N, d + spare)) * 0.5).astype(np.float32)
    coef = rng.normal(size=d) * 0.4 / np.sqrt(d)
    y = rng.gamma(2.0, np.exp(Xs[:, :d].astype(np.float64) @ coef + 0.2) / 2.0).astype(np.float32)
    mask = (np.arange(N) % 7 != 3).astype(np.uint8)
    return Xs, y, mask, coef


def _compare_layouts(ctx, Xs, y, mask, coef, d, ld_off=0):
    """the host layouts' outputs and launch counts, and the device rows' outputs (contiguous)"""
    ctx.set_kernel(b2.KERNEL_SIMT)         # the exact fp64 Gram: host and device S differ only in the order of sums
    out = {}
    try:
        for kind in ("pageable", "pinned"):
            r = Rows(ctx, Xs, y, mask, kind, d, ld_off)
            try:
                out[kind] = _calls(ctx, r, coef, 0.2)
            finally:
                r.free()
        r = Rows(ctx, np.ascontiguousarray(Xs[:, ld_off:ld_off + d]), y, mask, "device", d)
        try:
            out["device"] = _calls(ctx, r, coef, 0.2)
        finally:
            r.free()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
    for name, (res, launches) in out["pinned"].items():
        pag, pag_launches = out["pageable"][name]
        assert launches == pag_launches, name
        for k, v in res.items():
            assert np.array_equal(v, pag[k], equal_nan=True), (name, k)
    dev = {name: res for name, (res, _) in out["device"].items()}
    host = {name: res for name, (res, _) in out["pageable"].items()}
    worst = {}
    for name in ("fit", "moments", "loo", "score_std", "glm_predict", "logistic_predict"):
        for k, v in host[name].items():
            if k == "best":
                assert np.array_equal(v, dev[name][k])
                continue
            kept = mask == 1 if k == "cv" else slice(None)
            if k == "cv":
                assert np.isnan(v[~kept]).all() and np.isnan(dev[name][k][~kept]).all()
            worst[name, k] = rel(v[kept], dev[name][k][kept])
            assert worst[name, k] < (LOO_TOL if name == "loo" else ROW_TOL), (name, k, worst[name, k])
    print("\n[host vs device rows] " + ", ".join(f"{n}.{k} {e:.1e}" for (n, k), e in worst.items()))
    assert rel(host["score"]["yhat"], dev["score"]["yhat"]) < FP32_TOL
    sums = host["score"]["stats"]
    assert rel(sums, dev["score"]["stats"]) < FP32_TOL and sums[5] == dev["score"]["stats"][5] == mask.sum()
    for name in ("glm_pass", "logistic_pass", "logistic_grad"):
        for k in host[name]:
            assert rel(host[name][k], dev[name][k]) < PASS_TOL, (name, k)
    for name in ("line_search", "logistic_line_search"):
        assert rel(host[name]["ladder"], dev[name]["ladder"]) < PASS_TOL, name
    return host


@pytest.mark.parametrize("d", [8, 64])
def test_host_rows_stream_like_device_rows(ctx, d):
    Xs, y, mask, coef = _table(d, 70 + d)
    host = _compare_layouts(ctx, Xs, y, mask, coef, d)
    # per-row outputs: the same call on each staging block's rows alone
    parts = {"score": [], "score_std": [], "glm_predict": [], "logistic_predict": []}
    for r0 in range(0, N, BLOCK):
        sl = slice(r0, min(r0 + BLOCK, N))
        r = Rows(ctx, np.ascontiguousarray(Xs[sl]), np.ascontiguousarray(y[sl]), np.ascontiguousarray(mask[sl]),
                 "pageable", d)
        blk = _calls(ctx, r, coef, 0.2)
        r.free()
        for name in parts:
            parts[name].append(blk[name][0])
    assert np.array_equal(np.concatenate([p["yhat"] for p in parts["score"]]), host["score"]["yhat"])
    for k in ("ystd", "yhat"):
        assert np.array_equal(np.concatenate([p[k] for p in parts["score_std"]]), host["score_std"][k])
    assert np.array_equal(np.concatenate([p["mu"] for p in parts["glm_predict"]]), host["glm_predict"]["mu"])
    for k in ("decision", "proba", "label"):
        assert np.array_equal(np.concatenate([p[k] for p in parts["logistic_predict"]]), host["logistic_predict"][k])


def test_strided_host_rows(ctx):
    """rows of pitch d + 3 starting one element in: the ring's pitched copies (pinned) and the bounce copies (pageable)"""
    d = 64
    Xs, y, mask, coef = _table(d, 91, spare=3)
    _compare_layouts(ctx, Xs, y, mask, coef, d, ld_off=1)
