"""The fp64 tile passes on the 32-row tile ring of b2_dmma.cuh (glm_kernel, loo_kernel, score_std_kernel,
class_sums_kernel, classify_kernel) at row counts where every CTA walks many tiles: each slot of the three-stage ring is
refilled after the consumers released it, in both phases, and every per-CTA sum spans many tiles.

With G SMs, N_LONG = 32 (18 G + 5) + 17 rows are at least 9 tiles per CTA at two CTAs per SM (18 at one), uneven across
CTAs, then a direct tail; N_EDGE are the row counts where the split between the ring and the direct flavour changes.
Each pass runs on device rows in the layouts scoring's plan (plan_rows) streams through the ring (contiguous, X, y and,
for d <= 16, the mask 16-byte aligned) and in layouts it sends to the direct flavour (X or y 4 bytes past a 16-byte
boundary); _ring encodes that rule and every call's launch count must match the flavour it predicts.

  * long runs against the references of the other suites (NumpyGLMContext, NumpyLogisticContext,
    NumpyClassifierContext, loo_oracle on the exact SIMT Gram, bayes_oracle, a long-double decision);
  * ring against direct on the same rows: per-row outputs (cv, ystd, yhat, decision, label) bit-identical; the GLM and
    leave-one-out sums bit-identical at whole tiles, where both flavours give every tile to the same CTA (with a tail,
    the ring flavour reduces the tail tile after the ring's CTAs while the direct flavour adds it into one CTA's sums,
    so there they agree within the bound); class sums and counts within the bound (their CTAs per SM depend on the
    ring's shared memory);
  * the edge row counts, masks that empty whole tiles or whole CTAs (NaN and +-Inf in every dropped row), host rows
    across staging blocks for the class-sum and classify passes;
  * on the CPU, that each comparison's bound is at least 100x below what a dropped tile, a tile counted twice or a
    stale ring slot would do to the compared quantity.

Bounds are the other suites' (5x the worst case they measured), which the longer summation chains here stay within; the
worst case over this file, measured on one H100 80GB HBM3 (132 SMs) at a 700 W power limit, is in brackets:
  * GLM and logistic sums and ladders: test_gpu_glm.PASS_TOL = 3e-14 relative to the largest entry of each (1.3e-14);
  * class sums: test_gpu_ridge_classifier.SUM_TOL = 1e-13 of the sum of |x - c| per entry (2.8e-14);
  * decisions: test_gpu_ridge_classifier.DEC_TOL = 1e-14 of sum_j |x_j w_j| + |b| per entry (5.8e-16);
  * ystd and yhat: 1e-12 relative, test_gpu_bayes's bound (1.2e-15);
  * leave-one-out cv and mse: test_gpu_row_passes.LOO_TOL = 1e-9 relative (cv 1.0e-13 and mse 1.9e-14 at N_LONG;
    6.2e-12 at the edge row counts below d, where the centred Gram is singular);
  * counts equal.
Each GPU test prints the worst case it measured (run with -s).
"""
import ctypes as C
import math
from collections import defaultdict

import numpy as np
import pytest
from scipy.special import expit

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from bayes_oracle import score_std as std_oracle
from loo_oracle import ridge_loo
from test_glm_driver import NumpyGLMContext
from test_gpu_glm import PASS_TOL
from test_gpu_ridge_classifier import DEC_TOL, SUM_TOL, _longdouble_decision
from test_gpu_row_passes import LOO_TOL
from test_logistic_driver import NumpyLogisticContext
from test_ridge_classifier_driver import NumpyClassifierContext

STD_TOL = 1e-12                  # test_gpu_bayes: b2_score_std against numpy
TILE = 32
H100_SMS = 132                   # the CPU checks take the H100 SXM's SM count
DEV = native.MEM_DEVICE
ALPHAS = np.array([0.1, 1.0, 10.0, 100.0])
NEG, POS = 3.0, 7.0
B_GLM, B_BIN, STEP_B = 0.2, 0.5, -0.1
LOSSES = {"identity": (native.GLM_IDENTITY, 0.0), "log p=1.5": (native.GLM_LOG, 1.5), "binomial": None}
CLASSES = {2: np.float32([-4, 11]), 3: np.float32([-7, 0, 13]), 32: np.arange(32, dtype=np.float32) * 3 - 40}
WIDTHS = [("f32", d) for d in (1, 8, 15, 16, 20, 64, 128)] + [("bf16", d) for d in (8, 24, 128)]
GLM = NumpyGLMContext()
LOG = NumpyLogisticContext()
CLS = NumpyClassifierContext()


def n_long(G):
    return TILE * (9 * 2 * G + 5) + 17


def n_edge(G):
    return [0, 1, 31, 32, 33, TILE * G, TILE * G + 1, TILE * (3 * G + 1), TILE * (3 * 2 * G + 1),
            TILE * (3 * 2 * G + 1) + 31]


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def _ring(xp, yp, mp, d, ldx, es):
    """plan_rows: does a call on these pointers stream its whole tiles through the ring?"""
    a16 = lambda p: p is None or p % 16 == 0
    rows = ldx == d and a16(xp) and a16(yp)
    if rows and d <= 16:
        return a16(mp)
    return rows and d > 16 and d % 4 == 0 and (d * es) % 16 == 0


def _launches(n, ring, per_part, writes_sums=True):
    """split_ring_rows: the whole tiles in one ring launch, the rest in one direct launch (also for no rows when the
    pass writes sums), each followed by its ordered reduce where the pass has sums (per_part = 2)"""
    whole = n // TILE * TILE if ring else 0
    return per_part * (int(whole > 0) + int(n > whole or (n == 0 and writes_sums)))


# ---- data ---------------------------------------------------------------------------------------------------------
class Table:
    """n seeded rows of d features (fp32 or bf16) with every pass's y, model and mask.  dropped: rows whose X and y are
    NaN / +-Inf."""

    def __init__(self, kind, d, n, seed, dropped=None):
        rng = np.random.default_rng(seed)
        X = (rng.normal(size=(n, d)) * 0.5).astype(np.float32)
        self.kind, self.d, self.n = kind, d, n
        self.dt, self.es = (b2.BF16, 2) if kind == "bf16" else (b2.F32, 4)
        up = native.to_bf16_bits(X) if kind == "bf16" else X
        Xv = native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
        self.coef = rng.normal(size=d) * 0.4 / np.sqrt(d)
        self.step = rng.normal(size=d) * 0.2 / np.sqrt(d)
        lc = rng.normal(size=d)
        self.lcoef = lc * 3.0 / np.linalg.norm(lc)
        y = {"glm": rng.gamma(2.0, np.exp(Xv @ self.coef + B_GLM) / 2.0),
             "bin": np.where(rng.uniform(size=n) < expit(Xv @ self.lcoef + B_BIN), POS, NEG),
             "reg": Xv @ rng.uniform(-1, 1, d) + rng.normal(size=n)}
        for k, cl in CLASSES.items():
            y[f"cls{k}"] = cl[rng.integers(0, k, size=n)]
        y = {k: v.astype(np.float32) for k, v in y.items()}
        if n > 64:
            for k in ("bin", "cls2", "cls3", "cls32"):
                y[k][rng.choice(n, 6, replace=False)] = 5.0 if k == "bin" else 99.0   # neither label / no class
                y[k][rng.choice(n, 2, replace=False)] = [np.nan, -np.inf]
        self.W = {t: rng.normal(size=(t, d)) for t in (1, 3, 32)}
        self.bW = {t: rng.normal(size=t) for t in (1, 3, 32)}
        G = rng.normal(size=(d, d))
        self.std = (rng.normal(size=d), G @ G.T / d * 1e-3, 0.25, rng.normal(size=d), 1.5)
        if dropped is not None:
            bad = np.resize(np.float32([np.nan, np.inf, -np.inf]), (int(dropped.sum()), d))
            X[dropped] = bad
            up = native.to_bf16_bits(X) if kind == "bf16" else X
            Xv[dropped] = bad
            for k in y:
                y[k][dropped] = bad[:, 0]
        self.up, self.Xv, self.y = up, Xv, y


class Dev:
    """A Table's rows, every y and a mask on the device twice: at the allocation (16-byte aligned) and `off` bytes past a
    16-byte boundary (4 for X and y, 1 for the mask)."""

    def __init__(self, ctx, t, mask, keep=1):
        self.d, self.dt, self.es, self.keep, self._bufs = t.d, t.dt, t.es, keep, []
        self.x = self._put(ctx, t.up, 4)
        self.y = {k: self._put(ctx, v, 4) for k, v in t.y.items()}
        self.m = self._put(ctx, mask, 1) if mask is not None else (None, None)

    def _put(self, ctx, a, off):
        raw = np.ascontiguousarray(a).view(np.uint8).ravel()
        al, mis = ctx.to_device(raw), ctx.to_device(np.r_[np.zeros(off, np.uint8), raw])
        self._bufs += [al, mis]
        return al.ptr, mis.ptr + off

    def free(self):
        for a in self._bufs:
            a.free()


class Layout:
    """One layout of a Dev's rows: which of X, y and the mask sit past their 16-byte boundary."""

    def __init__(self, dev, name, x_off=False, y_off=False, m_off=False):
        self.name, self.d, self.dt, self.es, self.keep = name, dev.d, dev.dt, dev.es, dev.keep
        self.xp = dev.x[x_off]
        self.yp = {k: v[y_off] for k, v in dev.y.items()}
        self.mp = dev.m[m_off]

    def mask(self, masked):
        return self.mp if masked else None

    def ring(self, y=None, masked=False):
        return _ring(self.xp, None if y is None else self.yp[y], self.mask(masked), self.d, self.d, self.es)


def _layouts(dev, with_mask):
    out = {"ring": Layout(dev, "ring"), "x+4": Layout(dev, "x+4", x_off=True), "y+4": Layout(dev, "y+4", y_off=True)}
    if with_mask:
        out["mask+1"] = Layout(dev, "mask+1", m_off=True)
    return out


def _p(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


def _call(ctx, fn, *args):
    before = ctx.launch_count()
    rc = fn(*args)
    assert rc == 0, native.last_error()
    return ctx.launch_count() - before


# ---- the passes on device rows: (outputs, launches) -----------------------------------------------------------------
def _glm_got(sums, H, d, binomial):
    got = dict(zip(("loss", "const", "sum_y", "kept", "y_out_of_range", "h_nonpos", "y_nonfinite"), sums[:7]))
    got["grad"], got["hessian"] = sums[7:8 + d].copy(), H
    if binomial:
        got["correct"] = sums[8 + d]
    return got


def run_glm(ctx, t, L, n, masked, loss, hess=True):
    """b2_glm_pass / b2_logistic_pass and the line search of the same loss: the pass's outputs with the ladder, and the
    two calls' launches"""
    lib, d, mp = native.load(), L.d, L.mask(masked)
    sums, lad = np.empty(d + 9), np.empty(native.GLM_STEPS)
    H = np.empty((d + 1, d + 1)) if hess else None
    hp = H.ctypes.data if hess else None
    if loss == "binomial":
        yp, c = L.yp["bin"], t.lcoef
        l1 = _call(ctx, lib.b2_logistic_pass, ctx._h, L.xp, L.dt, yp, n, d, d, DEV, mp, L.keep, NEG, POS, c.ctypes.data,
                   B_BIN, 1, sums.ctypes.data, hp)
        l2 = _call(ctx, lib.b2_logistic_line_search, ctx._h, L.xp, L.dt, yp, n, d, d, DEV, mp, L.keep, NEG, POS,
                   c.ctypes.data, B_BIN, t.step.ctypes.data, STEP_B, native.GLM_STEPS, lad.ctypes.data)
    else:
        (link, power), yp, c = LOSSES[loss], L.yp["glm"], t.coef
        l1 = _call(ctx, lib.b2_glm_pass, ctx._h, L.xp, L.dt, yp, n, d, d, DEV, mp, L.keep, link, power, c.ctypes.data,
                   B_GLM, 1, sums.ctypes.data, hp)
        l2 = _call(ctx, lib.b2_glm_line_search, ctx._h, L.xp, L.dt, yp, n, d, d, DEV, mp, L.keep, link, power,
                   c.ctypes.data, B_GLM, t.step.ctypes.data, STEP_B, native.GLM_STEPS, lad.ctypes.data)
    assert H is None or np.array_equal(H, H.T)
    got = _glm_got(sums, H, d, loss == "binomial")
    got["ladder"] = lad
    ring = L.ring("bin" if loss == "binomial" else "glm", masked)
    assert (l1, l2) == (_launches(n, ring, 2),) * 2, (L.name, n, ring, l1, l2)
    return got, ring


def glm_ref(t, n, mask, keep, loss):
    X = t.Xv[:n]
    m = None if mask is None else mask[:n]
    if loss == "binomial":
        y = t.y["bin"][:n]
        want = LOG.logistic_pass(X, y, t.lcoef, B_BIN, NEG, POS, row_mask=m, mask_keep=keep, hessian=True)
        want["ladder"] = LOG.logistic_line_search(X, y, t.lcoef, B_BIN, t.step, STEP_B, NEG, POS, row_mask=m,
                                                  mask_keep=keep)
    else:
        (link, power), y = LOSSES[loss], t.y["glm"][:n]
        want = GLM.glm_pass(X, y, t.coef, B_GLM, link=link, power=power, row_mask=m, mask_keep=keep, hessian=True)
        want["ladder"] = GLM.glm_line_search(X, y, t.coef, B_GLM, t.step, STEP_B, link=link, power=power, row_mask=m,
                                             mask_keep=keep)
    return want


def run_loo(ctx, t, L, n, masked):
    """b2_ridge_loo on the exact fp64 Gram: (mse, cv, best), its launches, the Gram's own launches on the same rows and
    the statistic S it left"""
    lib, d, mp, yp = native.load(), L.d, L.mask(masked), L.yp["reg"]
    ctx.set_kernel(b2.KERNEL_SIMT)
    try:
        cvd = ctx.empty((max(n, 1), ALPHAS.size), "f64")
        mse, coef, b0, best = np.empty(ALPHAS.size), np.empty(d), np.empty(1), np.zeros(1, np.int32)
        try:
            launches = _call(ctx, lib.b2_ridge_loo, ctx._h, L.xp, L.dt, yp, n, d, d, DEV, mp, L.keep,
                             ALPHAS.ctypes.data, ALPHAS.size, 1, mse.ctypes.data, cvd.ptr, _p(best, C.c_int),
                             coef.ctypes.data, _p(b0, C.c_double))
            cv = cvd.to_host()[:n]
        finally:
            cvd.free()
        S, rows = np.empty((d + 2, d + 2)), np.zeros(1, np.int64)
        assert lib.b2_gram_export(ctx._h, S.ctypes.data, _p(rows, C.c_int64)) == 0, native.last_error()
        gram = _call(ctx, lib.b2_gram_reset, ctx._h, d)
        gram += _call(ctx, lib.b2_gram_accumulate, ctx._h, L.xp, L.dt, yp, n, d, d, DEV, mp, L.keep)
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
    return {"mse": mse, "cv": cv, "best": int(best[0])}, launches - gram, S, L.ring("reg", masked)


def loo_ref(t, n, mask, keep):
    with np.errstate(invalid="ignore"):                    # one kept row: e = 0 / 0
        mse, cv, best = ridge_loo(t.Xv[:n], t.y["reg"][:n], ALPHAS, None if mask is None else mask[:n], keep)
    return {"mse": mse, "cv": cv, "best": best}


def run_std(ctx, t, L, n):
    mean, sigma, nv, coef, b = t.std
    d, m = L.d, max(n, 1)
    out = ctx.empty((2, m), "f64")
    try:
        launches = _call(ctx, native.load().b2_score_std, ctx._h, L.xp, L.dt, n, d, d, DEV, mean.ctypes.data,
                         sigma.ctypes.data, nv, coef.ctypes.data, b, out.ptr, out.ptr + 8 * m)
        h = out.to_host()
    finally:
        out.free()
    ring = L.ring()
    assert launches == (_launches(n, ring, 1, writes_sums=False) if n > 0 else 0), (L.name, n, launches)
    return {"yhat": h[0, :n], "ystd": h[1, :n]}, ring


def std_ref(t, n):
    yhat, ystd = std_oracle(t.Xv[:n], *t.std)
    return {"yhat": yhat, "ystd": ystd}


def _center(t, n, mask, keep):
    X = t.Xv[:n] if mask is None else t.Xv[:n][mask[:n] == keep]
    return X.mean(axis=0) if len(X) else np.zeros(t.d)


def run_class_sums(ctx, t, L, n, masked, k, center):
    d, cl = L.d, CLASSES[k]
    sums, counts = np.empty((k, d + 1)), np.empty(3)
    launches = _call(ctx, native.load().b2_class_sums, ctx._h, L.xp, L.dt, L.yp[f"cls{k}"], n, d, d, DEV,
                     L.mask(masked), L.keep, cl.ctypes.data, k, center.ctypes.data, sums.ctypes.data,
                     counts.ctypes.data)
    ring = L.ring(f"cls{k}", masked)
    assert launches == _launches(n, ring, 2), (L.name, n, launches)
    return {"sums": sums, "counts": counts}, ring


def class_ref(t, n, mask, keep, k, center):
    """the class sums, counts and per entry the sum of |x - c| over the class (the scale of SUM_TOL)"""
    X, y = t.Xv[:n], t.y[f"cls{k}"][:n]
    m = None if mask is None else mask[:n]
    r = CLS.class_sums(X, y, CLASSES[k], center, row_mask=m, mask_keep=keep)
    kept = np.ones(n, bool) if m is None else m == keep
    scale = np.array([np.abs(X[kept & (y == c)] - center).sum(axis=0) for c in CLASSES[k]]).reshape(k, t.d)
    return {"sums": r["sums"], "counts": np.array([r["kept"], r["unmatched"], r["nonfinite"]]), "scale": scale}


def run_classify(ctx, t, L, n, masked, T, with_y):
    d, m, cl = L.d, max(n, 1), CLASSES[max(T, 2)]
    W, b = t.W[T], t.bW[T]
    dec, lab = ctx.empty((m, T), "f64"), ctx.empty((m,), "f32")
    counts = np.empty(2)
    yp = L.yp[f"cls{max(T, 2)}"] if with_y else None
    mp = L.mask(masked) if with_y else None
    try:
        launches = _call(ctx, native.load().b2_classify, ctx._h, L.xp, L.dt, yp, n, d, d, DEV, mp, L.keep,
                         W.ctypes.data, b.ctypes.data, T, cl.ctypes.data, dec.ptr, lab.ptr,
                         counts.ctypes.data if with_y else None)
        out = {"decision": dec.to_host()[:n], "label": lab.to_host()[:n]}
    finally:
        dec.free(); lab.free()
    if with_y:
        out["counts"] = counts
    ring = _ring(L.xp, yp, mp, d, d, L.es)
    assert launches == _launches(n, ring, 2 if with_y else 1), (L.name, n, T, with_y, launches)
    return out, ring


# ---- the comparisons: each returns the quantity its bound applies to ----------------------------------------------
def glm_err(got, want):
    """worst relative difference of the pass's fp64 sums and ladder (the Hessian where both have one)"""
    keys = ["loss", "grad"] + ([] if "correct" in want else ["const", "sum_y"])
    errs = [rel(got[k], want[k]) for k in keys]
    if got.get("hessian") is not None:
        errs.append(rel(got["hessian"], want["hessian"]))
    errs += [rel(got["ladder"][k], want["ladder"][k]) for k in range(native.GLM_STEPS)]
    return max(errs)


def glm_counts(got, want):
    keys = ["kept", "y_out_of_range", "h_nonpos", "y_nonfinite"] + (["correct", "sum_y"] if "correct" in want else [])
    bad = [k for k in keys if got[k] != want[k]]
    if "correct" in want and got["const"] != 0.0:
        bad.append("const")
    return bad


def rows_err(got, want):
    """per-row fp64 outputs (ystd, yhat), relative to the largest"""
    return rel(got, want)


def loo_err(got, want, kept):
    """(mse relative per alpha, cv of the kept rows relative to the largest); the dropped rows' cv must be NaN"""
    cv = got["cv"]
    assert np.isnan(cv[~kept]).all()
    w_mse, w_cv = np.asarray(want["mse"]), want["cv"]
    if not np.isfinite(w_mse).all():                       # one kept row with an intercept: 0 / 0, NaN everywhere
        assert np.isnan(w_cv).all() and np.isnan(got["mse"]).all() and np.isnan(cv[kept]).all()
        return 0.0, 0.0
    return (float(np.max(np.abs(got["mse"] - w_mse) / np.abs(w_mse))),
            float(np.max(np.abs(cv[kept] - w_cv)) / max(np.max(w_cv), 1e-300)))


def class_sums_err(sums, want, scale):
    """worst |difference| of a class-sum entry over the sum of |x - c| of the class"""
    d = scale.shape[1]
    return float(np.max(np.abs(sums[:, :d] - want[:, :d]) / np.maximum(scale, 1e-300))) if scale.size else 0.0


def decision_err(dec, X, W, b):
    """worst |decision - eta| / (sum_j |x_j w_j| + |b|) per entry, eta exact: a fp64 product screens every row, and
    the rows within 8x of DEC_TOL of it, and the 64 worst, are compared with the long-double decision"""
    if len(X) == 0:
        return 0.0
    ref, scale = X @ W.T + b, np.abs(X) @ np.abs(W).T + np.abs(b)
    row = np.max(np.abs(dec - ref) / scale, axis=1)
    row = np.where(np.isnan(row), np.inf, row)
    sel = np.union1d(np.flatnonzero(row > DEC_TOL / 8), np.argsort(row)[-64:])
    if sel.size > 20_000:
        return float(np.max(row))
    ld = _longdouble_decision(X[sel], W, b)
    e = np.abs(np.asarray(dec[sel], np.longdouble) - ld) / scale[sel]
    e = float(np.max(np.where(np.isnan(e), np.inf, e)))
    rest = np.delete(row, sel)
    return max(e, float(np.max(rest)) if rest.size else 0.0)


def check_labels(lab, X, W, b, classes):
    eta = X @ W.T + b
    if W.shape[0] == 1:
        ref, margin = classes[(eta[:, 0] > 0).astype(int)], np.abs(eta[:, 0])
    else:
        ref = classes[np.argmax(eta, axis=1)]
        top = np.sort(eta, axis=1)
        margin = top[:, -1] - top[:, -2]
    clear = margin > 1e-9
    assert np.array_equal(lab[clear], ref[clear])


def check_classify(out, t, n, kept, T, with_y):
    """decision within DEC_TOL and labels on the kept rows (every row without a mask), counts equal; the error"""
    W, b, cl = t.W[T], t.bW[T], CLASSES[max(T, 2)]
    X = t.Xv[:n][kept]
    err = decision_err(out["decision"][kept], X, W, b)
    assert err < DEC_TOL, err
    check_labels(out["label"][kept], X, W, b, cl)
    if with_y:
        y = t.y[f"cls{max(T, 2)}"][:n]
        assert out["counts"].tolist() == [kept.sum(), np.sum(kept & (y == out["label"]))]
    return err


def check_class_sums(out, want, t, n, mask, keep, k, center):
    """sums within SUM_TOL (the worst entry also against math.fsum), counts equal; the error"""
    sums, d = out["sums"], t.d
    assert np.array_equal(sums[:, d], want["sums"][:, d]) and np.array_equal(out["counts"], want["counts"])
    err = class_sums_err(sums, want["sums"], want["scale"])
    if want["scale"].size and err > 0:
        c, j = np.unravel_index(np.argmax(np.abs(sums[:, :d] - want["sums"][:, :d]) /
                                          np.maximum(want["scale"], 1e-300)), (k, d))
        y = t.y[f"cls{k}"][:n]
        kept = np.ones(n, bool) if mask is None else mask[:n] == keep
        v = t.Xv[:n][kept & (y == CLASSES[k][c]), j] - center[j]
        err = max(err, abs(sums[c, j] - math.fsum(v)) / max(want["scale"][c, j], 1e-300))
    assert err < SUM_TOL, err
    return err


def _same(a, b):
    return all(np.array_equal(a[k], b[k], equal_nan=True) for k in a if a[k] is not None)


# ---- (1) and (2): long runs against the references, ring against direct on the same rows -------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", WIDTHS, ids=[f"{k}-d{d}" for k, d in WIDTHS])
def test_long_runs_against_reference_and_ring_against_direct(ctx, kind, d):
    G = ctx.info()["sm_count"]
    n = n_long(G)
    whole = n // TILE * TILE                       # the same rows without the tail: both flavours give tile i to CTA i
    sizes = (n, whole, whole + 1)
    t = Table(kind, d, n, seed=100 * d + (7 if kind == "bf16" else 0))
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    lay = _layouts(dev, with_mask=True)
    worst = defaultdict(float)
    rings = defaultdict(set)                       # pass -> the (layout, ring) pairs that ran

    def note(group, err):
        worst[group] = max(worst[group], err)

    try:
        for masked in (False, True):
            m = mask if masked else None
            kept = np.ones(n, bool) if m is None else m == 1
            names = ["ring", "x+4", "y+4"] + (["mask+1"] if masked else [])
            # the GLM and logistic passes with their line search
            for loss in LOSSES:
                want = glm_ref(t, n, m, 1, loss)
                base = {}
                for nn in sizes:
                    base[nn], ring = run_glm(ctx, t, lay["ring"], nn, masked, loss)
                    assert ring
                    again, _ = run_glm(ctx, t, lay["ring"], nn, masked, loss)
                    assert _same(base[nn], again), (loss, nn)
                got = base[n]
                assert not glm_counts(got, want), (loss, masked, glm_counts(got, want))
                err = glm_err(got, want)
                assert err < PASS_TOL, (loss, masked, err)
                note("glm/logistic", err)
                grad, _ = run_glm(ctx, t, lay["ring"], n, masked, loss, hess=False)   # two CTAs per SM
                assert not glm_counts(grad, want) and glm_err(grad, want) < PASS_TOL, (loss, glm_err(grad, want))
                note("glm/logistic", glm_err(grad, want))
                for name in names[1:]:
                    for nn in sizes:
                        other, ring = run_glm(ctx, t, lay[name], nn, masked, loss)
                        rings["glm"].add((name, ring))
                        if not ring and nn == whole:
                            assert _same(other, base[nn]), (loss, name)
                        elif nn == n:
                            assert not glm_counts(other, want) and glm_err(other, want) < PASS_TOL, (loss, name)
            # the leave-one-out pass on the exact Gram
            want = loo_ref(t, n, m, 1)
            base = {nn: run_loo(ctx, t, lay["ring"], nn, masked) for nn in sizes}
            got, _, S_ring, ring = base[n]
            assert ring and got["best"] == want["best"]
            e_mse, e_cv = loo_err(got, want, kept)
            assert e_mse < LOO_TOL and e_cv < LOO_TOL, (masked, e_mse, e_cv)
            note("loo mse", e_mse); note("loo cv", e_cv)
            again = run_loo(ctx, t, lay["ring"], n, masked)[0]
            assert _same(again, got)
            for name in names[1:]:
                for nn in sizes:
                    other, launches, S, ring = run_loo(ctx, t, lay[name], nn, masked)
                    rings["loo"].add((name, ring))
                    r_got, r_launches, r_S, _ = base[nn]
                    # the pass's own launches: one pass-and-reduce pair per flavour part
                    assert r_launches - launches == _launches(nn, True, 2) - _launches(nn, ring, 2), (name, nn)
                    if np.array_equal(S, r_S):
                        assert np.array_equal(other["cv"], r_got["cv"], equal_nan=True), (name, nn)
                        if nn == whole or ring:
                            assert np.array_equal(other["mse"], r_got["mse"]), (name, nn)
                    else:    # another Gram summation order moves the model, and every e with it, within the Gram's error
                        worst["loo: S differs between layouts"] = 1.0
                        k = kept[:nn]
                        assert max(loo_err(other, loo_ref(t, nn, None if m is None else m[:nn], 1), k)) < LOO_TOL
                    if nn == n:
                        assert max(loo_err(other, want, kept)) < LOO_TOL, name
            # the class sums at K = 2 and 32
            center = _center(t, n, m, 1)
            for k in (2, 32):
                want = {nn: class_ref(t, nn, m, 1, k, center) for nn in sizes[:2]}
                got, ring = run_class_sums(ctx, t, lay["ring"], n, masked, k, center)
                assert ring
                note("class sums", check_class_sums(got, want[n], t, n, m, 1, k, center))
                assert _same(run_class_sums(ctx, t, lay["ring"], n, masked, k, center)[0], got)
                for name in names[1:]:
                    for nn in sizes[:2]:
                        other, ring = run_class_sums(ctx, t, lay[name], nn, masked, k, center)
                        rings["class sums"].add((name, ring))
                        note("class sums", check_class_sums(other, want[nn], t, nn, m, 1, k, center))
        # score_std: no y, no mask
        want = std_ref(t, n)
        base = {nn: run_std(ctx, t, lay["ring"], nn) for nn in sizes}
        got = base[n][0]
        assert base[n][1]
        for key in ("ystd", "yhat"):
            err = rows_err(got[key], want[key])
            assert err < STD_TOL, (key, err)
            note("score_std", err)
        assert _same(run_std(ctx, t, lay["ring"], n)[0], got)
        for nn in sizes:
            other, ring = run_std(ctx, t, lay["x+4"], nn)
            assert not ring and _same(other, base[nn][0]), nn
        # classify at T = 1, 3, 32 with and without y
        for T in (1, 3, 32):
            for with_y in (False, True):
                for masked in ((False, True) if with_y else (False,)):
                    kept = mask == 1 if masked else np.ones(n, bool)
                    base = {nn: run_classify(ctx, t, lay["ring"], nn, masked, T, with_y) for nn in sizes}
                    got, ring = base[n]
                    assert ring
                    note("decision", check_classify(got, t, n, np.ones(n, bool), T, False))
                    if with_y:
                        check_classify(got, t, n, kept, T, True)
                    assert _same(run_classify(ctx, t, lay["ring"], n, masked, T, with_y)[0], got)
                    names = ["x+4"] + (["y+4"] if with_y else []) + (["mask+1"] if masked else [])
                    for name in names:
                        for nn in sizes:
                            other, ring = run_classify(ctx, t, lay[name], nn, masked, T, with_y)
                            rings["classify"].add((name, ring))
                            assert np.array_equal(other["decision"], base[nn][0]["decision"]), (name, nn)
                            assert np.array_equal(other["label"], base[nn][0]["label"]), (name, nn)
                            if with_y:
                                assert np.array_equal(other["counts"], base[nn][0]["counts"]), (name, nn)
    finally:
        dev.free()
    # X or y off its 16-byte boundary never takes the ring; a misaligned mask only for d <= 16
    for pas, seen in rings.items():
        for name, ring in seen:
            assert ring == (name == "mask+1" and d > 16), (pas, name, ring)
    print(f"\n[long {kind} d={d}, n={n}, G={G}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (3) edge row counts --------------------------------------------------------------------------------------------
EDGES = [("f32", 8), ("f32", 128), ("bf16", 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", EDGES, ids=[f"{k}-d{d}" for k, d in EDGES])
def test_edge_row_counts(ctx, kind, d):
    G = ctx.info()["sm_count"]
    sizes = n_edge(G)
    t = Table(kind, d, max(sizes), seed=300 + d)
    mask = (np.arange(t.n) % 7 != 3).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    L = Layout(dev, "ring")
    worst = defaultdict(float)
    lib = native.load()
    try:
        for n in sizes:
            for masked in (False, True):
                m = mask[:n] if masked else None
                kept = np.ones(n, bool) if m is None else m == 1
                for loss in ("log p=1.5", "binomial"):
                    got, ring = run_glm(ctx, t, L, n, masked, loss)
                    want = glm_ref(t, n, m, 1, loss)
                    assert ring and not glm_counts(got, want), (n, loss, glm_counts(got, want))
                    err = glm_err(got, want)
                    assert err < PASS_TOL, (n, loss, err)
                    worst["glm/logistic"] = max(worst["glm/logistic"], err)
                    if n == 0:      # no rows: zero sums, a zero Hessian and a zero ladder
                        assert not np.any(got["ladder"]) and not np.any(got["hessian"]) and not np.any(got["grad"])
                if n == 0:          # b2_ridge_loo refuses a call without a kept row (include/b2gram.h)
                    out = np.empty(ALPHAS.size)
                    rc = lib.b2_ridge_loo(ctx._h, L.xp, L.dt, L.yp["reg"], 0, d, d, DEV, L.mask(masked), 1,
                                          ALPHAS.ctypes.data, ALPHAS.size, 1, out.ctypes.data, None,
                                          _p(np.zeros(1, np.int32), C.c_int), np.empty(d).ctypes.data,
                                          _p(np.empty(1), C.c_double))
                    assert rc == native.E_ARG and "no row kept" in native.last_error()
                else:
                    got = run_loo(ctx, t, L, n, masked)[0]
                    e_mse, e_cv = loo_err(got, loo_ref(t, n, m, 1), kept)
                    assert e_mse < LOO_TOL and e_cv < LOO_TOL, (n, e_mse, e_cv)
                    worst["loo"] = max(worst["loo"], e_mse, e_cv)
                center = _center(t, n, m, 1)
                got, _ = run_class_sums(ctx, t, L, n, masked, 32, center)
                err = check_class_sums(got, class_ref(t, n, m, 1, 32, center), t, n, m, 1, 32, center)
                worst["class sums"] = max(worst["class sums"], err)
                got, _ = run_classify(ctx, t, L, n, masked, 3, True)
                worst["decision"] = max(worst["decision"], check_classify(got, t, n, np.ones(n, bool), 3, False))
                check_classify(got, t, n, kept, 3, True)
            got, _ = run_std(ctx, t, L, n)       # n = 0: no launch, nothing written
            want = std_ref(t, n)
            for key in ("ystd", "yhat"):
                err = rows_err(got[key], want[key])
                assert err < STD_TOL, (n, key, err)
                worst["score_std"] = max(worst["score_std"], err)
    finally:
        dev.free()
    print(f"\n[edges {kind} d={d}, n in {sizes}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (4) masks that empty whole tiles and whole CTAs ----------------------------------------------------------------
def _tile_masks(n, G):
    tile = np.arange(n) // TILE
    third = (tile % 3 != 2).astype(np.uint8)
    return [("every third tile", third, 1), ("tiles t = 0 mod G", (tile % G != 0).astype(np.uint8), 1),
            ("all rows", np.zeros(n, np.uint8), 1), ("mask_keep = 0", third, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", [("f32", 8), ("f32", 64)], ids=["f32-d8", "f32-d64"])
def test_masks_that_empty_tiles(ctx, kind, d):
    G = ctx.info()["sm_count"]
    n = n_long(G)
    worst = defaultdict(float)
    for label, mask, keep in _tile_masks(n, G):
        kept = mask == keep
        t = Table(kind, d, n, seed=500 + d, dropped=~kept)
        dev = Dev(ctx, t, mask, keep)
        lay = _layouts(dev, with_mask=False)
        try:
            for name in ("ring", "x+4"):
                L = lay[name]
                for loss in ("log p=1.5", "binomial"):
                    got, ring = run_glm(ctx, t, L, n, True, loss)
                    assert ring == (name == "ring")
                    want = glm_ref(t, n, mask, keep, loss)
                    assert not glm_counts(got, want), (label, name, loss, glm_counts(got, want))
                    assert all(np.all(np.isfinite(got[k])) for k in ("loss", "grad", "hessian", "ladder"))
                    err = glm_err(got, want)
                    assert err < PASS_TOL, (label, name, loss, err)
                    worst["glm/logistic"] = max(worst["glm/logistic"], err)
                lib = native.load()
                if not kept.any():
                    out = np.empty(ALPHAS.size)
                    rc = lib.b2_ridge_loo(ctx._h, L.xp, L.dt, L.yp["reg"], n, d, d, DEV, L.mp, keep,
                                          ALPHAS.ctypes.data, ALPHAS.size, 1, out.ctypes.data, None,
                                          _p(np.zeros(1, np.int32), C.c_int), np.empty(d).ctypes.data,
                                          _p(np.empty(1), C.c_double))
                    assert rc == native.E_ARG and "no row kept" in native.last_error(), label
                else:
                    got = run_loo(ctx, t, L, n, True)[0]
                    assert np.all(np.isfinite(got["mse"]))
                    e_mse, e_cv = loo_err(got, loo_ref(t, n, mask, keep), kept)
                    assert e_mse < LOO_TOL and e_cv < LOO_TOL, (label, name, e_mse, e_cv)
                    worst["loo"] = max(worst["loo"], e_mse, e_cv)
                center = _center(t, n, mask, keep)
                got, _ = run_class_sums(ctx, t, L, n, True, 32, center)
                assert np.all(np.isfinite(got["sums"]))
                err = check_class_sums(got, class_ref(t, n, mask, keep, 32, center), t, n, mask, keep, 32, center)
                worst["class sums"] = max(worst["class sums"], err)
                got, _ = run_classify(ctx, t, L, n, True, 32, True)
                err = check_classify(got, t, n, kept, 32, True)
                worst["decision"] = max(worst["decision"], err)
        finally:
            dev.free()
    print(f"\n[tile masks {kind} d={d}, n={n}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (5) the bounds see the faults this file targets (CPU) ----------------------------------------------------------
def _fault_rows(n, t_row, how):
    """row order of the pass with tile t_row dropped or counted twice"""
    idx = np.arange(n)
    tile = idx[t_row * TILE:(t_row + 1) * TILE]
    return np.delete(idx, tile) if how == "dropped" else np.r_[idx, tile]


def test_bounds_see_the_faults():
    G = H100_SMS
    n = n_long(G)
    t = Table("f32", 16, n, seed=5)
    bad = 3 * 2 * G + 5                # a tile after the first wrap of a CTA at two CTAs per SM
    stale = bad - 3 * 2 * G            # the tile that CTA streamed three tiles earlier through the same slot
    rows_bad, rows_stale = slice(bad * TILE, (bad + 1) * TILE), slice(stale * TILE, (stale + 1) * TILE)
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)

    def faulty(how):
        """a Table view whose rows are those of the faulty pass"""
        r = _fault_rows(n, bad, how)
        f = Table.__new__(Table)
        f.__dict__.update(t.__dict__)
        f.Xv, f.y, f.n = t.Xv[r], {k: v[r] for k, v in t.y.items()}, len(r)
        return f, mask[r]

    moved = {}
    for how in ("dropped", "twice"):
        f, fm = faulty(how)
        for loss in LOSSES:
            want = glm_ref(t, n, mask, 1, loss)
            moved[loss, how] = glm_err(glm_ref(f, f.n, fm, 1, loss), want) / PASS_TOL
        center = _center(t, n, mask, 1)
        for k in (2, 32):
            want = class_ref(t, n, mask, 1, k, center)
            got = class_ref(f, f.n, fm, 1, k, center)
            moved[f"class sums K={k}", how] = class_sums_err(got["sums"], want["sums"], want["scale"]) / SUM_TOL
        # the leave-one-out sums: the per-alpha sums of e^2 over the pass's rows, over the kept rows of the Gram
        want = loo_ref(t, n, mask, 1)
        e2 = np.full((n, ALPHAS.size), 0.0)
        e2[mask == 1] = want["cv"]
        r = _fault_rows(n, bad, how)
        got = {"mse": e2[r].sum(axis=0) / mask.sum(), "cv": np.where(mask[:, None] == 1, e2, np.nan)}
        moved["loo mse", how] = loo_err(got, want, mask == 1)[0] / LOO_TOL
    # per-row outputs: the stale slot's rows in place of the tile's
    want = std_ref(t, n)
    for key in ("ystd", "yhat"):
        got = want[key].copy()
        got[rows_bad] = want[key][rows_stale]
        moved[key, "stale"] = rows_err(got, want[key]) / STD_TOL
    want = loo_ref(t, n, None, 1)
    got = {"mse": want["mse"], "cv": want["cv"].copy()}
    got["cv"][rows_bad] = want["cv"][rows_stale]
    moved["loo cv", "stale"] = loo_err(got, want, np.ones(n, bool))[1] / LOO_TOL
    for T in (1, 3, 32):
        W, b = t.W[T], t.bW[T]
        dec = t.Xv @ W.T + b
        dec[rows_bad] = dec[rows_stale]
        moved[f"decision T={T}", "stale"] = decision_err(dec, t.Xv, W, b) / DEC_TOL
    small = {k: v for k, v in moved.items() if not v >= 100}
    assert not small, small


# ---- (6) host rows across staging blocks ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_host_rows_class_sums_and_classify(ctx):
    """b2_class_sums (K = 32) and b2_classify (T = 32, 256 bytes of decision per row) on three staging blocks of
    pageable and pinned host rows"""
    d, n = 64, 2 * (1 << 18) + 4321
    t = Table("f32", d, n, seed=77)
    mask = (np.arange(n) % 7 != 3).astype(np.uint8)
    kept = mask == 1
    y = t.y["cls32"]
    center = _center(t, n, mask, 1)
    W, b, cl = t.W[32], t.bW[32], CLASSES[32]
    lib = native.load()
    out = {}
    for kind in ("pageable", "pinned"):
        keep_alive = []
        if kind == "pageable":
            xp, yp, mp = t.up.ctypes.data, y.ctypes.data, mask.ctypes.data
        else:
            ptrs = []
            for a in (t.up, y, mask):
                p = ctx.pinned(a.shape, a.dtype)
                p.array[:] = a
                keep_alive.append(p)
                ptrs.append(p.ptr)
            xp, yp, mp = ptrs
        try:
            sums, counts = np.empty((32, d + 1)), np.empty(3)
            l1 = _call(ctx, lib.b2_class_sums, ctx._h, xp, b2.F32, yp, n, d, d, native.MEM_HOST, mp, 1,
                       cl.ctypes.data, 32, center.ctypes.data, sums.ctypes.data, counts.ctypes.data)
            dec, lab, cc = np.empty((n, 32)), np.empty(n, np.float32), np.empty(2)
            l2 = _call(ctx, lib.b2_classify, ctx._h, xp, b2.F32, yp, n, d, d, native.MEM_HOST, mp, 1, W.ctypes.data,
                       b.ctypes.data, 32, cl.ctypes.data, dec.ctypes.data, lab.ctypes.data, cc.ctypes.data)
        finally:
            for p in keep_alive:
                p.free()
        out[kind] = ({"sums": sums, "counts": counts}, {"decision": dec, "label": lab, "counts": cc}, (l1, l2))
    pag, pin = out["pageable"], out["pinned"]
    assert pag[2] == pin[2]
    assert _same(pag[0], pin[0]) and _same(pag[1], pin[1])
    e_sums = check_class_sums(pag[0], class_ref(t, n, mask, 1, 32, center), t, n, mask, 1, 32, center)
    e_dec = check_classify(pag[1], t, n, np.ones(n, bool), 32, False)
    check_classify(pag[1], t, n, kept, 32, True)
    print(f"\n[host rows, 3 staging blocks, d={d}] class sums {e_sums:.2e}, decision {e_dec:.2e}")
