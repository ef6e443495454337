"""Multinomial LogisticRegression on the H100: b2_multinomial_pass / b2_multinomial_line_search against scikit-learn's
LinearModelLoss(HalfMultinomialLoss) on float64 copies of the same stored rows (the numpy stand-in of
tests/test_multinomial_driver.py), on every row layout; b2_softmax_rows against sklearn.utils.extmath.softmax; the
estimator against LogisticRegression(solver="newton-cholesky"); a 1 M x 128 fit from float64 host columns with device
labels; and the ABI refusals."""
import warnings

import numpy as np
import pytest
from scipy.special import softmax as sp_softmax
from sklearn import linear_model
from sklearn.metrics import accuracy_score
from sklearn.utils.extmath import softmax as sk_softmax

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from test_multinomial_driver import NumpyMultinomialContext, make_data, rel_err

pytestmark = pytest.mark.gpu

E_ARG, E_UNSUPPORTED = -1, -6
PASS_TOL = 1e-13
REF = NumpyMultinomialContext()


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def _rows(n, d, k, seed, kind):
    """(stored rows with 3 spare columns, their float64 values, y (k fp32 labels, a few rows of no class), classes,
    coef (k, d + 1), step (k, d + 1))"""
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d + 3)) * 0.5).astype(np.float32)
    up = b2.native.to_bf16_bits(X) if kind == "bf16" else X
    Xv = b2.native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
    classes = np.sort(rng.choice(np.arange(-50, 50), size=k, replace=False)).astype(np.float32)
    coef = rng.normal(size=(k, d + 1)) * 3.0 / np.sqrt(d)
    eta = Xv[:, :d] @ coef[:, :d].T + coef[:, d]
    cdf = np.cumsum(sp_softmax(eta, axis=1), axis=1)
    t = np.minimum((cdf < rng.uniform(size=(n, 1))).sum(axis=1), k - 1)   # a draw from each row's softmax
    y = classes[t]
    y[[11, 12]] = 1000.0                              # no class
    y[13] = np.nan
    y[14] = np.inf
    step = rng.normal(size=(k, d + 1)) * 2.0 / np.sqrt(d)
    return up, Xv, y, classes, coef, step


def _raw_pass(ctx, ptr, dt, yp, n, d, ldx, mk, mp, classes, coef, fi, hess):
    k = classes.size
    sums = np.empty(5 + k * (d + 1))
    H = np.empty((k, k, d + 1, d + 1)) if hess else None
    rc = native.load().b2_multinomial_pass(ctx._h, ptr, dt, yp, n, d, ldx, mk, mp, 1, classes.ctypes.data, k,
                                           coef.ctypes.data, int(fi), sums.ctypes.data, H.ctypes.data if hess else None)
    assert rc == 0, native.last_error()
    return sums, H


def _raw_ladder(ctx, ptr, dt, yp, n, d, ldx, mk, mp, classes, coef, step):
    out = np.empty(21)
    rc = native.load().b2_multinomial_line_search(ctx._h, ptr, dt, yp, n, d, ldx, mk, mp, 1, classes.ctypes.data,
                                                  classes.size, coef.ctypes.data, step.ctypes.data, 21, out.ctypes.data)
    assert rc == 0, native.last_error()
    return out


def _check(sums, H, want, k, d):
    got = dict(zip(("loss", "kept", "unmatched", "nonfinite", "correct"), sums[:5]))
    for key in ("kept", "unmatched", "nonfinite", "correct"):
        assert got[key] == want[key], (key, got[key], want[key])
    errs = [rel(got["loss"], want["loss"]), rel(sums[5:].reshape(k, d + 1), want["grad"])]
    if H is not None:
        for a in range(k):
            for c in range(k):
                assert np.array_equal(H[a, c], H[a, c].T) and np.array_equal(H[a, c], H[c, a])
                errs.append(rel(H[a, c], want["hessian"][a, c]))
    return max(errs)


def _reference(Xref, y, classes, coef, fi, mref):
    """the sums over the kept rows: the stand-in's on the rows of some class, and by hand on the rows of none (NaN and
    inf included), whose loss is log(s) + m and whose g is p"""
    keep = np.ones(len(y), bool) if mref is None else mref == 1
    t = REF._targets(y, classes)
    known, other = keep & (t >= 0), keep & (t < 0)
    want = REF.multinomial_pass(Xref, y, classes, coef, row_mask=known.astype(np.uint8), fit_intercept=fi)
    W = coef.copy()
    if not fi:
        W[:, -1] = 0.0
    Z = np.c_[Xref[other], np.ones(int(other.sum()))]
    eta = Z @ W.T
    m = eta.max(axis=1)
    e = np.exp(eta - m[:, None])
    sm = e.sum(axis=1)
    p = e / sm[:, None]
    want["loss"] += np.sum(np.log(sm) + m)
    want["grad"] = want["grad"] + p.T @ Z
    k = classes.size
    for a in range(k):
        for c in range(k):
            h = p[:, a] * (1.0 - p[:, a]) if a == c else -p[:, a] * p[:, c]
            want["hessian"][a, c] += Z.T @ (h[:, None] * Z)
    want["kept"] = float(keep.sum())
    want["unmatched"] = float(other.sum())
    want["nonfinite"] = float(np.sum(keep & ~np.isfinite(y)))
    return want


def _reference_ladder(Xref, y, classes, coef, step, mref):
    keep = np.ones(len(y), bool) if mref is None else mref == 1
    t = REF._targets(y, classes)
    known, other = keep & (t >= 0), keep & (t < 0)
    lw = REF.multinomial_line_search(Xref, y, classes, coef, step, row_mask=known.astype(np.uint8))
    Z = np.c_[Xref[other], np.ones(int(other.sum()))]
    eta, deta = Z @ coef.T, Z @ step.T
    for s in range(21):
        v = eta + 0.5 ** s * deta
        m = v.max(axis=1)
        lw[s] += np.sum(np.log(np.exp(v - m[:, None]).sum(axis=1)) + m)
    return lw


LAYOUT_D = [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128]


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", LAYOUT_D)
def test_pass_sums_every_layout(ctx, kind, d):
    n = 4133                                         # ring tiles, then a partial tile on the direct kernel
    dt = b2.BF16 if kind == "bf16" else b2.F32
    es = 2 if kind == "bf16" else 4
    worst = 0.0
    for k, fi in ((3, True), (10, False), (32, True)):
        if k == 32 and d not in (1, 17, 128):
            continue
        up, Xv, y, classes, coef, step = _rows(n, d, k, 100 * d + k, kind)
        mask = (np.arange(n) % 5 != 2).astype(np.uint8)
        cont = np.ascontiguousarray(up[:, :d])
        Xd, yd, md = ctx.to_device(cont, kind), ctx.to_device(y), ctx.to_device(mask)
        Xs = ctx.to_device(np.ascontiguousarray(up), kind)         # ldx = d + 3, starting one element in
        try:
            layouts = [("host", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, None, Xv[:, :d], None),
                       ("device", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, None, Xv[:, :d], None),
                       ("strided", Xs.ptr + es, yd.ptr, d + 3, native.MEM_DEVICE, None, Xv[:, 1:d + 1], None),
                       ("device masked", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, md.ptr, Xv[:, :d], mask),
                       ("host masked", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, mask.ctypes.data,
                        Xv[:, :d], mask)]
            for name, xp, yp, ldx, mk, mp, Xref, mref in layouts:
                sums, H = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, coef, fi, True)
                sums2, H2 = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, coef, fi, True)
                assert np.array_equal(sums, sums2) and np.array_equal(H, H2), name
                g_only, _ = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, coef, fi, False)
                assert np.array_equal(sums[1:5], g_only[1:5]), name
                ladder = _raw_ladder(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, coef, step)
                assert np.array_equal(ladder, _raw_ladder(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, coef, step))
                want = _reference(Xref, y, classes, coef, fi, mref)
                err = max(_check(sums, H, want, k, d), _check(g_only, None, want, k, d))
                lw = _reference_ladder(Xref, y, classes, coef, step, mref)
                err = max(err, max(rel(ladder[s], lw[s]) for s in range(21)))
                assert err < PASS_TOL, (name, k, err)
                worst = max(worst, err)
        finally:
            for a in (Xd, yd, md, Xs):
                a.free()
    print(f"\n[multinomial pass {kind} d={d}] worst relative difference {worst:.2e}")


def test_many_tiles_per_cta_and_host_blocks(ctx):
    """K = 10 (55 pairs, two row slices): every CTA streams many ring tiles; host rows span three staging blocks of
    262 144 rows, the last one partial, whose sums each add to the previous ones; repeats are bit-identical"""
    n, d, k = 2 * (1 << 18) + 32 * 132 * 9 + 17, 24, 10
    up, Xv, y, classes, coef, step = _rows(n, d, k, 7, "f32")
    y[11:15] = classes[0]
    Xc = np.ascontiguousarray(up[:, :d])
    Xd, yd = ctx.to_device(Xc), ctx.to_device(y)
    try:
        want = REF.multinomial_pass(Xv[:, :d], y, classes, coef, hessian=True)
        lw = REF.multinomial_line_search(Xv[:, :d], y, classes, coef, step)
        for xp, yp, mk in ((Xd.ptr, yd.ptr, native.MEM_DEVICE), (Xc.ctypes.data, y.ctypes.data, native.MEM_HOST)):
            sums, H = _raw_pass(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, coef, True, True)
            sums2, H2 = _raw_pass(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, coef, True, True)
            assert np.array_equal(sums, sums2) and np.array_equal(H, H2)
            g_only, _ = _raw_pass(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, coef, True, False)
            assert max(_check(sums, H, want, k, d), _check(g_only, None, want, k, d)) < PASS_TOL
            ladder = _raw_ladder(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, coef, step)
            assert max(rel(ladder[s], lw[s]) for s in range(21)) < PASS_TOL
    finally:
        Xd.free()
        yd.free()


@pytest.mark.parametrize("k", [3, 10, 32])
def test_softmax_rows_matches_sklearn(ctx, k):
    rng = np.random.default_rng(k)
    v = rng.normal(size=(5003, k)) * 20.0
    want = sk_softmax(v.copy())
    dv = ctx.to_device(v)
    try:
        ctx.softmax_rows(dv)
        got = dv.to_host()
    finally:
        dv.free()
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-15)
    host = v.copy()
    ctx.softmax_rows(host)
    assert np.array_equal(host, got)


def _fit_both(ctx, X, y, **kw):
    ours = b2.B200MultinomialLogisticRegression(ctx=ctx, **kw)
    ref = linear_model.LogisticRegression(solver="newton-cholesky", **kw)
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X, y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X.astype(np.float32).astype(np.float64), y)
    return ours, ref, [w.category for w in w_ours], [w.category for w in w_ref]


@pytest.mark.parametrize("k", [3, 4, 7, 32])
@pytest.mark.parametrize("C", [1e-2, 1.0, 1e4, np.inf])
def test_estimator_matches_sklearn(ctx, k, C):
    X, t = make_data(n=16384, d=24, k=k, seed=k)
    ours, ref, cat_ours, cat_ref = _fit_both(ctx, X, t, C=C)
    assert cat_ours == cat_ref
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    tol = 1e-10 if C != 1e4 else 1e-8                # 1e4: the class-mean direction held by the tiny penalty alone
    assert rel_err(ours, ref) <= tol, rel_err(ours, ref)
    assert rel_err(ours, ref, centred=True) <= 1e-10
    assert np.array_equal(ours.predict(X), ref.predict(X))
    np.testing.assert_allclose(ours.predict_proba(X), ref.predict_proba(X), rtol=0, atol=1e-12)
    assert ours.score(X, t) == accuracy_score(t, ref.predict(X))
    Xd = ctx.to_device(X.astype(np.float32))
    try:
        proba = ours.predict_proba(Xd)
        # the device softmax of the same decisions: CUDA's exp against the host's, each within an ulp or so
        np.testing.assert_allclose(proba.to_host(), ours.predict_proba(X), rtol=0, atol=4e-15)
        proba.free()
        lab = ours.predict(Xd)
        np.testing.assert_array_equal(lab.to_host(), ours.predict(X).astype(np.float32))
        lab.free()
    finally:
        Xd.free()


def test_large_fit_from_float64_columns_with_device_labels(ctx):
    n, d, k = 1_000_000, 128, 10
    rng = np.random.default_rng(5)
    X = rng.normal(size=(n, d)).astype(np.float32).astype(np.float64)
    B = rng.normal(size=(d, k)) / np.sqrt(d)
    t = np.argmax(X @ B + rng.gumbel(size=(n, k)), axis=1)
    y = (2.0 * t - 3.0).astype(np.float32)
    Xd = ctx.upload_columns([X[:, j] for j in range(d)])
    yd = ctx.to_device(y)
    try:
        ours = b2.B200MultinomialLogisticRegression(ctx=ctx).fit(Xd, yd)
    finally:
        yd.free()
    try:
        assert list(ours.classes_) == list(np.unique(y)) and ours.classes_.dtype == np.float32
        ref = linear_model.LogisticRegression(solver="newton-cholesky").fit(X, y)
        assert np.array_equal(ours.n_iter_, ref.n_iter_)
        assert rel_err(ours, ref) <= 1e-10, rel_err(ours, ref)
        assert np.mean(ours.predict(Xd).to_host() == ref.predict(X)) == 1.0
    finally:
        Xd.free()


def test_abi_refusals(ctx):
    lib = native.load()
    n, d = 64, 4
    X = np.zeros((n, d), np.float32)
    y = np.zeros(n, np.float32)
    cl = np.array([0, 1, 2], np.float32)
    coef = np.zeros((3, d + 1))
    sums = np.empty(5 + 3 * (d + 1))
    out = np.empty(21)
    args = (ctx._h, X.ctypes.data, b2.F32, y.ctypes.data, n, d, d, native.MEM_HOST, None, 1)

    def mp(classes, k, s=sums.ctypes.data):
        return lib.b2_multinomial_pass(*args, classes.ctypes.data, k, coef.ctypes.data, 1, s, None)

    assert mp(cl, 3) == 0
    assert mp(cl[:2], 2) == E_ARG                       # two classes: the binary pass
    big = np.arange(33, dtype=np.float32)
    assert mp(big, 33) == E_ARG
    assert mp(np.array([0, 2, 1], np.float32), 3) == E_ARG
    assert mp(np.array([0, np.nan, 2], np.float32), 3) == E_ARG
    assert mp(np.array([0, 0, 2], np.float32), 3) == E_ARG
    assert mp(cl, 3, None) == E_ARG
    ls = lambda steps, o=out.ctypes.data: lib.b2_multinomial_line_search(  # noqa: E731
        *args, cl.ctypes.data, 3, coef.ctypes.data, coef.ctypes.data, steps, o)
    assert ls(21) == 0
    assert ls(0) == E_ARG and ls(22) == E_ARG and ls(5, None) == E_ARG
    assert lib.b2_softmax_rows(ctx._h, None, 4, 3, native.MEM_DEVICE) == E_ARG
    assert lib.b2_softmax_rows(ctx._h, out.ctypes.data, 1, 0, native.MEM_HOST) == E_ARG
    # two contexts of one device attached as ranks 0 and 1: the passes' sums are not exchanged, so both refuse
    other = b2.Context(0)
    try:
        b2.Context.comm_p2p_attach_local([ctx, other])
        assert mp(cl, 3) == E_UNSUPPORTED
        assert ls(21) == E_UNSUPPORTED
    finally:
        for c in (ctx, other):
            c.comm_p2p_detach()
        other.close()
    assert mp(cl, 3) == 0 and ls(21) == 0                # detached: one rank again
