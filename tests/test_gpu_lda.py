"""LinearDiscriminantAnalysis on the H100: b2_class_scatter against a float64 numpy statement of the pass on the same
stored rows, on every row layout, with many tiles per CTA and over several host staging blocks; the estimator against
scikit-learn on float64 copies of the staged rows; a 1 M x 128 fit from device rows and device labels; the ABI
refusals."""
import warnings

import numpy as np
import pytest
from sklearn.discriminant_analysis import LinearDiscriminantAnalysis

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native

pytestmark = pytest.mark.gpu

E_ARG = -1
PASS_TOL = 1e-13


def _raw(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means, weights):
    cl = np.ascontiguousarray(classes, dtype=np.float32)
    m = np.ascontiguousarray(means, dtype=np.float64)
    w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64)
    S = np.full((d, d), np.nan)
    counts = np.full(3, np.nan)
    rc = native.load().b2_class_scatter(ctx._h, xp, dt, yp, n, d, ldx, mk, mp, 1, cl.ctypes.data, cl.size,
                                        m.ctypes.data, w.ctypes.data if w is not None else None, S.ctypes.data,
                                        counts.ctypes.data)
    assert rc == 0, native.last_error()
    return S, counts


def _reference(Xv, y, keep, classes, means, weights):
    """(sum w (x - m)(x - m)^T, sum w |x - m||x - m|^T, counts) in float64 over the kept rows"""
    Xk, yk = Xv[keep], y[keep]
    w = np.ones(len(classes)) if weights is None else weights
    d = Xv.shape[1]
    S, B = np.zeros((d, d)), np.zeros((d, d))
    for k, c in enumerate(np.asarray(classes, np.float32)):
        U = Xk[yk == c] - means[k]
        S += (w[k] * U).T @ U
        B += (w[k] * np.abs(U)).T @ np.abs(U)
    unmatched = np.sum(~np.isin(yk, np.asarray(classes, np.float32)))
    return S, B, [float(len(yk)), float(unmatched), float(np.sum(~np.isfinite(yk)))]


def _check(S, counts, want):
    Sw, B, c = want
    assert list(counts) == c, (counts, c)
    assert np.array_equal(S, S.T)
    err = np.abs(S - Sw)
    assert np.all(err <= PASS_TOL * B), float(np.max(err / np.maximum(B, 1e-300)))
    return float(np.max(err / np.maximum(B, 1e-300)))


def _rows(n, d, k, seed, kind):
    """stored rows (fp32 or bf16 bits) with 3 extra columns, their float64 values, labels of k classes (some of no
    class and some NaN), the classes and means near the class means"""
    rng = np.random.default_rng(seed)
    classes = np.sort(rng.choice(np.arange(-40, 40), size=k, replace=False)).astype(np.float32) * 0.5
    t = rng.integers(0, k, size=n)
    X = (rng.normal(size=(n, d + 3)) + 3.0 * rng.normal(size=(k, d + 3))[t] + 50.0).astype(np.float32)
    up = b2.native.to_bf16_bits(X) if kind == "bf16" else X
    Xv = b2.native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
    y = classes[t].copy()
    y[rng.uniform(size=n) < 0.02] = 1000.0           # no class
    y[rng.uniform(size=n) < 0.01] = np.nan
    return rng, up, Xv, y, classes, t


def _means(Xv, t, k, rng):
    return np.array([Xv[t == c].mean(axis=0) for c in range(k)]) + rng.normal(size=(k, Xv.shape[1])) * 1e-3


LAYOUT_D = [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128]


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", LAYOUT_D)
def test_pass_every_layout(ctx, kind, d):
    """K = 2, 3, 10, 32, weights none and random: counts exact, every entry within 1e-13 of sum w |u_i u_j|, the
    output bitwise symmetric, repeated calls bit-identical"""
    n = 4133                                         # ring tiles, then a partial tile on the direct kernel
    dt = b2.BF16 if kind == "bf16" else b2.F32
    es = 2 if kind == "bf16" else 4
    worst = 0.0
    for k in (2, 3, 10, 32):
        rng, up, Xv, y, classes, t = _rows(n, d, k, 100 * d + k + (kind == "bf16"), kind)
        mask = (np.arange(n) % 5 != 2).astype(np.uint8)
        cont = np.ascontiguousarray(up[:, :d])
        Xd, yd, md = ctx.to_device(cont, kind), ctx.to_device(y), ctx.to_device(mask)
        Xs = ctx.to_device(np.ascontiguousarray(up), kind)         # ldx = d + 3, starting one element in
        try:
            layouts = [("host", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, None, 0, None),
                       ("device", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, None, 0, None),
                       ("strided", Xs.ptr + es, yd.ptr, d + 3, native.MEM_DEVICE, None, 1, None),
                       ("device masked", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, md.ptr, 0, mask),
                       ("host masked", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, mask.ctypes.data, 0,
                        mask)]
            for name, xp, yp, ldx, mk, mp, c0, mref in layouts:
                keep = np.ones(n, bool) if mref is None else mref == 1
                Xref = Xv[:, c0:c0 + d]
                means = _means(Xref, t, k, rng)
                for weights in (None, rng.uniform(0.1, 3.0, size=k)):
                    S, counts = _raw(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means, weights)
                    S2, counts2 = _raw(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means, weights)
                    assert np.array_equal(S, S2) and np.array_equal(counts, counts2), name
                    worst = max(worst, _check(S, counts, _reference(Xref, y, keep, classes, means, weights)))
        finally:
            for a in (Xd, yd, md, Xs):
                a.free()
    print(f"\n[class scatter {kind} d={d}] worst entry error / sum w|u_i u_j| {worst:.2e}")


def test_many_tiles_per_cta_and_host_blocks(ctx):
    """every CTA streams many ring tiles; host rows span three staging blocks of 262 144 rows, the last one partial,
    whose sums each add to the previous ones; repeats are bit-identical"""
    n, d, k = 2 * (1 << 18) + 32 * (9 * ctx.info()["sm_count"] + 5) + 17, 24, 10
    rng, up, Xv, y, classes, t = _rows(n, d, k, 7, "f32")
    Xc = np.ascontiguousarray(up[:, :d])
    means = _means(Xv[:, :d], t, k, rng)
    weights = rng.uniform(0.5, 2.0, size=k)
    want = _reference(Xv[:, :d], y, np.ones(n, bool), classes, means, weights)
    Xd, yd = ctx.to_device(Xc), ctx.to_device(y)
    try:
        for xp, yp, mk in ((Xd.ptr, yd.ptr, native.MEM_DEVICE), (Xc.ctypes.data, y.ctypes.data, native.MEM_HOST)):
            S, counts = _raw(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, means, weights)
            S2, counts2 = _raw(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, means, weights)
            assert np.array_equal(S, S2) and np.array_equal(counts, counts2)
            _check(S, counts, want)
    finally:
        Xd.free()
        yd.free()


def test_zero_rows_and_abi_refusals(ctx):
    lib = native.load()
    n, d, k = 64, 4, 3
    X = np.zeros((n, d), np.float32)
    y = np.zeros(n, np.float32)
    cl = np.array([0, 1, 2], np.float32)
    m = np.zeros((k, d))
    w = np.ones(k)
    S, counts = np.full((d, d), np.nan), np.full(3, np.nan)

    def call(X=X.ctypes.data, y=y.ctypes.data, n=n, cl=cl.ctypes.data, k=k, m=m.ctypes.data, w=None,
             S=S.ctypes.data, c=counts.ctypes.data):
        return lib.b2_class_scatter(ctx._h, X, b2.F32, y, n, d, d, native.MEM_HOST, None, 1, cl, k, m, w, S, c)
    assert call(X=None, y=None, n=0) == 0
    assert not np.any(S) and not np.any(counts)
    assert call(k=1) == E_ARG and call(k=33) == E_ARG
    bad = np.array([0, 2, 1], np.float32)
    assert call(cl=bad.ctypes.data) == E_ARG
    nan_cl = np.array([0, 1, np.nan], np.float32)
    assert call(cl=nan_cl.ctypes.data) == E_ARG
    assert call(m=None) == E_ARG and call(S=None) == E_ARG and call(c=None) == E_ARG
    mn = m.copy()
    mn[1, 2] = np.inf
    assert call(m=mn.ctypes.data) == E_ARG
    for bw in (np.array([1.0, -0.5, 1.0]), np.array([1.0, np.nan, 1.0])):
        assert call(w=bw.ctypes.data) == E_ARG
    assert call(w=w.ctypes.data) == 0
    assert call(X=None) == E_ARG
    sums = ctx.class_scatter(X, y, cl, m, row_mask=np.zeros(n, np.uint8))
    assert sums["kept"] == 0 and not np.any(sums["scatter"])


def _fit_pair(X, y, **kw):
    ctx_kw = kw.pop("ctx")
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours = b2.B200LinearDiscriminantAnalysis(ctx=ctx_kw, **kw).fit(X, y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref = LinearDiscriminantAnalysis(**kw).fit(X.astype(np.float32).astype(np.float64), y)
    assert [str(w.message) for w in w_ours] == [str(w.message) for w in w_ref]
    return ours, ref


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - b)) / max(np.max(np.abs(b)), 1e-300))


@pytest.mark.parametrize("k", [2, 3, 10, 32])
def test_estimator_matches_sklearn(ctx, k):
    rng = np.random.default_rng(k)
    n, d = 16384, 24
    t = rng.integers(0, k, size=n)
    t[:k] = np.arange(k)
    A = rng.normal(size=(d, d)) / np.sqrt(d)
    X = rng.normal(size=(k, d))[t] * 1.5 + rng.normal(size=(n, d)) @ A + 0.3 * rng.normal(size=(n, d)) + 100.0
    X64 = X.astype(np.float32).astype(np.float64)
    p = rng.uniform(0.5, 2.0, size=k)
    worst = 0.0
    for kw in (dict(solver="svd"), dict(solver="svd", priors=p, store_covariance=True), dict(solver="lsqr"),
               dict(solver="lsqr", shrinkage=0.3, priors=p / p.sum()), dict(solver="eigen"),
               dict(solver="eigen", shrinkage=0.1, priors=p)):
        ours, ref = _fit_pair(X, t, ctx=ctx, **kw)
        scale = max(np.max(np.abs(ref.coef_)), np.max(np.abs(ref.intercept_)))
        err = max(np.max(np.abs(ours.coef_ - ref.coef_)), np.max(np.abs(ours.intercept_ - ref.intercept_))) / scale
        for name in ("means_", "priors_", "xbar_", "covariance_", "explained_variance_ratio_"):
            assert hasattr(ours, name) == hasattr(ref, name), name
            if hasattr(ref, name):
                err = max(err, _rel(getattr(ours, name), getattr(ref, name)))
        assert err <= 1e-10, (kw, err)
        worst = max(worst, err)
        assert np.array_equal(ours.predict(X), ref.predict(X64))
        assert np.max(np.abs(ours.predict_proba(X) - ref.predict_proba(X64))) <= 1e-9
        if ref.solver != "lsqr":
            T, Tr = ours.transform(X), ref.transform(X64)
            s = np.sign(np.sum(T * Tr, axis=0))
            bound = np.abs(X64) @ np.abs(ref.scalings_[:, : Tr.shape[1]])
            assert np.max(np.abs(T * s - Tr) / bound) <= 1e-10
    print(f"\n[LDA k={k}] worst relative difference {worst:.2e}")


def test_large_fit_from_device_rows_and_labels(ctx):
    n, d, k = 1_000_000, 128, 10
    rng = np.random.default_rng(6)
    t = rng.integers(0, k, size=n)
    X = (rng.normal(size=(k, d))[t] * 0.5 + rng.normal(size=(n, d)) + 10.0).astype(np.float32)
    labels = (np.arange(k, dtype=np.float32) * 3.0 - 7.0)
    y = labels[t]
    Xd, yd = ctx.to_device(X), ctx.to_device(y)
    X64 = X.astype(np.float64)
    try:
        ours = b2.B200LinearDiscriminantAnalysis(ctx=ctx).fit(Xd, yd)
        assert np.array_equal(ours.classes_, labels) and ours.classes_.dtype == np.float32
        ref = LinearDiscriminantAnalysis().fit(X64, y)
        err = _rel(ours.coef_, ref.coef_)
        print(f"\n[LDA 1M x 128 device, 10 classes] coef_ {err:.2e}")
        assert err <= 1e-9
        lab = ours.predict(Xd)
        assert np.array_equal(lab.to_host(), ref.predict(X64))
        lab.free()
        pd = ours.predict_proba(Xd)             # the device softmax sums in column order, numpy pairwise
        assert np.max(np.abs(pd.to_host() - ours.predict_proba(X))) <= 1e-15
        pd.free()
        Td = ours.transform(Xd)
        T, Tr = Td.to_host(), ref.transform(X64)
        Td.free()
        s = np.sign(np.sum(T * Tr, axis=0))
        bound = np.abs(X64) @ np.abs(ref.scalings_[:, : Tr.shape[1]])
        assert np.max(np.abs(T * s - Tr) / bound) <= 1e-9
    finally:
        Xd.free()
        yd.free()
