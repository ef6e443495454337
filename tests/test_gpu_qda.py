"""QuadraticDiscriminantAnalysis on the H100: b2_class_scatters and b2_qda_decision against float64 numpy statements of
the passes on the same stored rows, on every row layout, with balanced and skewed labels, many gathers per work item,
host rows over several staging blocks and a call longer than one index span; the ABI refusals; the estimator against
scikit-learn on float64 copies of the staged rows; a 1 M x 128 fit from device rows and device labels."""
import warnings

import numpy as np
import pytest
from sklearn.discriminant_analysis import QuadraticDiscriminantAnalysis

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native

pytestmark = pytest.mark.gpu

E_ARG = -1
PASS_TOL = 1e-13
LAYOUT_D = [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128]


def _scatters(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means):
    cl = np.ascontiguousarray(classes, dtype=np.float32)
    m = np.ascontiguousarray(means, dtype=np.float64)
    S = np.full((cl.size, d, d), np.nan)
    nk, counts = np.full(cl.size, np.nan), np.full(3, np.nan)
    rc = native.load().b2_class_scatters(ctx._h, xp, dt, yp, n, d, ldx, mk, mp, 1, cl.ctypes.data, cl.size,
                                         m.ctypes.data, S.ctypes.data, nk.ctypes.data, counts.ctypes.data)
    assert rc == 0, native.last_error()
    return S, nk, counts


def _scatters_reference(Xv, y, keep, classes, means):
    """per class (sum (x - m)(x - m)^T, sum |x - m||x - m|^T, rows) in float64 over the kept rows, and the counts"""
    Xk, yk = Xv[keep], y[keep]
    d = Xv.shape[1]
    S, B, nk = np.zeros((len(classes), d, d)), np.zeros((len(classes), d, d)), np.zeros(len(classes))
    for k, c in enumerate(np.asarray(classes, np.float32)):
        U = Xk[yk == c] - means[k]
        S[k], B[k], nk[k] = U.T @ U, np.abs(U).T @ np.abs(U), len(U)
    unmatched = np.sum(~np.isin(yk, np.asarray(classes, np.float32)))
    return S, B, nk, [float(len(yk)), float(unmatched), float(np.sum(~np.isfinite(yk)))]


def _check_scatters(got, want):
    S, nk, counts = got
    Sw, B, nkw, c = want
    assert list(counts) == c, (counts, c)
    assert np.array_equal(nk, nkw), (nk, nkw)
    assert np.array_equal(S, np.transpose(S, (0, 2, 1)))
    err = np.abs(S - Sw)
    assert np.all(err <= PASS_TOL * B), float(np.max(err / np.maximum(B, 1e-300)))
    return float(np.max(err / np.maximum(B, 1e-300), initial=0.0))


def _labels(n, k, rng, skewed):
    """class indices: balanced, or skewed (class 0 95 %, classes 1 and 2 of two rows, class k - 1 without rows)"""
    if not skewed:
        return rng.integers(0, k, size=n)
    t = np.zeros(n, np.int64)
    rest = rng.permutation(n)[: n // 20]
    t[rest] = rng.integers(1, max(k - 1, 2), size=rest.size) if k > 2 else 1
    if k > 3:
        t[t == 1], t[t == 2] = 3 % (k - 1), 3 % (k - 1)
        two = rng.permutation(np.flatnonzero(t == 0))[:4]
        t[two[:2]], t[two[2:]] = 1, 2
    return t


def _rows(n, d, k, seed, kind, skewed=False):
    """stored rows (fp32 or bf16 bits) with 3 extra columns, their float64 values, labels of k classes (some of no
    class and some NaN), the classes and class indices"""
    rng = np.random.default_rng(seed)
    classes = np.sort(rng.choice(np.arange(-40, 40), size=k, replace=False)).astype(np.float32) * 0.5
    t = _labels(n, k, rng, skewed)
    X = (rng.normal(size=(n, d + 3)) * rng.uniform(0.5, 2.0, size=k)[t, None] + 3.0 * rng.normal(size=(k, d + 3))[t]
         + 50.0).astype(np.float32)
    up = b2.native.to_bf16_bits(X) if kind == "bf16" else X
    Xv = b2.native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
    y = classes[t].copy()
    y[rng.uniform(size=n) < 0.02] = 1000.0           # no class
    y[rng.uniform(size=n) < 0.01] = np.nan
    return rng, up, Xv, y, classes, t


def _means(Xv, t, k, rng):
    return np.array([Xv[t == c].mean(axis=0) if np.any(t == c) else Xv[0] for c in range(k)]) + \
        rng.normal(size=(k, Xv.shape[1])) * 1e-3


def _layouts(ctx, up, y, mask, d, kind):
    """(name, X, y, ldx, mem_kind, mask pointer, first column, mask for the reference) of every layout, and the buffers"""
    es = 2 if kind == "bf16" else 4
    cont = np.ascontiguousarray(up[:, :d])
    Xd, yd, md = ctx.to_device(cont, kind), ctx.to_device(y), ctx.to_device(mask)
    Xs = ctx.to_device(np.ascontiguousarray(up), kind)         # ldx = d + 3, starting one element in
    return [("host", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, None, 0, None),
            ("device", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, None, 0, None),
            ("strided", Xs.ptr + es, yd.ptr, d + 3, native.MEM_DEVICE, None, 1, None),
            ("device masked", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, md.ptr, 0, mask),
            ("host masked", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, mask.ctypes.data, 0, mask)], \
        (Xd, yd, md, Xs, cont)


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", LAYOUT_D)
def test_scatters_every_layout(ctx, kind, d):
    """K = 2, 3, 10, 32, balanced and skewed labels: counts exact, every entry within 1e-13 of sum |u_i u_j| over the
    class, each output bitwise symmetric, repeated calls bit-identical"""
    n = 4133
    dt = b2.BF16 if kind == "bf16" else b2.F32
    worst = 0.0
    for k in (2, 3, 10, 32):
        for skewed in (False, True):
            rng, up, Xv, y, classes, t = _rows(n, d, k, 100 * d + k + (kind == "bf16") + 7 * skewed, kind, skewed)
            mask = (np.arange(n) % 5 != 2).astype(np.uint8)
            layouts, bufs = _layouts(ctx, up, y, mask, d, kind)
            try:
                for name, xp, yp, ldx, mk, mp, c0, mref in layouts:
                    keep = np.ones(n, bool) if mref is None else mref == 1
                    Xref = Xv[:, c0:c0 + d]
                    means = _means(Xref, t, k, rng)
                    got = _scatters(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means)
                    again = _scatters(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means)
                    assert all(np.array_equal(a, b) for a, b in zip(got, again)), name
                    worst = max(worst, _check_scatters(got, _scatters_reference(Xref, y, keep, classes, means)))
            finally:
                for a in bufs[:4]:
                    a.free()
    print(f"\n[class scatters {kind} d={d}] worst entry error / sum |u_i u_j| {worst:.2e}")


def test_scatters_many_gathers_and_host_blocks(ctx):
    """each work item gathers many 32-row groups; host rows span three staging blocks of 262 144 rows, the last one
    partial, whose sums each add to the previous ones; repeats are bit-identical"""
    n, d, k = 2 * (1 << 18) + 32 * (9 * ctx.info()["sm_count"] + 5) + 17, 24, 10
    for skewed in (False, True):
        rng, up, Xv, y, classes, t = _rows(n, d, k, 7 + skewed, "f32", skewed)
        Xc = np.ascontiguousarray(up[:, :d])
        means = _means(Xv[:, :d], t, k, rng)
        want = _scatters_reference(Xv[:, :d], y, np.ones(n, bool), classes, means)
        Xd, yd = ctx.to_device(Xc), ctx.to_device(y)
        try:
            for xp, yp, mk in ((Xd.ptr, yd.ptr, native.MEM_DEVICE), (Xc.ctypes.data, y.ctypes.data, native.MEM_HOST)):
                got = _scatters(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, means)
                again = _scatters(ctx, xp, b2.F32, yp, n, d, d, mk, None, classes, means)
                assert all(np.array_equal(a, b) for a, b in zip(got, again))
                _check_scatters(got, want)
        finally:
            Xd.free()
            yd.free()


def test_scatters_longer_than_one_span(ctx):
    """device rows beyond one span of 2^24 row indices: the second span's sums add to the first's"""
    n, d, k = (1 << 24) + 3 * 8192 + 5, 2, 3
    rng = np.random.default_rng(3)
    t = rng.integers(0, k, size=n)
    X = (rng.normal(size=(n, d)) + np.array([[0.0, 1.0], [5.0, -2.0], [-3.0, 4.0]])[t] + 20.0).astype(np.float32)
    classes = np.array([1.0, 2.0, 3.0], np.float32)
    y = classes[t]
    y[n - 3] = np.nan
    Xv = X.astype(np.float64)
    means = np.array([Xv[t == c].mean(axis=0) for c in range(k)])
    Xd, yd = ctx.to_device(X), ctx.to_device(y)
    try:
        got = _scatters(ctx, Xd.ptr, b2.F32, yd.ptr, n, d, d, native.MEM_DEVICE, None, classes, means)
    finally:
        Xd.free()
        yd.free()
    _check_scatters(got, _scatters_reference(Xv, y, np.ones(n, bool), classes, means))


def _decision(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means, W, c, diff=False):
    """the decisions, labels, d_1 - d_0 (or None) and counts as host arrays; the outputs live where the rows do"""
    cl = np.ascontiguousarray(classes, dtype=np.float32)
    k = cl.size
    m, Wc, cc = (np.ascontiguousarray(a, dtype=np.float64) for a in (means, W, c))
    outs = [ctx._out(mk, shape, kind) for shape, kind in (((n, k), "f64"), ((n,), "f32"), ((n,), "f64"))]
    counts = np.full(2, np.nan)
    rc = native.load().b2_qda_decision(ctx._h, xp, dt, yp, n, d, ldx, mk, mp, 1, cl.ctypes.data, k, m.ctypes.data,
                                       Wc.ctypes.data, cc.ctypes.data, outs[0][1], outs[1][1],
                                       outs[2][1] if diff else None, counts.ctypes.data)
    assert rc == 0, native.last_error()
    host = []
    for a, _ in outs:
        if isinstance(a, native.DeviceArray):
            h = a.to_host()
            a.free()
            a = h
        host.append(a)
    return host[0], host[1], host[2] if diff else None, counts


def _decision_operands(rng, Xv, t, k, d):
    means = _means(Xv, t, k, rng)
    W = rng.normal(size=(k, d, d)) / np.sqrt(d) * rng.uniform(0.5, 2.0, size=(k, 1, 1))
    c = rng.normal(size=k) * 10.0
    return means, W, c


def _decision_reference(Xv, means, W, c):
    """(decisions, bound): d_k = -1/2 |(x - m_k) W_k|^2 + c_k and 1/2 sum_l (sum_j |u_j W_jl|)^2 + |c_k| in float64"""
    dec = np.stack([-0.5 * np.sum(((Xv - m) @ Wk) ** 2, axis=1) + ck for m, Wk, ck in zip(means, W, c)], axis=1)
    bound = np.stack([0.5 * np.sum((np.abs(Xv - m) @ np.abs(Wk)) ** 2, axis=1) + abs(ck)
                      for m, Wk, ck in zip(means, W, c)], axis=1)
    return dec, bound


def _check_decision(got, want, classes, y, keep):
    dec, lab, dif, counts = got
    ref, bound = want
    err = np.abs(dec - ref)
    assert np.all(err <= PASS_TOL * bound), float(np.max(err / bound))
    top2 = np.sort(ref, axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * PASS_TOL * bound.max(axis=1)
    assert np.array_equal(lab[clear], np.asarray(classes, np.float32)[np.argmax(ref, axis=1)][clear])
    assert np.array_equal(lab, np.asarray(classes, np.float32)[np.argmax(dec, axis=1)])   # the first largest
    assert counts[0] == keep.sum() and counts[1] == np.sum(keep & (y == lab))
    if dif is not None:
        assert np.array_equal(dif, dec[:, 1] - dec[:, 0])
    return float(np.max(err / bound))


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", LAYOUT_D)
def test_decision_every_layout(ctx, kind, d):
    """K = 2, 3, 10, 32 on every layout (the contiguous ones on the ring flavour, then the direct one for the partial
    tile): every entry within 1e-13 of 1/2 sum_l (sum_j |u_j W_jl|)^2 + |c_k|, labels of the first largest, counts
    exact, d_1 - d_0 for two classes, repeats bit-identical"""
    n = 4133
    dt = b2.BF16 if kind == "bf16" else b2.F32
    worst = 0.0
    for k in (2, 3, 10, 32):
        rng, up, Xv, y, classes, t = _rows(n, d, k, 300 * d + k + (kind == "bf16"), kind)
        mask = (np.arange(n) % 5 != 2).astype(np.uint8)
        layouts, bufs = _layouts(ctx, up, y, mask, d, kind)
        try:
            for name, xp, yp, ldx, mk, mp, c0, mref in layouts:
                keep = np.ones(n, bool) if mref is None else mref == 1
                Xref = Xv[:, c0:c0 + d]
                means, W, c = _decision_operands(rng, Xref, t, k, d)
                got = _decision(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means, W, c, diff=k == 2)
                again = _decision(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, means, W, c, diff=k == 2)
                assert all(np.array_equal(a, b) for a, b in zip(got, again) if a is not None), name
                worst = max(worst, _check_decision(got, _decision_reference(Xref, means, W, c), classes, y, keep))
        finally:
            for a in bufs[:4]:
                a.free()
    print(f"\n[qda decision {kind} d={d}] worst entry error / bound {worst:.2e}")


def test_decision_many_tiles_and_host_blocks(ctx):
    """every CTA streams many tiles; host rows over three staging blocks; labels and counts without the decisions
    (through the context's scratch) equal those with them"""
    n, d, k = 2 * (1 << 18) + 32 * (9 * ctx.info()["sm_count"] + 5) + 17, 24, 10
    rng, up, Xv, y, classes, t = _rows(n, d, k, 11, "f32")
    Xc = np.ascontiguousarray(up[:, :d])
    means, W, c = _decision_operands(rng, Xv[:, :d], t, k, d)
    want = _decision_reference(Xv[:, :d], means, W, c)
    Xd, yd = ctx.to_device(Xc), ctx.to_device(y)
    try:
        for X in (Xd, Xc):
            yy = yd if X is Xd else y
            got = ctx.qda_decision(X, means, W, c, classes, yy, decision=True, label=True)
            dec = got["decision"].to_host() if X is Xd else got["decision"]
            lab = got["label"].to_host() if X is Xd else got["label"]
            _check_decision((dec, lab, None, np.array([got["kept"], got["correct"]])), want, classes, y,
                            np.ones(n, bool))
            only = ctx.qda_decision(X, means, W, c, classes, yy, label=True)
            lab2 = only["label"].to_host() if X is Xd else only["label"]
            assert np.array_equal(lab2, lab) and (only["kept"], only["correct"]) == (got["kept"], got["correct"])
            for a in list(got.values()) + list(only.values()):
                if isinstance(a, native.DeviceArray):
                    a.free()
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
    S, nk, counts = np.full((k, d, d), np.nan), np.full(k, np.nan), np.full(3, np.nan)

    def scat(X=X.ctypes.data, y=y.ctypes.data, n=n, cl=cl.ctypes.data, k=k, m=m.ctypes.data, S=S.ctypes.data,
             nk=nk.ctypes.data, c=counts.ctypes.data):
        return lib.b2_class_scatters(ctx._h, X, b2.F32, y, n, d, d, native.MEM_HOST, None, 1, cl, k, m, S, nk, c)
    assert scat(X=None, y=None, n=0) == 0
    assert not np.any(S) and not np.any(nk) and not np.any(counts)
    assert scat(k=1) == E_ARG and scat(k=33) == E_ARG
    bad = np.array([0, 2, 1], np.float32)
    nan_cl = np.array([0, 1, np.nan], np.float32)
    assert scat(cl=bad.ctypes.data) == E_ARG and scat(cl=nan_cl.ctypes.data) == E_ARG
    assert scat(m=None) == E_ARG and scat(S=None) == E_ARG and scat(nk=None) == E_ARG and scat(c=None) == E_ARG
    mn = m.copy()
    mn[1, 2] = np.inf
    assert scat(m=mn.ctypes.data) == E_ARG
    assert scat(X=None) == E_ARG and scat(y=None) == E_ARG
    assert scat() == 0 and nk[0] == n and not np.any(S)
    sums = ctx.class_scatters(X, y, cl, m, row_mask=np.zeros(n, np.uint8))
    assert sums["kept"] == 0 and not np.any(sums["scatters"]) and not np.any(sums["class_counts"])

    W, c = np.ones((k, d, d)), np.zeros(k)
    dec, lab, dif, cnt = np.empty((n, k)), np.empty(n, np.float32), np.empty(n), np.empty(2)

    def qd(X=X.ctypes.data, y=y.ctypes.data, n=n, cl=cl.ctypes.data, k=k, m=m.ctypes.data, W=W.ctypes.data,
           c=c.ctypes.data, dec=dec.ctypes.data, lab=lab.ctypes.data, dif=None, cnt=cnt.ctypes.data):
        return lib.b2_qda_decision(ctx._h, X, b2.F32, y, n, d, d, native.MEM_HOST, None, 1, cl, k, m, W, c, dec, lab,
                                   dif, cnt)
    assert qd() == 0 and qd(X=None, y=None, n=0) == 0
    assert qd(k=1) == E_ARG and qd(k=33) == E_ARG and qd(cl=bad.ctypes.data) == E_ARG
    assert qd(cl=nan_cl.ctypes.data) == E_ARG
    assert qd(m=None) == E_ARG and qd(W=None) == E_ARG and qd(c=None) == E_ARG
    assert qd(dec=None, lab=None, cnt=None) == E_ARG
    assert qd(y=None) == E_ARG and qd(X=None) == E_ARG
    assert qd(dif=dif.ctypes.data) == E_ARG                          # d_1 - d_0 needs two classes
    for a, name in ((m, "m"), (W, "W"), (c, "c")):
        bad_a = a.copy()
        bad_a.flat[1] = np.nan
        assert qd(**{name: bad_a.ctypes.data}) == E_ARG


def _fit_pair(X, y, ctx, **kw):
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours = b2.B200QuadraticDiscriminantAnalysis(ctx=ctx, **kw).fit(X, y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref = QuadraticDiscriminantAnalysis(**kw).fit(X.astype(np.float32).astype(np.float64), y)
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
    X = np.empty((n, d))
    for c in range(k):
        Q, _ = np.linalg.qr(rng.normal(size=(d, d)))
        X[t == c] = rng.normal(size=d) * 2 + (rng.normal(size=((t == c).sum(), d)) * np.geomspace(0.3, 3, d)) @ Q.T
    X += 100.0
    X64 = X.astype(np.float32).astype(np.float64)
    worst = 0.0
    for kw in (dict(solver="svd"), dict(solver="svd", reg_param=0.1, store_covariance=True),
               dict(solver="eigen"), dict(solver="eigen", shrinkage=0.2, priors=np.full(k, 1.0 / k),
                                          store_covariance=True)):
        ours, ref = _fit_pair(X, t, ctx, **kw)
        err = max(_rel(ours.means_, ref.means_), _rel(ours.priors_, ref.priors_))
        for j in range(k):
            err = max(err, _rel(ours.scalings_[j], ref.scalings_[j]))
            s = np.sign(np.sum(ours.rotations_[j] * ref.rotations_[j], axis=0))
            err = max(err, _rel(ours.rotations_[j] * s, ref.rotations_[j]))
            if hasattr(ref, "covariance_"):
                err = max(err, _rel(ours.covariance_[j], ref.covariance_[j]))
        err = max(err, _rel(ours.decision_function(X), ref.decision_function(X64)))
        assert err <= 1e-10, (kw, err)
        worst = max(worst, err)
        assert np.array_equal(ours.predict(X), ref.predict(X64))
        assert np.max(np.abs(ours.predict_proba(X) - ref.predict_proba(X64))) <= 1e-9
        assert ours.score(X, ref.predict(X64)) == 1.0
    print(f"\n[QDA k={k}] worst relative difference {worst:.2e}")


def test_large_fit_from_device_rows_and_labels(ctx):
    n, d, k = 1_000_000, 128, 10
    rng = np.random.default_rng(6)
    t = rng.integers(0, k, size=n)
    X = (rng.normal(size=(k, d))[t] * 0.5 + rng.normal(size=(n, d)) * rng.uniform(0.5, 2.0, size=k)[t, None]
         + 10.0).astype(np.float32)
    labels = (np.arange(k, dtype=np.float32) * 3.0 - 7.0)
    y = labels[t]
    Xd, yd = ctx.to_device(X), ctx.to_device(y)
    try:
        ours = b2.B200QuadraticDiscriminantAnalysis(ctx=ctx, reg_param=0.01).fit(Xd, yd)
        host = b2.B200QuadraticDiscriminantAnalysis(ctx=ctx, reg_param=0.01).fit(X, y)
        assert np.array_equal(ours.classes_, labels) and ours.classes_.dtype == np.float32
        err = max(_rel(ours.means_, host.means_), _rel(ours.priors_, host.priors_))
        for j in range(k):
            err = max(err, _rel(ours.scalings_[j], host.scalings_[j]))
            s = np.sign(np.sum(ours.rotations_[j] * host.rotations_[j], axis=0))
            err = max(err, _rel(ours.rotations_[j] * s, host.rotations_[j]))
        print(f"\n[QDA 1M x 128 device vs host, 10 classes] attributes {err:.2e}")
        assert err <= 1e-10
        lab = ours.predict(Xd)
        assert np.array_equal(lab.to_host(), host.predict(X))
        lab.free()
        pd = ours.predict_proba(Xd)             # the device softmax against scikit-learn's formula
        assert np.max(np.abs(pd.to_host() - host.predict_proba(X))) <= 1e-12
        pd.free()
        assert ours.score(Xd, yd) == host.score(X, y)
    finally:
        Xd.free()
        yd.free()
