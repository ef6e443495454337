"""RidgeClassifier on the H100: b2_class_sums against math.fsum on every row layout, b2_solve_classes against
scipy.linalg.solve on designed statistics, b2_classify against an extended-precision dot product, b2_label_values against
np.unique, and the estimator against scikit-learn's RidgeClassifier on float64 copies of the rows.  Each test prints the
worst case it measured (run with -s).

Bounds:
  * class sums: per entry within 1e-13 of the sum of |x - c| over the class (the fsum of the same fp64 differences),
    counts equal, repeated calls bit-identical;
  * the solve: 1e-11 relative to the largest coefficient (scipy's Cholesky rounds differently);
  * decisions: 1e-14 relative to sum_j |x_j w_j| + |b| per entry; labels equal wherever the two largest decisions differ
    by more than 1e-9; counts equal to the returned labels' matches;
  * the estimator: coefficients within 1e-10 relative and equal predict on the exact fp64 Gram (KERNEL_SIMT); within
    test_gpu_parity.COEF_TOL relative and predict agreement >= 0.999 on the default (tensor-core) Gram.
"""
import io
import math

import joblib
import numpy as np
import pytest
import scipy.linalg
from sklearn import linear_model

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from test_gpu_parity import COEF_TOL

pytestmark = pytest.mark.gpu

SUM_TOL = 1e-13
SOLVE_TOL = 1e-11
DEC_TOL = 1e-14
SIMT_TOL = 1e-10


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _rows(n, d, seed, kind, offset=0.0):
    """(stored rows with 3 spare columns, their float64 values)"""
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d + 3)) + offset).astype(np.float32)
    up = b2.native.to_bf16_bits(X) if kind == "bf16" else X
    Xv = b2.native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
    return up, Xv


def _layouts(ctx, up, d, kind, y, mask):
    """(name, X ptr, y ptr, ldx, mem_kind, mask ptr, which columns of the spare-padded rows, mask or None), the device
    buffers to free"""
    es = 2 if kind == "bf16" else 4
    cont = np.ascontiguousarray(up[:, :d])
    Xd, yd, md = ctx.to_device(cont, kind), ctx.to_device(y), ctx.to_device(mask)
    Xs = ctx.to_device(np.ascontiguousarray(up), kind)          # ldx = d + 3, starting one element in
    return [("host", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, None, 0, None),
            ("device", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, None, 0, None),
            ("strided", Xs.ptr + es, yd.ptr, d + 3, native.MEM_DEVICE, None, 1, None),
            ("device masked", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, md.ptr, 0, mask),
            ("host masked", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, mask.ctypes.data, 0, mask)], \
        (Xd, yd, md, Xs), cont


def _raw_class_sums(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, center):
    sums, counts = np.empty((classes.size, d + 1)), np.empty(3)
    rc = native.load().b2_class_sums(ctx._h, xp, dt, yp, n, d, ldx, mk, mp, 1, classes.ctypes.data, classes.size,
                                     center.ctypes.data, sums.ctypes.data, counts.ctypes.data)
    assert rc == 0, native.last_error()
    return sums, counts


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128])
def test_class_sums_every_layout(ctx, kind, d):
    n = 4133                                          # ring tiles, then a partial tile on the direct kernel
    up, Xv = _rows(n, d, 40 + d, kind, offset=1e4 if d % 2 else 0.0)
    dt = b2.BF16 if kind == "bf16" else b2.F32
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    rng = np.random.default_rng(d)
    worst = 0.0
    for k in (2, 3, 32):
        classes = np.sort(rng.choice(np.arange(-40, 40), size=k, replace=False)).astype(np.float32)
        y = classes[rng.integers(0, k, size=n)]
        y[[5, 6]] = 99.0                              # no class
        y[7], y[8] = np.nan, -np.inf
        layouts, owned, _ = _layouts(ctx, up, d, kind, y, mask)
        try:
            for name, xp, yp, ldx, mk, mp, c0, mref in layouts:
                Xr = Xv[:, c0:c0 + d]
                keep = np.ones(n, bool) if mref is None else mref == 1
                center = Xr[keep].mean(axis=0)
                sums, counts = _raw_class_sums(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, center)
                again, counts2 = _raw_class_sums(ctx, xp, dt, yp, n, d, ldx, mk, mp, classes, center)
                assert np.array_equal(sums, again) and np.array_equal(counts, counts2), name
                yk = y[keep]
                assert counts.tolist() == [keep.sum(), np.sum(~np.isin(yk, classes)), np.sum(~np.isfinite(yk))], name
                for c in range(k):
                    V = Xr[keep & (y == classes[c])] - center
                    assert sums[c, d] == len(V), name
                    for j in range(d):
                        scale = max(math.fsum(np.abs(V[:, j])), 1e-300)
                        err = abs(sums[c, j] - math.fsum(V[:, j])) / scale
                        assert err < SUM_TOL, (name, k, c, j, err)
                        worst = max(worst, err)
        finally:
            for a in owned:
                a.free()
    print(f"\n[class sums {kind} d={d}] worst {worst:.2e}")


def _designed(d, k, seed, fit_intercept, alpha):
    """(S, class sums (k, d + 1), the scipy solution W (T, d), b (T,)) of random rows and labels"""
    rng = np.random.default_rng(seed)
    n = 4 * d + 50 * k
    X = rng.normal(size=(n, d)) * rng.uniform(0.5, 2.0, size=d) + rng.normal(size=d)
    t = rng.integers(0, k, size=n)
    t[:k] = np.arange(k)
    Z = np.c_[X, np.ones(n), t]
    S = Z.T @ Z
    m = X.mean(axis=0) if fit_intercept else np.zeros(d)
    sums = np.array([np.r_[(X[t == c] - m).sum(axis=0), np.sum(t == c)] for c in range(k)])
    Y = np.where(t[:, None] == np.arange(k)[None, :], 1.0, -1.0)[:, [1] if k == 2 else slice(None)]
    Xc, Yc = (X - m, Y - Y.mean(axis=0)) if fit_intercept else (X, Y)
    W = scipy.linalg.solve(Xc.T @ Xc + alpha * np.eye(d), Xc.T @ Yc, assume_a="pos").T
    b = (Y.mean(axis=0) - m @ W.T) if fit_intercept else np.zeros(W.shape[0])
    return S, sums, W, b


@pytest.mark.parametrize("d", [1, 7, 33, 128])
@pytest.mark.parametrize("k", [2, 3, 32])
def test_solve_classes_designed(ctx, d, k):
    worst = 0.0
    for fit_intercept in (True, False):
        for alpha in (0.0, 1.0):
            S, sums, W, b = _designed(d, k, 100 * d + k, fit_intercept, alpha)
            ctx.gram_import(S)
            coef, b0 = ctx.solve_classes(sums, alpha, fit_intercept)
            assert coef.shape == W.shape and b0.shape == b.shape
            err = rel(np.c_[coef, b0], np.c_[W, b])
            assert err < SOLVE_TOL, (fit_intercept, alpha, err)
            again = ctx.solve_classes(None, alpha, fit_intercept, n_classes=k)
            assert np.array_equal(again[0], coef) and np.array_equal(again[1], b0)
            worst = max(worst, err)
    print(f"\n[solve classes d={d} k={k}] worst {worst:.2e}")


def test_solve_classes_refuses_a_singular_system(ctx):
    rng = np.random.default_rng(3)
    X = rng.normal(size=(500, 6))
    X[:, 5] = X[:, 2]
    t = rng.integers(0, 4, size=500)
    Z = np.c_[X, np.ones(500), t]
    ctx.gram_import(Z.T @ Z)
    sums = np.array([np.r_[(X[t == c] - X.mean(0)).sum(0), np.sum(t == c)] for c in range(4)])
    with pytest.raises(np.linalg.LinAlgError, match="not positive"):
        ctx.solve_classes(sums, 0.0, True)
    coef, _ = ctx.solve_classes(sums, 1e-3, True)
    assert np.all(np.isfinite(coef))


def _longdouble_decision(Xr, W, b):
    return np.asarray(Xr, np.longdouble) @ np.asarray(W, np.longdouble).T + np.asarray(b, np.longdouble)


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", [1, 9, 64, 128])
@pytest.mark.parametrize("t", [1, 3, 10, 32])
def test_classify_every_layout(ctx, kind, d, t):
    n = 4133
    up, Xv = _rows(n, d, 7 * d + t, kind)
    dt = b2.BF16 if kind == "bf16" else b2.F32
    rng = np.random.default_rng(t)
    W, b = rng.normal(size=(t, d)), rng.normal(size=t)
    k = max(t, 2)
    classes = np.sort(rng.choice(np.arange(-50, 50), size=k, replace=False)).astype(np.float32)
    y = classes[rng.integers(0, k, size=n)]
    y[3] = np.nan
    mask = (np.arange(n) % 7 != 3).astype(np.uint8)
    layouts, owned, _ = _layouts(ctx, up, d, kind, y, mask)
    lib, worst = native.load(), 0.0
    try:
        for name, xp, yp, ldx, mk, mp, c0, mref in layouts:
            Xr = Xv[:, c0:c0 + d]
            if mk == native.MEM_HOST:
                dec, lab = np.empty((n, t)), np.empty(n, np.float32)
                dp, lp = dec.ctypes.data, lab.ctypes.data
            else:
                dec_d, lab_d = ctx.empty((n, t), "f64"), ctx.empty((n,), "f32")
                dp, lp = dec_d.ptr, lab_d.ptr
            counts = np.empty(2)
            rc = lib.b2_classify(ctx._h, xp, dt, yp, n, d, ldx, mk, mp, 1, W.ctypes.data, b.ctypes.data, t,
                                 classes.ctypes.data, dp, lp, counts.ctypes.data)
            assert rc == 0, native.last_error()
            if mk == native.MEM_DEVICE:
                dec, lab = dec_d.to_host(), lab_d.to_host()
                dec_d.free(); lab_d.free()
            want = _longdouble_decision(Xr, W, b)
            scale = np.abs(Xr) @ np.abs(W).T + np.abs(b)
            err = float(np.max(np.abs(dec - want.astype(np.float64)) / scale))
            assert err < DEC_TOL, (name, err)
            worst = max(worst, err)
            want = want.astype(np.float64)
            ref = classes[(want[:, 0] > 0).astype(int)] if t == 1 else classes[np.argmax(want, axis=1)]
            srt = np.sort(np.c_[want, np.zeros(n)] if t == 1 else want, axis=1)
            clear = np.abs(srt[:, -1] - srt[:, -2]) > 1e-9
            assert np.array_equal(lab[clear], ref[clear]), name
            keep = np.ones(n, bool) if mref is None else mref == 1
            assert counts.tolist() == [keep.sum(), np.sum(keep & (y == lab))], name
    finally:
        for a in owned:
            a.free()
    print(f"\n[classify {kind} d={d} t={t}] worst {worst:.2e}")


def test_label_values_match_numpy(ctx):
    rng = np.random.default_rng(5)
    n = 300_001
    vals = np.array([-3.0, -0.0, 0.0, 2.0, 7.0, 1e6], np.float32)
    y = vals[rng.integers(0, vals.size, size=n)]
    y[[10, 20]] = np.nan
    mask = (rng.uniform(size=n) < 0.6).astype(np.uint8)
    y[np.flatnonzero(mask == 0)[:5]] = 123.0          # a value of the dropped rows only
    yd, md = ctx.to_device(y), ctx.to_device(mask)
    try:
        for row_mask, keep in ((None, 1), (md, 1), (md, 0)):
            yk = y if row_mask is None else y[mask == keep]
            want = np.unique(yk[np.isfinite(yk)] + np.float32(0))
            got, more = ctx.label_values(yd, row_mask, keep)
            assert not more and got.dtype == np.float32 and np.array_equal(got, want)
            zero = got[got == 0]
            assert zero.size == 1 and not np.signbit(zero[0])
            got2, more2 = ctx.label_values(yd, row_mask, keep, max_values=3)
            assert more2 and np.array_equal(got2, want[:3])
        many = rng.permutation(np.repeat(np.arange(40, dtype=np.float32) - 20, 100))
        md2 = ctx.to_device(many)
        try:
            got, more = ctx.label_values(md2)
            assert more and np.array_equal(got, np.arange(32, dtype=np.float32) - 20)
            got, more = ctx.label_values(md2, max_values=32)
            assert more and got.size == 32
        finally:
            md2.free()
        empty = ctx.to_device(np.array([np.nan, np.inf], np.float32))
        try:
            assert ctx.label_values(empty)[0].size == 0
        finally:
            empty.free()
    finally:
        yd.free(); md.free()


def _data(n, d, k, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) + offset).astype(np.float32).astype(np.float64)
    t = np.argmax((X - offset) @ rng.normal(size=(d, k)) + rng.normal(size=(n, k)), axis=1)
    t[:k] = np.arange(k)
    return X, t


def _flat(m):
    """[coef_ | intercept_] as a (T, d + 1) array"""
    W = np.atleast_2d(m.coef_)
    return np.c_[W, np.broadcast_to(np.ravel(m.intercept_), (W.shape[0],))]


@pytest.mark.parametrize("k", [2, 3, 10, 32])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_estimator_matches_sklearn(ctx, k, fit_intercept):
    X, t = _data(20_000, 24, k, seed=k, offset=3.0)
    labels = np.array([f"c{i:02d}" for i in range(k)])
    y = labels[t]
    ref = linear_model.RidgeClassifier(alpha=1.0, fit_intercept=fit_intercept).fit(X, y)
    ref_pred = ref.predict(X)
    worst = {}
    try:
        for kernel, tol in ((b2.KERNEL_SIMT, SIMT_TOL), (b2.KERNEL_AUTO, COEF_TOL)):
            ctx.set_kernel(kernel)
            ours = b2.B200RidgeClassifier(alpha=1.0, fit_intercept=fit_intercept, ctx=ctx).fit(X, y)
            assert ours.coef_.shape == ref.coef_.shape and np.shape(ours.intercept_) == np.shape(ref.intercept_)
            assert np.array_equal(ours.classes_, ref.classes_) and ours.solver_ == "cholesky"
            err = rel(_flat(ours), _flat(ref))
            assert err < tol, (kernel, err)
            pred = ours.predict(X)
            agree = float(np.mean(pred == ref_pred))
            if kernel == b2.KERNEL_SIMT:
                assert agree == 1.0
            else:
                assert agree >= 0.999, agree
            assert abs(ours.score(X, y) - ref.score(X, y)) <= 1.0 - agree + 1e-12
            assert rel(ours.decision_function(X), ref.decision_function(X)) < max(tol, 1e-12) * 10
            worst[kernel] = err
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
    buf = io.BytesIO()
    joblib.dump(ours.to_sklearn(), buf)
    reg = joblib.load(io.BytesIO(buf.getvalue()))
    assert np.array_equal(reg.predict(X), ours.predict(X))
    print(f"\n[ridge classifier k={k} intercept={fit_intercept}] simt {worst[b2.KERNEL_SIMT]:.2e} "
          f"auto {worst[b2.KERNEL_AUTO]:.2e}")


def test_masks_and_rank_deficient_fallback(ctx):
    X, t = _data(6000, 10, 4, seed=21)
    mask = (np.random.default_rng(2).uniform(size=6000) < 0.8).astype(np.uint8)
    try:
        ctx.set_kernel(b2.KERNEL_SIMT)
        ours = b2.B200RidgeClassifier(alpha=0.5, ctx=ctx).fit(X, t, row_mask=mask, mask_keep=1)
        ref = linear_model.RidgeClassifier(alpha=0.5).fit(X[mask == 1], t[mask == 1])
        assert rel(ours.coef_, ref.coef_) < SIMT_TOL
        assert ours.score(X, t, row_mask=mask, mask_keep=0) == ref.score(X[mask == 0], t[mask == 0])
        Xs = np.c_[X, X[:, 3]]
        ours = b2.B200RidgeClassifier(alpha=0.0, ctx=ctx).fit(Xs, t)
        reduced = linear_model.RidgeClassifier(alpha=0.0).fit(X, t)
        assert ours.solver_ == "svd"
        assert np.mean(ours.predict(Xs) == reduced.predict(X)) >= 0.999
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)


def test_device_rows_and_device_labels(ctx):
    """1 M x 128: float64 host columns through upload_columns, ten fp32 labels on the device."""
    n, d, k = 1_000_000, 128, 10
    X, t = _data(n, d, k, seed=31)
    y = (np.arange(k, dtype=np.float32) * 3 - 7)[t]
    Xd = ctx.upload_columns([X[:, j] for j in range(d)])
    yd = ctx.to_device(y)
    try:
        ours = b2.B200RidgeClassifier(alpha=10.0, ctx=ctx).fit(Xd, yd)
        ref = linear_model.RidgeClassifier(alpha=10.0).fit(X, y)
        assert ours.classes_.dtype == np.float32 and np.array_equal(ours.classes_, ref.classes_)
        err = rel(_flat(ours), _flat(ref))
        assert err < COEF_TOL, err
        lab, dec = ours.predict(Xd), ours.decision_function(Xd)
        assert isinstance(lab, b2.DeviceArray) and lab.kind == "f32" and dec.shape == (n, k)
        agree = float(np.mean(lab.to_host() == ref.predict(X).astype(np.float32)))
        assert agree >= 0.999, agree
        assert abs(ours.score(Xd, yd) - ref.score(X, y)) <= 1.0 - agree + 1e-12
        lab.free(); dec.free()
    finally:
        Xd.free(); yd.free()
    print(f"\n[ridge classifier 1M x 128, 10 device labels] coef {err:.2e}, predict agreement {agree}")


def test_refusals_and_errors(ctx):
    lib = native.load()
    cl = np.array([0, 1, 2], np.float32)
    X = np.zeros((4, 2), np.float32)
    y = np.zeros(4, np.float32)
    out, counts = np.empty((3, 3)), np.empty(3)
    assert lib.b2_class_sums(ctx._h, X.ctypes.data, b2.F32, y.ctypes.data, 4, 2, 2, native.MEM_HOST, None, 1,
                             cl.ctypes.data, 1, None, out.ctypes.data, counts.ctypes.data) == -1
    bad = np.array([0, 2, 1], np.float32)
    assert lib.b2_class_sums(ctx._h, X.ctypes.data, b2.F32, y.ctypes.data, 4, 2, 2, native.MEM_HOST, None, 1,
                             bad.ctypes.data, 3, None, out.ctypes.data, counts.ctypes.data) == -1
    assert lib.b2_class_sums(ctx._h, X.ctypes.data, b2.F32, y.ctypes.data, 4, 2, 2, native.MEM_HOST, None, 1,
                             cl.ctypes.data, 33, None, out.ctypes.data, counts.ctypes.data) == -1
    w, b0 = np.zeros(2), np.zeros(1)
    assert lib.b2_classify(ctx._h, X.ctypes.data, b2.F32, None, 4, 2, 2, native.MEM_HOST, None, 1, w.ctypes.data,
                           b0.ctypes.data, 1, cl.ctypes.data, None, None, None) == -1
    assert lib.b2_classify(ctx._h, X.ctypes.data, b2.F32, None, 4, 2, 2, native.MEM_HOST, None, 1, w.ctypes.data,
                           b0.ctypes.data, 0, cl.ctypes.data, out.ctypes.data, None, None) == -1
    with pytest.raises(ValueError, match="alpha"):
        ctx.gram_reset(2)
        ctx.solve_classes(np.zeros((3, 3)), -1.0)
    with pytest.raises(ValueError, match="max_values"):
        yd = ctx.to_device(y)
        try:
            ctx.label_values(yd, max_values=33)
        finally:
            yd.free()
    Xd, yd = ctx.to_device(X), ctx.to_device(np.array([0.5, 1, 2, 3], np.float32))
    try:
        with pytest.raises(ValueError, match="Unknown label type"):
            b2.B200RidgeClassifier(ctx=ctx).fit(Xd, yd)
        with pytest.raises(ValueError, match="device y needs device rows"):
            b2.B200RidgeClassifier(ctx=ctx).fit(X, yd)
    finally:
        Xd.free(); yd.free()
