"""LinearSVC / LinearSVR on the H100: b2_svm_pass against a float64 numpy statement of the pass on the same stored rows,
on every row layout, at controlled numbers of rows changing side and with rows exactly on the margin; the estimators
against scikit-learn's liblinear primal solver; a 1 M x 128 fit from device rows and device labels; the ABI refusals."""
import warnings

import numpy as np
import pytest
from sklearn import svm

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native

pytestmark = pytest.mark.gpu

E_ARG = -1
HINGE, EPS = native.SVM_SQUARED_HINGE, native.SVM_SQUARED_EPSILON
PASS_TOL = 1e-13


def rel(a, b, scale=None):
    a, b = np.asarray(a, float), np.asarray(b, float)
    s = max(np.max(np.abs(b)) if scale is None else scale, 1e-300)
    return float(np.max(np.abs(a - b)) / s) if b.size else 0.0


def _raw(ctx, xp, dt, yp, n, d, ldx, mk, mp, loss, param, wf, bf, w, b, fi=True, hess=True):
    sums = np.empty(d + 8)
    H = np.empty((d + 1, d + 1)) if hess else None
    rc = native.load().b2_svm_pass(ctx._h, xp, dt, yp, n, d, ldx, mk, mp, 1, loss, float(param),
                                   wf.ctypes.data if wf is not None else None, float(bf), w.ctypes.data, float(b),
                                   int(fi), sums.ctypes.data, H.ctypes.data if hess else None)
    assert rc == 0, native.last_error()
    return sums, H


def _active(eta, y, loss, param):
    if loss == HINGE:
        return 1.0 - np.where(y == param, 1.0, -1.0) * eta > 0.0
    return np.abs(eta - y) > param


def _reference(Xv, y, loss, param, wf, bf, w, b, keep, fi=True):
    """the pass in float64: counts, loss, gradient, the Hessian change, and the Gram of the rows active at w"""
    Xk, yk = Xv[keep], y[keep]
    Z = np.c_[Xk, np.ones(len(yk))]
    b = b if fi else 0.0
    eta = Xk @ w + b
    act = _active(eta, yk, loss, param)
    act_f = np.zeros_like(act) if wf is None else _active(Xk @ wf + (bf if fi else 0.0), yk, loss, param)
    if loss == HINGE:
        t = np.where(yk == param, 1.0, -1.0)
        lo, g = (1.0 - t * eta) ** 2, eta - t
    else:
        r = eta - yk
        g = np.where(r > param, r - param, r + param)
        lo = g * g
    sg = act.astype(float) - act_f.astype(float)
    return {"loss": np.sum(lo[act]), "counts": [len(yk), act.sum(), np.sum(act & ~act_f), np.sum(act_f & ~act),
                                                np.sum(yk == param) if loss == HINGE else 0, np.sum(~np.isfinite(yk))],
            "grad": Z.T @ np.where(act, g, 0.0), "dH": (Z * sg[:, None]).T @ Z, "gram": Z[act].T @ Z[act]}


def _check(sums, H, want):
    assert list(sums[1:7]) == [float(c) for c in want["counts"]], (sums[1:7], want["counts"])
    assert sums[2] >= 0 and sums[3] >= 0 and sums[4] >= 0
    err = max(rel(sums[0], want["loss"]), rel(sums[7:], want["grad"]))
    if H is not None:
        assert np.array_equal(H, H.T)
        err = max(err, rel(H, want["dH"], scale=np.max(np.abs(want["gram"])) + np.max(np.abs(want["dH"]))))
    return err


def _rows(n, d, seed, kind):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d + 3)) * 0.7 + 0.2).astype(np.float32)
    up = b2.native.to_bf16_bits(X) if kind == "bf16" else X
    Xv = b2.native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
    return rng, up, Xv


LAYOUT_D = [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128]


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", LAYOUT_D)
def test_pass_every_layout(ctx, kind, d):
    """both losses at a step from an accepted point; counts exact, active(to) = active(from) + entering - leaving,
    sums to 1e-13, ΔH(∅→w0) + ΔH(w0→w1) = ΔH(∅→w1), repeated calls bit-identical"""
    n = 4133                                         # ring tiles, then a partial tile on the direct kernel
    dt = b2.BF16 if kind == "bf16" else b2.F32
    es = 2 if kind == "bf16" else 4
    rng, up, Xv = _rows(n, d, 10 * d + (kind == "bf16"), kind)
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    cont = np.ascontiguousarray(up[:, :d])
    w0 = rng.normal(size=d) / np.sqrt(d)
    w1 = w0 + rng.normal(size=d) * 0.3 / np.sqrt(d)
    score = Xv[:, :d] @ w0
    worst = 0.0
    for loss in (HINGE, EPS):
        if loss == HINGE:
            y = np.where(score + rng.normal(size=n) * 0.5 > 0, 7.0, 3.0).astype(np.float32)
            param = 7.0
        else:
            y = (score + rng.normal(size=n) * 0.5).astype(np.float32)
            param = 0.4
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
                keep = np.ones(n, bool) if mref is None else mref == 1
                args = (ctx, xp, dt, yp, n, d, ldx, mk, mp, loss, param)
                for fi in (True, False):
                    s0, H0 = _raw(*args, None, 0.0, w0, 0.3, fi)
                    s1, H1 = _raw(*args, w0, 0.3, w1, -0.2, fi)
                    s1b, H1b = _raw(*args, w0, 0.3, w1, -0.2, fi)
                    assert np.array_equal(s1, s1b) and np.array_equal(H1, H1b), name
                    g1, _ = _raw(*args, w0, 0.3, w1, -0.2, fi, False)
                    assert np.array_equal(g1[1:7], s1[1:7]) and rel(g1, s1) < PASS_TOL, name   # other CTAs per SM
                    sd, Hd = _raw(*args, None, 0.0, w1, -0.2, fi)
                    assert s1[2] == s0[2] + s1[3] - s1[4] and sd[2] == s1[2], name
                    err = max(_check(s0, H0, _reference(Xref, y, loss, param, None, 0.0, w0, 0.3, keep, fi)),
                              _check(s1, H1, _reference(Xref, y, loss, param, w0, 0.3, w1, -0.2, keep, fi)))
                    err = max(err, rel(H0 + H1, Hd, scale=np.max(np.abs(Hd))))
                    assert err < PASS_TOL, (name, loss, fi, err)
                    worst = max(worst, err)
        finally:
            for a in (Xd, yd, md, Xs):
                a.free()
    print(f"\n[svm pass {kind} d={d}] worst relative difference {worst:.2e}")


def test_changed_rows_many_tiles_per_cta(ctx):
    """0, fewer than 32, not a multiple of 32 and all rows changing side, with every CTA streaming many ring tiles"""
    n, d = 32 * (18 * ctx.info()["sm_count"] + 5) + 17, 24     # at least 18 ring tiles per CTA, then a direct tail
    rng, up, Xv = _rows(n, d, 3, "f32")
    Xc = np.ascontiguousarray(up[:, :d])
    y = np.full(n, 1.0, np.float32)                  # every row positive: an intercept shift db moves m by -db
    w = rng.normal(size=d) / np.sqrt(d)
    m = 1.0 - (Xv[:, :d] @ w)
    pos_m = np.sort(m[m > 0])
    Xd, yd = ctx.to_device(Xc), ctx.to_device(y)
    keep = np.ones(n, bool)
    try:
        for c in (0, 5, 100, 777):
            db = 0.0 if c == 0 else 0.5 * (pos_m[c - 1] + pos_m[c])   # rows with 0 < m <= db leave
            for xp, yp, mk in ((Xd.ptr, yd.ptr, native.MEM_DEVICE), (Xc.ctypes.data, y.ctypes.data, native.MEM_HOST)):
                s, H = _raw(ctx, xp, b2.F32, yp, n, d, d, mk, None, HINGE, 1.0, w, 0.0, w, db)
                assert s[3] + s[4] == c, (c, s[3], s[4])
                assert _check(s, H, _reference(Xv[:, :d], y, HINGE, 1.0, w, 0.0, w, db, keep)) < PASS_TOL
                s2, H2 = _raw(ctx, xp, b2.F32, yp, n, d, d, mk, None, HINGE, 1.0, w, 0.0, w, db)
                assert np.array_equal(s, s2) and np.array_equal(H, H2)
        zero = np.zeros(d)
        s, H = _raw(ctx, Xd.ptr, b2.F32, yd.ptr, n, d, d, native.MEM_DEVICE, None, HINGE, 1.0, None, 0.0, zero, 0.0)
        assert s[3] == n and s[2] == n                 # all rows enter: the Gram of [x 1]
        Z = np.c_[Xv[:, :d], np.ones(n)]
        assert rel(H, Z.T @ Z) < PASS_TOL
    finally:
        Xd.free()
        yd.free()


def test_rows_exactly_on_the_margin(ctx):
    """integer rows and dyadic coefficients: eta is exact, so rows with m = 0 or |r| = eps exactly are inactive"""
    rng = np.random.default_rng(4)
    n, d = 3000, 5
    X = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    w = rng.integers(-4, 5, size=d) / 4.0
    b = 0.5
    eta = X.astype(np.float64) @ w + b
    y = np.where(rng.uniform(size=n) < 0.5, 1.0, -1.0).astype(np.float32)
    y[eta == 1.0] = 1.0                                # on the margin: t eta = 1
    y[eta == -1.0] = -1.0
    keep = np.ones(n, bool)
    on = int(np.sum(np.abs(eta) == 1.0))
    assert on > 20
    s, H = _raw(ctx, X.ctypes.data, b2.F32, y.ctypes.data, n, d, d, native.MEM_HOST, None, HINGE, 1.0, None, 0.0, w, b)
    assert _check(s, H, _reference(X.astype(np.float64), y, HINGE, 1.0, None, 0.0, w, b, keep)) < PASS_TOL
    ye = (eta + rng.choice([-0.5, 0.5, 0.25], size=n)).astype(np.float32)   # |r| = eps = 0.5 on a third of the rows
    s, H = _raw(ctx, X.ctypes.data, b2.F32, ye.ctypes.data, n, d, d, native.MEM_HOST, None, EPS, 0.5, None, 0.0, w, b)
    want = _reference(X.astype(np.float64), ye, EPS, 0.5, None, 0.0, w, b, keep)
    assert _check(s, H, want) < PASS_TOL and want["counts"][1] < n * 0.5


def _fit_both(ours, ref, X, y):
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X, y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X.astype(np.float32).astype(np.float64), y)
    return [w.category for w in w_ours], [w.category for w in w_ref]


@pytest.mark.parametrize("k,C", [(2, 1.0), (2, 100.0), (3, 0.01), (10, 1.0)])
def test_linear_svc_matches_sklearn(ctx, k, C):
    rng = np.random.default_rng(k)
    X = rng.normal(size=(16384, 24)) + 0.3
    t = np.argmax(X @ rng.normal(size=(24, k)) + rng.normal(size=(16384, k)) * 2.0, axis=1)
    ours, ref = b2.B200LinearSVC(C=C, ctx=ctx), svm.LinearSVC(C=C, dual=False)
    w_ours, w_ref = _fit_both(ours, ref, X, t)
    assert w_ours == w_ref
    assert ours.n_iter_ == ref.n_iter_
    err = rel(np.c_[ours.coef_, ours.intercept_], np.c_[ref.coef_, ref.intercept_])
    print(f"\n[LinearSVC k={k} C={C}] n_iter {ours.n_iter_}, coefficients {err:.2e}")
    assert err < 1e-10
    assert np.mean(ours.predict(X) == ref.predict(X)) > 0.9999


@pytest.mark.parametrize("epsilon", [0.0, 0.5])
def test_linear_svr_matches_sklearn(ctx, epsilon):
    rng = np.random.default_rng(9)
    X = rng.normal(size=(16384, 24))
    y = (X @ rng.normal(size=24) + 1.0 + rng.normal(size=16384)).astype(np.float32)
    kw = dict(epsilon=epsilon, loss="squared_epsilon_insensitive")
    ours, ref = b2.B200LinearSVR(ctx=ctx, **kw), svm.LinearSVR(dual=False, **kw)
    _fit_both(ours, ref, X, y.astype(np.float64))
    assert ours.n_iter_ == ref.n_iter_
    err = rel(np.r_[ours.coef_, ours.intercept_], np.r_[ref.coef_, ref.intercept_])
    print(f"\n[LinearSVR eps={epsilon}] n_iter {ours.n_iter_}, coefficients {err:.2e}")
    assert err < 1e-10
    np.testing.assert_allclose(ours.predict(X), ref.predict(X.astype(np.float32).astype(np.float64)), rtol=1e-9,
                               atol=1e-9)
    assert abs(ours.score(X, y) - ref.score(X.astype(np.float32).astype(np.float64), y)) < 1e-9


def test_large_fit_from_device_rows_and_labels(ctx):
    n, d = 1_000_000, 128
    rng = np.random.default_rng(6)
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = np.where(X.astype(np.float64) @ rng.normal(size=d) / np.sqrt(d) + rng.normal(size=n) * 0.5 > 0, 4.0,
                 -2.0).astype(np.float32)
    Xd, yd = ctx.to_device(X), ctx.to_device(y)
    try:
        ours = b2.B200LinearSVC(ctx=ctx).fit(Xd, yd)
        assert list(ours.classes_) == [-2.0, 4.0] and ours.classes_.dtype == np.float32
        ref = svm.LinearSVC(dual=False).fit(X.astype(np.float64), y)
        assert ours.n_iter_ == ref.n_iter_
        err = rel(np.c_[ours.coef_, ours.intercept_], np.c_[ref.coef_, ref.intercept_])
        print(f"\n[LinearSVC 1M x 128 device] n_iter {ours.n_iter_}, coefficients {err:.2e}")
        assert err < 1e-9
        lab = ours.predict(Xd)
        assert np.mean(lab.to_host() == ref.predict(X.astype(np.float64))) > 0.9999
        lab.free()
    finally:
        Xd.free()
        yd.free()


def test_abi_refusals(ctx):
    lib = native.load()
    n, d = 64, 4
    X = np.zeros((n, d), np.float32)
    y = np.zeros(n, np.float32)
    w = np.zeros(d)
    sums = np.empty(d + 8)
    args = (ctx._h, X.ctypes.data, b2.F32, y.ctypes.data, n, d, d, native.MEM_HOST, None, 1)
    assert lib.b2_svm_pass(*args, 2, 1.0, None, 0.0, w.ctypes.data, 0.0, 1, sums.ctypes.data, None) == E_ARG
    assert lib.b2_svm_pass(*args, EPS, -0.1, None, 0.0, w.ctypes.data, 0.0, 1, sums.ctypes.data, None) == E_ARG
    assert lib.b2_svm_pass(*args, HINGE, np.nan, None, 0.0, w.ctypes.data, 0.0, 1, sums.ctypes.data, None) == E_ARG
    assert lib.b2_svm_pass(*args, HINGE, 1.0, None, 0.0, None, 0.0, 1, sums.ctypes.data, None) == E_ARG
    assert lib.b2_svm_pass(*args, HINGE, 1.0, None, 0.0, w.ctypes.data, 0.0, 1, None, None) == E_ARG
    empty = (ctx._h, None, b2.F32, None, 0, d, d, native.MEM_HOST, None, 1)
    assert lib.b2_svm_pass(*empty, HINGE, 1.0, None, 0.0, w.ctypes.data, 0.0, 1, sums.ctypes.data, None) == 0
    assert not np.any(sums)
