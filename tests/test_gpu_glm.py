"""PoissonRegressor / GammaRegressor / TweedieRegressor on the H100: the passes (b2_glm_pass, b2_glm_line_search,
b2_glm_predict) against scikit-learn's pointwise losses on float64 copies of the same rounded rows, on every row layout;
the estimators against scikit-learn's solver="newton-cholesky" on float64 copies of the rows.  Each test prints the
worst case it measured (run with -s).

Bounds are 5x the worst case measured on one H100 80GB HBM3 at a 700 W power limit:
  * the pass sums (loss, constant, gradient, Hessian, every ladder entry) and mu, relative to the largest entry of each:
    3e-14 (worst 5.9e-15; mu 3.5e-16); the counts are equal and repeated calls bit-identical;
  * the estimators against scikit-learn, 16 384 x D: coef_ / intercept_ relative 1.8e-14 (worst 3.5e-15), predict
    (relative) and score (absolute) 1.9e-14 (worst 3.8e-15), equal n_iter_ and the same warnings.
"""
import io
import warnings

import joblib
import numpy as np
import pytest
from sklearn import linear_model

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from test_glm_driver import CASES, NumpyGLMContext, make_data

pytestmark = pytest.mark.gpu

E_ARG, E_UNSUPPORTED = -1, -6
PASS_TOL = 3e-14
COEF_TOL = 1.8e-14
PRED_TOL = 1.9e-14
LOSSES = [(native.GLM_IDENTITY, 0.0), (native.GLM_LOG, 0.0), (native.GLM_LOG, 1.0), (native.GLM_LOG, 1.5),
          (native.GLM_LOG, 2.0), (native.GLM_LOG, 3.0)]
REF = NumpyGLMContext()


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def _rows(n, d, seed, kind):
    """(stored rows (float32 or bf16 bits) with 3 spare columns, their float64 values, y float32, coef, step)"""
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d + 3)) * 0.5).astype(np.float32)
    up = b2.native.to_bf16_bits(X) if kind == "bf16" else X
    Xv = b2.native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
    coef = rng.normal(size=d) * 0.4 / np.sqrt(d)
    y = rng.gamma(2.0, np.exp(Xv[:, :d] @ coef + 0.2) / 2.0).astype(np.float32)
    step = rng.normal(size=d) * 0.2 / np.sqrt(d)
    return up, Xv, y, coef, step


def _raw_pass(ctx, ptr, dt, yp, n, d, ldx, mk, mp, link, power, coef, b, hess):
    sums = np.empty(d + 8)
    H = np.empty((d + 1, d + 1)) if hess else None
    rc = native.load().b2_glm_pass(ctx._h, ptr, dt, yp, n, d, ldx, mk, mp, 1, link, power, coef.ctypes.data, b, 1,
                                   sums.ctypes.data, H.ctypes.data if hess else None)
    assert rc == 0, native.last_error()
    return sums, H


def _raw_ladder(ctx, ptr, dt, yp, n, d, ldx, mk, mp, link, power, coef, b, step, db):
    out = np.empty(21)
    rc = native.load().b2_glm_line_search(ctx._h, ptr, dt, yp, n, d, ldx, mk, mp, 1, link, power, coef.ctypes.data, b,
                                          step.ctypes.data, db, 21, out.ctypes.data)
    assert rc == 0, native.last_error()
    return out


def _check_sums(sums, H, want, d):
    got = dict(zip(("loss", "const", "sum_y", "kept", "y_out_of_range", "h_nonpos", "y_nonfinite"), sums[:7]))
    for k in ("kept", "y_out_of_range", "h_nonpos", "y_nonfinite"):
        assert got[k] == want[k], k
    errs = [rel(got[k], want[k]) for k in ("loss", "const", "sum_y")] + [rel(sums[7:], want["grad"])]
    if H is not None:
        assert np.array_equal(H, H.T)
        errs.append(rel(H, want["hessian"]))
    return max(errs)


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128])
def test_pass_sums_every_layout(ctx, kind, d):
    n = 4133                                         # ring tiles, then a partial tile on the direct kernel
    up, Xv, y, coef, step = _rows(n, d, 10 + d, kind)
    dt = b2.BF16 if kind == "bf16" else b2.F32
    es = 2 if kind == "bf16" else 4
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    cont = np.ascontiguousarray(up[:, :d])
    Xd, yd, md = ctx.to_device(cont, kind), ctx.to_device(y), ctx.to_device(mask)
    Xs = ctx.to_device(np.ascontiguousarray(up), kind)         # ldx = d + 3, starting one element in
    worst = 0.0
    try:
        for i, (link, power) in enumerate(LOSSES):
            b = 0.1 * i
            kw = dict(link=link, power=power)
            layouts = [("host", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, None, Xv[:, :d], None),
                       ("device", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, None, Xv[:, :d], None),
                       ("strided", Xs.ptr + es, yd.ptr, d + 3, native.MEM_DEVICE, None, Xv[:, 1:d + 1], None),
                       ("device masked", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, md.ptr, Xv[:, :d], mask),
                       ("host masked", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, mask.ctypes.data,
                        Xv[:, :d], mask)]
            for name, xp, yp, ldx, mk, mp, Xref, mref in layouts:
                want = REF.glm_pass(Xref, y, coef, b, row_mask=mref, hessian=True, **kw)
                sums, H = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, link, power, coef, b, True)
                err = _check_sums(sums, H, want, d)
                sums2, H2 = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, link, power, coef, b, True)
                assert np.array_equal(sums, sums2) and np.array_equal(H, H2), name
                sums3, _ = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, link, power, coef, b, False)
                assert np.array_equal(sums, sums3), name      # the Hessian does not touch the other sums
                lw = REF.glm_line_search(Xref, y, coef, b, step, -0.05, row_mask=mref, **kw)
                ladder = _raw_ladder(ctx, xp, dt, yp, n, d, ldx, mk, mp, link, power, coef, b, step, -0.05)
                assert np.array_equal(ladder, _raw_ladder(ctx, xp, dt, yp, n, d, ldx, mk, mp, link, power, coef, b,
                                                           step, -0.05))
                err = max(err, max(rel(ladder[k], lw[k]) for k in range(21)))
                assert err < PASS_TOL, (name, link, power, err)
                worst = max(worst, err)
        mu = ctx.glm_predict(cont, coef, 0.3, link=native.GLM_LOG)
        worst_mu = rel(mu, np.exp(Xv[:, :d] @ coef + 0.3))
        mud = ctx.glm_predict(Xd, coef, 0.3, link=native.GLM_IDENTITY)
        worst_mu = max(worst_mu, rel(mud.to_host(), Xv[:, :d] @ coef + 0.3))
        mud.free()
        assert worst_mu < PASS_TOL
    finally:
        for a in (Xd, yd, md, Xs):
            a.free()
    print(f"\n[glm pass {kind} d={d}] worst relative difference {worst:.2e} (mu {worst_mu:.2e})")


def test_out_of_range_and_hessian_counts(ctx):
    rng = np.random.default_rng(1)
    n, d = 1000, 4
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.normal(size=n).astype(np.float32)
    y[7] = np.nan
    y[9] = np.inf
    coef = np.zeros(d)
    for link, power in LOSSES:
        got = ctx.glm_pass(X, y, coef, 0.5, link=link, power=power)
        want = REF.glm_pass(X, y, coef, 0.5, link=link, power=power)
        for k in ("kept", "y_out_of_range", "h_nonpos", "y_nonfinite"):
            assert got[k] == want[k], (link, power, k)
    got = ctx.glm_pass(X, y, coef, 0.5, row_mask=np.ones(n, np.uint8), mask_keep=0)
    assert got["kept"] == 0 and got["loss"] == 0 and not np.any(got["grad"]) and not np.any(got["hessian"])


@pytest.mark.parametrize("label,ours_cls,sk_cls,extra,family", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("alpha", [0.0, 1e-3, 1.0])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_estimators_match_sklearn(ctx, label, ours_cls, sk_cls, extra, family, alpha, fit_intercept):
    X, y = make_data(family, n=16_384, d=24, seed=7)
    ours = ours_cls(ctx=ctx, alpha=alpha, fit_intercept=fit_intercept, **extra)
    ref = sk_cls(solver="newton-cholesky", alpha=alpha, fit_intercept=fit_intercept, **extra)
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X.astype(np.float32), y.astype(np.float32))
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X, y)
    assert [w.category for w in w_ours] == [w.category for w in w_ref]
    assert ours.n_iter_ == ref.n_iter_
    err = rel(np.r_[ours.coef_, ours.intercept_], np.r_[ref.coef_, ref.intercept_])
    assert err < COEF_TOL, err
    perr = rel(ours.predict(X.astype(np.float32)), ref.predict(X))
    serr = abs(ours.score(X.astype(np.float32), y.astype(np.float32)) - ref.score(X, y))
    assert perr < PRED_TOL and serr < PRED_TOL, (perr, serr)
    print(f"\n[glm {label} alpha={alpha} fit_intercept={fit_intercept}] n_iter {ours.n_iter_}, coef {err:.2e}, "
          f"predict {perr:.2e}, score {serr:.2e}")


@pytest.mark.parametrize("d", [1, 128])
def test_poisson_every_width_warm_start_and_device_rows(ctx, d):
    X, y = make_data("poisson", n=16_384, d=d, seed=11)
    X32, y32 = X.astype(np.float32), y.astype(np.float32)
    ref = linear_model.PoissonRegressor(solver="newton-cholesky", alpha=1e-3, warm_start=True, max_iter=2)
    ours = b2.B200PoissonRegressor(ctx=ctx, alpha=1e-3, warm_start=True, max_iter=2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref.fit(X, y)
        ours.fit(X32, y32)
    ref.max_iter = ours.max_iter = 100
    ref.fit(X[:12_000], y[:12_000])
    Xd, yd = ctx.to_device(np.ascontiguousarray(X32[:12_000])), ctx.to_device(np.ascontiguousarray(y32[:12_000]))
    try:
        ours.fit(Xd, yd)
        mu = ours.predict(Xd)
        assert isinstance(mu, b2.DeviceArray)
        perr = rel(mu.to_host(), ref.predict(X[:12_000]))
        mu.free()
    finally:
        Xd.free(); yd.free()
    err = rel(np.r_[ours.coef_, ours.intercept_], np.r_[ref.coef_, ref.intercept_])
    assert ours.n_iter_ == ref.n_iter_ and err < COEF_TOL and perr < PRED_TOL, (err, perr)
    print(f"\n[glm poisson d={d} warm start, device rows] coef {err:.2e}, predict {perr:.2e}")


def test_masked_rows_repeats_and_joblib(ctx):
    X, y = make_data("gamma", n=16_384, d=16, seed=12)
    mask = (np.arange(len(y)) % 4 != 1).astype(np.uint8)
    Xn = X.astype(np.float32)
    yn = y.astype(np.float32)
    Xn[mask == 0, 3] = np.nan
    yn[mask == 0] = -np.inf
    ref = linear_model.GammaRegressor(solver="newton-cholesky", alpha=1e-3).fit(X[mask == 1], y[mask == 1])
    fits = [b2.B200GammaRegressor(ctx=ctx, alpha=1e-3).fit(Xn, yn, row_mask=mask) for _ in range(2)]
    Xd, yd, md = ctx.to_device(Xn), ctx.to_device(yn), ctx.to_device(mask)
    try:
        fits.append(b2.B200GammaRegressor(ctx=ctx, alpha=1e-3).fit(Xd, yd, row_mask=md))
    finally:
        Xd.free(); yd.free(); md.free()
    for f in fits:
        assert np.array_equal(f.coef_, fits[0].coef_) and f.intercept_ == fits[0].intercept_
    err = rel(np.r_[fits[0].coef_, fits[0].intercept_], np.r_[ref.coef_, ref.intercept_])
    assert fits[0].n_iter_ == ref.n_iter_ and err < COEF_TOL, err
    buf = io.BytesIO()
    joblib.dump(fits[0].to_sklearn(), buf)
    buf.seek(0)
    sk = joblib.load(buf)
    X32 = X.astype(np.float32)
    assert rel(sk.predict(X32.astype(np.float64)), fits[0].predict(X32)) < PRED_TOL
    assert abs(sk.score(X[mask == 1], y[mask == 1]) - fits[0].score(X32[mask == 1], y[mask == 1].astype(np.float32))) \
        < PRED_TOL


def test_refusals_and_errors(ctx):
    X, y = make_data("poisson", n=1000, d=4)
    X32, y32 = X.astype(np.float32), y.astype(np.float32)
    with pytest.raises(ValueError, match="sample_weight"):
        b2.B200PoissonRegressor(ctx=ctx).fit(X32, y32, sample_weight=np.ones(1000))
    with pytest.raises(ValueError, match="newton-cholesky"):
        b2.B200GammaRegressor(ctx=ctx, solver="lbfgs").fit(X32, y32 + 1)
    with pytest.raises(ValueError, match="power 0 only"):
        b2.B200TweedieRegressor(ctx=ctx, power=1.5, link="identity").fit(X32, y32)
    with pytest.raises(ValueError, match="0 sample"):
        b2.B200PoissonRegressor(ctx=ctx).fit(X32, y32, row_mask=np.zeros(1000, np.uint8))
    Xn = X32.copy()
    Xn[5, 2] = np.nan
    with pytest.raises(ValueError, match="NaN, infinity"):
        b2.B200PoissonRegressor(ctx=ctx).fit(Xn, y32)
    with pytest.raises(ValueError, match="'HalfGammaLoss'"):
        b2.B200GammaRegressor(ctx=ctx).fit(X32, y32)             # Poisson counts include 0
    coef, o = np.zeros(4), np.zeros(16)
    lib = native.load()
    args = (ctx._h, X32.ctypes.data, b2.F32, y32.ctypes.data, 1000, 4, 4, native.MEM_HOST, None, 1)
    assert lib.b2_glm_pass(*args, native.GLM_IDENTITY, 1.0, coef.ctypes.data, 0.0, 1, o.ctypes.data, None) == E_ARG
    assert lib.b2_glm_pass(*args, native.GLM_LOG, float("nan"), coef.ctypes.data, 0.0, 1, o.ctypes.data, None) == E_ARG
    assert lib.b2_glm_pass(*args, 2, 1.0, coef.ctypes.data, 0.0, 1, o.ctypes.data, None) == E_ARG
    assert lib.b2_glm_pass(*args, native.GLM_LOG, 1.0, coef.ctypes.data, 0.0, 1, None, None) == E_ARG
    assert lib.b2_glm_line_search(*args, native.GLM_LOG, 1.0, coef.ctypes.data, 0.0, coef.ctypes.data, 0.0, 22,
                                  o.ctypes.data) == E_ARG
    assert lib.b2_glm_predict(ctx._h, X32.ctypes.data, b2.F32, 1000, 4, 4, native.MEM_HOST, native.GLM_LOG,
                              coef.ctypes.data, 0.0, None) == E_ARG
    other = b2.Context(0)
    try:
        b2.Context.comm_p2p_attach_local([ctx, other])
        rc = lib.b2_glm_pass(*args, native.GLM_LOG, 1.0, coef.ctypes.data, 0.0, 1, o.ctypes.data, None)
        assert rc == E_UNSUPPORTED, rc
    finally:
        for c in (ctx, other):
            c.comm_p2p_detach()
        other.close()
