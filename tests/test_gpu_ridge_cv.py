"""RidgeCV on the H100: b2_solve_eigh (two-sided Jacobi) and b2_ridge_loo (the leave-one-out pass) against the numpy
oracle (tests/loo_oracle.py) and scikit-learn's RidgeCV.

Tolerances (asserted; the worst case measured on one H100 80GB HBM3 is printed by each test with -s):
  * eigh, designed statistics at every D in 1..128: ||Q^T Q - I||_max <= 8 D eps (worst 0.48 of it),
    ||A Q - Q L||_max / ||A||_max <= 8 D eps (worst 0.18), eigenvalues within 8 D eps lambda_max of eigvalsh of the same
    fp64 centred Gram (worst 0.12).
  * LOO on the exact (SIMT) Gram path, D in {1, 3, 8, 16, 17, 40, 127, 128}: mse relative 1e-10 (worst 6.2e-14), cv
    max |difference| / max cv 1e-9 (worst 2.7e-13).
  * every Gram path, mse relative to the oracle of the same (rounded) rows, on offset and correlated tables: per path,
    5x the worst measured (tensor core 3.3e-7 .. 1.1e-5, narrow 6.4e-11 .. 3.4e-9, SIMT 6.2e-9: the fp64 raw statistic
    cancels at mean / sigma = 1e4, as in test_gpu_columns) -- the pass is fp64 from the stored values, so the error is
    that of S, which moves beta(alpha) and through it every residual.
  * without an intercept on a moderately offset table (SIMT): mse relative 1e-15 kappa, kappa of the uncentred Gram
    (measured 0.15 eps kappa at kappa = 6.8e3).
  * row masks with NaN / Inf in the dropped rows (narrow path): mse relative 1e-8, cv 1e-7 of the largest (2.8e-8).
  * the estimator's cv_results_ against sklearn's: 1e-10 of the largest on the SIMT path (1.3e-14), 1e-6 on the narrow
    path of the 100-alpha chunked fit (6.1e-9).
  * host rows against device rows on the exact path: identical up to one staging block (262 144 rows); beyond it the
    Gram's sums split differently: cv within 1e-10 of the largest, mse relative 1e-12.
Measured on one H100 80GB HBM3 at a 700 W power limit.
"""
import ctypes as C

import numpy as np
import pytest
from sklearn.linear_model import RidgeCV

import bodywork_mlops_demo_b200 as b2
from loo_oracle import ridge_loo
from solve_oracle import EPS, designed_statistic, random_orthogonal
from test_gpu_columns import PATHS, _table

pytestmark = pytest.mark.gpu

E_ARG, E_UNSUPPORTED = -1, -6
N = 1024
ALPHAS = [0.01, 0.1, 1.0, 10.0, 100.0]


def _fp64_centred(S, fit_intercept=True):
    d = S.shape[0] - 2
    if not fit_intercept:
        return S[:d, :d].copy()
    n = S[d, d]
    m = S[:d, d] * (1.0 / n)
    return S[:d, :d] - (n * m)[:, None] * m[None, :]


def _eigh_designs(d):
    rng = np.random.RandomState(9000 + d)
    u = rng.uniform(1.0, 2.0, d)
    out = [("eig[1,2]", u), ("geom 1e6", np.geomspace(1.0, 1e-6, d)), ("geom 1e11", np.geomspace(1.0, 1e-11, d)),
           ("multiplicity D", np.full(d, 1.5))]
    if d >= 8:
        e = u.copy(); e[:8] = 1.25
        out.append(("multiplicity 8", e))
    if d >= 2:
        e = u.copy(); e[0] = 0.0
        out.append(("null direction", e))
    designs = [(name, designed_statistic(d, e, n=N, seed=d)[0]) for name, e in out]
    designs.append(("all columns constant", designed_statistic(d, np.zeros(d), n=N, Q=np.eye(d),
                                                               means=np.full(d, 0.25))[0]))
    if d >= 2:
        e = u.copy(); e[0] = 0.0
        Q = np.zeros((d, d)); Q[0, 0] = 1.0; Q[1:, 1:] = random_orthogonal(d - 1, d)
        designs.append(("one zero column", designed_statistic(d, e, n=N, Q=Q)[0]))
    return designs


@pytest.mark.parametrize("dims", [(1, 65), (65, 129)])
def test_eigh_at_every_d(ctx, dims):
    worst = [0.0, 0.0, 0.0]
    for d in range(*dims):
        for name, S in _eigh_designs(d):
            for fi in (True, False):
                ctx.gram_import(S)
                lam, Q = ctx.solve_eigh(fit_intercept=fi)
                A = _fp64_centred(S, fi)
                amax = float(np.max(np.abs(A))) or 1.0
                tol = 8 * d * EPS
                orth = float(np.max(np.abs(Q.T @ Q - np.eye(d))))
                res = float(np.max(np.abs(A @ Q - Q * lam))) / amax
                ref = np.maximum(np.linalg.eigvalsh(A), 0.0)
                lmax = max(float(np.max(np.abs(np.linalg.eigvalsh(A)))), 1e-300)
                ev = float(np.max(np.abs(lam - ref))) / lmax if lmax > 1e-300 else float(np.max(np.abs(lam)))
                assert np.all(np.diff(lam) >= 0) and np.all(lam >= 0), f"{name}: D = {d}"
                assert orth <= tol, f"{name}: D = {d}, intercept {fi}: ||Q^T Q - I|| {orth:.3e} > {tol:.3e}"
                assert res <= tol, f"{name}: D = {d}, intercept {fi}: ||AQ - QL|| / ||A|| {res:.3e} > {tol:.3e}"
                assert ev <= tol, f"{name}: D = {d}, intercept {fi}: eigenvalue error {ev:.3e} > {tol:.3e}"
                worst = [max(worst[0], orth / tol), max(worst[1], res / tol), max(worst[2], ev / tol)]
    print(f"\neigh D in {dims}: worst / bound: orthogonality {worst[0]:.3g}, residual {worst[1]:.3g}, "
          f"eigenvalues {worst[2]:.3g}")


def _rows(n, d, seed, offset=0.0, corr=0.0):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    if corr:
        X[:, 1:] = corr * X[:, :1] + (1 - corr) * X[:, 1:]
    X = (X + offset).astype(np.float32)
    y = (X.astype(np.float64) @ rng.uniform(-1, 1, d) + rng.standard_normal(n)).astype(np.float32)
    return X, y


def _loo_device(ctx, X, y, alphas, kind="f32", mask=None, kernel=b2.KERNEL_AUTO, fit_intercept=True, store_cv=True):
    Xd = ctx.to_device(X if kind == "f32" else b2.native.to_bf16_bits(X), kind)
    yd = ctx.to_device(y)
    md = ctx.to_device(mask) if mask is not None else None
    ctx.set_kernel(kernel)
    try:
        mse, best, coef, b0, cv = ctx.ridge_loo(Xd, yd, alphas, md, 1, fit_intercept=fit_intercept, store_cv=store_cv)
        cvh = cv.to_host() if cv is not None else None
        if cv is not None:
            cv.free()
        return mse, best, coef, b0, cvh
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        for a in (Xd, yd, md):
            if a is not None:
                a.free()


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b)) / np.abs(np.asarray(b))))


@pytest.mark.parametrize("d", [1, 3, 8, 16, 17, 40, 127, 128])
def test_exact_path_matches_oracle_and_sklearn(ctx, d):
    X, y = _rows(3000 + d, d, d, offset=2.0, corr=0.5)
    mse, best, coef, b0, cv = _loo_device(ctx, X, y, ALPHAS, kernel=b2.KERNEL_SIMT)
    mse_o, cv_o, best_o = ridge_loo(X, y, ALPHAS)
    e_mse, e_cv = _rel(mse, mse_o), float(np.max(np.abs(cv - cv_o)) / np.max(cv_o))
    print(f"\nD = {d}: mse rel {e_mse:.3e}, cv {e_cv:.3e}")
    assert e_mse <= 1e-10 and e_cv <= 1e-9
    sk = RidgeCV(alphas=ALPHAS).fit(X.astype(np.float64), y.astype(np.float64))
    assert best == best_o and ALPHAS[best] == sk.alpha_
    assert -mse[best] == pytest.approx(sk.best_score_, rel=1e-9)


# path -> bound on the mse's relative error, 5x the worst of the offset and correlated tables measured on the H100.  The
# pass is fp64 from the stored values; what separates the paths is the error of S (test_gpu_columns), which moves
# beta(alpha) and every residual with it.
PATH_TOL = {"f32-d128": 5e-5, "f32-d72": 3e-5, "f32-d100": 4e-5, "packed-d24": 1e-5, "packed-d32": 1.5e-5,
            "packed-d48": 2e-5, "rawb-d128": 2e-6, "bf16-d96": 4e-5, "tc-d8": 4e-6, "narrow-d1": 5e-10,
            "narrow-d4": 3e-9, "narrow-d16": 7e-9, "narrow-bf16-d1": 6e-10, "narrow-bf16-d4": 2e-8,
            "narrow-bf16-d16": 1.2e-8, "simt-d8": 3e-8}


@pytest.mark.parametrize("family", ["offset", "correlated"])
@pytest.mark.parametrize("path", list(PATHS))
def test_every_gram_path(ctx, path, family):
    d, kind, kernel = PATHS[path]
    Xr, up, y = _table(20_000, d, family, kind, seed=d + 5)
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    ctx.set_kernel(kernel)
    try:
        mse, best, _, _, _ = ctx.ridge_loo(Xd, yd, ALPHAS)
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        Xd.free(); yd.free()
    mse_o, _, best_o = ridge_loo(Xr, y, ALPHAS)
    e = _rel(mse, mse_o)
    print(f"\n{path} {family}: mse rel {e:.3e}")
    assert e <= PATH_TOL[path], f"{path} {family}: {e:.3e}"


def test_layouts_host_device_tails_and_alpha_counts(ctx):
    """On the exact Gram path: a host block of up to 262 144 rows runs the Gram and the pass exactly as the same rows on
    the device (identical results); more rows split the Gram's sums differently (rounding-level differences)."""
    ctx.set_kernel(b2.KERNEL_SIMT)
    try:
        for d, n in ((1, 20), (3, 1013), (16, 70_001), (17, 4099), (127, 2050), (128, 300_001)):
            X, y = _rows(n, d, n, offset=1.0)
            for alphas in ([3.0], list(np.logspace(-3, 3, 64))):
                mse_d, best_d, coef_d, b0_d, cv_d = _loo_device(ctx, X, y, alphas, kernel=b2.KERNEL_SIMT)
                ctx.set_kernel(b2.KERNEL_SIMT)                  # _loo_device restores AUTO
                mse_h, best_h, coef_h, b0_h, cv_h = ctx.ridge_loo(X, y, alphas, store_cv=True)
                assert best_h == best_d
                if n <= 262_144:
                    assert np.array_equal(cv_d, cv_h) and np.array_equal(mse_d, mse_h), f"D = {d}, n = {n}"
                    assert np.array_equal(coef_d, coef_h) and b0_d == b0_h
                else:
                    assert float(np.max(np.abs(cv_d - cv_h)) / np.max(cv_d)) <= 1e-10 and _rel(mse_h, mse_d) <= 1e-12
                if n <= 5000:
                    mse_o, cv_o, _ = ridge_loo(X, y, alphas)
                    assert _rel(mse_d, mse_o) <= 1e-10
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)


def test_strided_rows(ctx):
    n, d, ld = 5000, 24, 29
    X, y = _rows(n, d, 3, offset=1.0)
    Xs = np.zeros((n, ld), np.float32); Xs[:, :d] = X; Xs[:, d:] = np.nan
    Xd, yd = ctx.to_device(Xs), ctx.to_device(y)
    ctx.set_kernel(b2.KERNEL_SIMT)
    try:
        al = np.asarray(ALPHAS)
        mse = np.empty(al.size); coef = np.empty(d); b0, best = C.c_double(0), C.c_int(0)
        rc = b2.native.load().b2_ridge_loo(ctx._h, Xd.ptr, b2.F32, yd.ptr, n, d, ld, 0, None, 1, al.ctypes.data,
                                           al.size, 1, mse.ctypes.data, None, C.byref(best), coef.ctypes.data,
                                           C.byref(b0))
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        Xd.free(); yd.free()
    assert rc == 0, b2.native.last_error()
    assert _rel(mse, ridge_loo(X, y, ALPHAS)[0]) <= 1e-10


def test_mask_with_nan_in_dropped_rows(ctx):
    n, d = 9000, 12
    X, y = _rows(n, d, 11, offset=3.0)
    mask = (np.random.RandomState(2).uniform(size=n) < 0.7).astype(np.uint8)
    X[mask == 0, 0] = np.nan; X[mask == 0, 1] = np.inf; y[mask == 0] = np.nan
    for where in ("device", "host"):
        if where == "device":
            mse, best, coef, b0, cv = _loo_device(ctx, X, y, ALPHAS, mask=mask)
        else:
            mse, best, coef, b0, cv = ctx.ridge_loo(X, y, ALPHAS, mask, 1, store_cv=True)
        assert np.all(np.isfinite(mse)) and np.all(np.isfinite(coef))
        assert np.array_equal(np.isnan(cv).all(axis=1), mask == 0) and not np.isnan(cv[mask == 1]).any()
        mse_o, cv_o, _ = ridge_loo(X, y, ALPHAS, mask=mask)
        assert _rel(mse, mse_o) <= 1e-8                  # the narrow Gram path (D = 12)
        assert float(np.max(np.abs(cv[mask == 1] - cv_o)) / np.max(cv_o)) <= 1e-7   # measured 2.8e-8


def test_without_intercept_on_offset_rows(ctx):
    X, y = _rows(6000, 8, 21, offset=20.0, corr=0.3)
    mse, best, _, _, cv = _loo_device(ctx, X, y, ALPHAS, kernel=b2.KERNEL_SIMT, fit_intercept=False)
    mse_o, cv_o, best_o = ridge_loo(X, y, ALPHAS, fit_intercept=False)
    Xf = X.astype(np.float64)
    kappa = float(np.linalg.cond(Xf.T @ Xf))
    e = _rel(mse, mse_o)
    print(f"\nno intercept: kappa {kappa:.3e}, mse rel {e:.3e} = {e / (EPS * kappa):.3g} eps kappa")
    assert e <= 1e-15 * kappa and best == best_o


def test_bit_identity_and_the_fit_at_the_chosen_alpha(ctx):
    X, y = _rows(200_000, 64, 31, offset=5.0, corr=0.8)
    Xd, yd = ctx.to_device(X), ctx.to_device(y)
    try:
        grid = list(np.logspace(-2, 4, 13))
        r1 = ctx.ridge_loo(Xd, yd, grid, store_cv=True)
        S1 = ctx.gram_export()
        r2 = ctx.ridge_loo(Xd, yd, grid, store_cv=True)
        assert np.array_equal(r1[0], r2[0]) and r1[1] == r2[1]
        assert np.array_equal(r1[4].to_host(), r2[4].to_host())
        r1[4].free(); r2[4].free()
        coef, b0 = ctx.fit(Xd, yd, alpha=grid[r1[1]])
        assert np.array_equal(coef, r1[2]) and b0 == r1[3]
        assert np.array_equal(S1, ctx.gram_export())
    finally:
        Xd.free(); yd.free()


def _sk(X, y, alphas, **kw):
    return RidgeCV(alphas=alphas, store_cv_results=True, **kw).fit(np.asarray(X, np.float64), np.asarray(y, np.float64))


def test_estimator_against_sklearn(ctx, tmp_path):
    import joblib
    X, y = _rows(4000, 10, 41, offset=2.0, corr=0.6)
    for rows in ("f32", "f64", "device"):
        Xin = X.astype(np.float64) if rows == "f64" else X
        if rows == "device":
            Xin, yin = ctx.to_device(X), ctx.to_device(y)
        else:
            yin = y
        est = b2.B200RidgeCV(ALPHAS, store_cv_results=True, ctx=ctx).fit(Xin, yin)
        sk = _sk(X, y, ALPHAS)
        assert est.alpha_ == sk.alpha_ and est.n_features_in_ == 10
        assert est.best_score_ == pytest.approx(sk.best_score_, rel=1e-3)
        np.testing.assert_allclose(est.coef_, sk.coef_, rtol=1e-3, atol=1e-5)
        assert est.cv_results_.shape == sk.cv_results_.shape
        e_cv = float(np.max(np.abs(est.cv_results_ - sk.cv_results_)) / np.max(sk.cv_results_))
        print(f"\nestimator, {rows} rows: cv_results_ {e_cv:.3e}")
        assert e_cv <= 1e-10                                      # SIMT Gram (40-byte rows), measured 1.3e-14
        if rows == "device":
            Xin.free(); yin.free()
    # float64 host rows large enough for the upload path, a 100-alpha grid (two calls, merged by the first minimum)
    Xb, yb = _rows(70_000, 8, 43, offset=1.0, corr=0.5)
    grid = np.logspace(-3, 5, 100)
    mask = (np.random.RandomState(44).uniform(size=Xb.shape[0]) < 0.8).astype(np.uint8)
    est = b2.B200RidgeCV(grid, store_cv_results=True, ctx=ctx).fit(Xb.astype(np.float64), yb, row_mask=mask)
    sk = _sk(Xb[mask == 1], yb[mask == 1], grid)
    assert est.alpha_ == sk.alpha_ and est.best_score_ == pytest.approx(sk.best_score_, rel=1e-3)
    assert est.cv_results_.shape == sk.cv_results_.shape == (int(mask.sum()), 100)   # chunks in alpha order, kept rows
    e_cv = float(np.max(np.abs(est.cv_results_ - sk.cv_results_)) / np.max(sk.cv_results_))
    print(f"\nestimator, 100 alphas, masked float64 rows: cv_results_ {e_cv:.3e}")
    assert e_cv <= 1e-6                                          # narrow Gram path
    path = tmp_path / "ridge.joblib"
    joblib.dump(est.to_sklearn(), path)
    reg = joblib.load(path)
    assert type(reg) is RidgeCV and reg.alpha_ == est.alpha_
    np.testing.assert_allclose(reg.predict(Xb[:100].astype(np.float64)), est.predict(Xb[:100]), rtol=1e-5, atol=1e-4)


def test_errors(ctx):
    X, y = _rows(500, 4, 51)
    with pytest.raises(ValueError, match=r"alphas\[1\] == 0.0, must be > 0.0."):
        b2.B200RidgeCV([1.0, 0.0], ctx=ctx).fit(X, y)
    with pytest.raises(ValueError, match=r"alphas\[0\] == -1.0, must be > 0.0."):
        b2.B200RidgeCV([-1.0], ctx=ctx).fit(X, y)
    with pytest.raises(ValueError):
        b2.B200RidgeCV([float("nan")], ctx=ctx).fit(X, y)
    with pytest.raises(ValueError, match="0 sample"):
        b2.B200RidgeCV(ctx=ctx).fit(X, y, row_mask=np.zeros(500, np.uint8))
    for alphas in ([], [1.0] * 65, [0.0], [float("nan")], [float("inf")]):
        with pytest.raises(RuntimeError, match="code -1"):
            ctx.ridge_loo(X, y, alphas)
    al = np.asarray(ALPHAS)
    coef, b0, best = np.empty(4), C.c_double(0), C.c_int(0)
    rc = b2.native.load().b2_ridge_loo(ctx._h, X.ctypes.data, b2.F32, y.ctypes.data, 500, 4, 4, 1, None, 1,
                                       al.ctypes.data, al.size, 1, None, None, C.byref(best), coef.ctypes.data,
                                       C.byref(b0))
    assert rc == E_ARG
    other = b2.Context(0)
    try:
        b2.Context.comm_p2p_attach_local([ctx, other])
        with pytest.raises(RuntimeError, match="code -6"):
            ctx.ridge_loo(X, y, ALPHAS)
    finally:
        for c in (ctx, other):
            c.comm_p2p_detach()
        other.close()
