"""The three fp64 solve kernels of csrc/solve.cu (the blocked LDL^T with its DMMA trailing update, the Householder +
Sturm eigenvalue kernel, the Jacobi minimum-norm kernel) and the estimator's rank rule, on designed statistics
(tests/solve_oracle.py).  Every statistic goes in through ``gram_import``, so no Gram-kernel rounding enters; row-based
statistics use integer-valued rows and the SIMT kernel, whose statistic of such rows is exact in fp64.

Tolerances, eps = 2^-52 (largest measured value / bound on one H100 80GB HBM3 at a 400 W power limit):
  LDL^T, every D in 1 .. 128, four spectra up to kappa 1e11, alpha in {0, 1e-3 lambda_max}, with and without an
  intercept, zero and non-zero means: normwise backward error against the longdouble system of the statistic
      eta <= 8 (D + 1) eps  (+ 2 eps n max|m_i| max|m_j| / ||A||_inf with non-zero means: the fp64 centring);
      measured 0.023 of the bound
  intercept against ybar - m.beta^ in longdouble:  2 (D + 2) eps (|ybar| + sum |m_i beta^_i|);  measured 0.042
  eigenvalues, every D, ten spectra: |lambda^_i - lambda_i| <= 8 D eps lambda_max against eigvalsh of the same fp64
      centred Gram;  measured 0.10
  minimum-norm coefficients against the truncated solution in longdouble, kappa_kept up to 1e8, 1 .. D-1 dropped
      directions (0, 1e-14 lambda_max, -1e-9 lambda_max):
      ||beta^ - beta_ref||_inf <= 8 D eps (lambda_max / lambda_min,kept) ||r||_inf / lambda_min,kept;  measured 0.12
      up to D = 33, and at D = 128 for kappa_kept <= 1e4.  At D = 128, kappa_kept = 1e8 the kernel misses it (up to
      29 times the bound, an expected failure, strict): see below.
  the minimum-norm kernel's kept eigenvalues against the eigenvalue kernel's: 8 D eps lambda_max, as above.
  Its dropped eigenvalues cannot meet that bound, for a reason of principle: one-sided Jacobi on A rotates every
  column against the D - 1 others in each of up to JACOBI_SWEEPS sweeps; the products and the sum of a rotation round,
  leaving about 2 eps times the norms of the pair.  A column whose eigenvalue is zero never converges (its cosines with
  the others are rounding noise), so such a statistic runs every sweep and that column's norm (its lambda^) ends at up
  to NULL = 2 JACOBI_SWEEPS D eps ||A||_F;  measured 0.47 NULL (6.5e-13 lambda_max at D = 128: a factor 1.5 below the
  1e-12 cutoff, which is why the estimator takes rank_ and singular_ from the eigenvalue kernel).  The same rounding
  reaches the kept columns, which is what the D = 128, kappa_kept = 1e8 case shows; a Jacobi that leaves numerically
  null columns alone would remove it.  The sweeps' stopping threshold plays no part: a sweep that finds every cosine
  below it has already rotated them to rounding level (quadratic convergence), and raising it from 1e-13 to 1e-8
  changes none of these results.
  power-of-two scalings: bit for bit.
"""
import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc
from solve_oracle import (EPS, backward_error, designed_statistic, exact_centred, integer_window_rows, ldlt_pivots,
                          random_orthogonal, truncated_solution)

pytestmark = pytest.mark.gpu

N = 1024                       # rows of a designed statistic: a power of two, so n m and S / n are exact
JACOBI_SWEEPS = 24             # solve_spectral_kernel's sweep limit
JACOBI_XFAIL = ("solve_spectral_kernel at D = 128, kappa_kept = 1e8: with a null direction the Jacobi sweeps run to "
                "their limit and the coefficients end up to 29 times the 8 D eps bound off (see the module docstring)")


def _means(d, seed, scale=2.0 ** -5):
    """exactly representable means whose centring term n m_i m_j = j_i j_j / 64 (scale 2^-5, n = 1024) is exact"""
    return np.random.RandomState(seed).randint(-4, 5, d) / 8.0 * scale


def _col_scaled(S, k):
    """the statistic of the columns x_j * 2^k_j: S_xx, S_x1, S_xy scaled exactly"""
    d = S.shape[0] - 2
    t = np.ones(d + 2)
    t[:d] = np.exp2(k)
    return S * np.outer(t, t)


def _sweep_designs(d):
    """(name, S, means) for the LDL^T sweep at one D"""
    rng = np.random.RandomState(4000 + d)
    spectra = [("eig[1,2]", rng.uniform(1.0, 2.0, d)), ("geom 1e6", np.geomspace(1.0, 1e-6, d)),
               ("geom 1e11", np.geomspace(1.0, 1e-11, d)), ("scales 2^k", rng.uniform(1.0, 2.0, d))]
    ks = rng.randint(-8, 9, d)
    for name, eigs in spectra:
        for with_means in (False, True):
            m = _means(d, d + 17) if with_means else None
            S, _, _ = designed_statistic(d, eigs, n=N, means=m, ybar=1.5 if with_means else 0.0, seed=d)
            if name == "scales 2^k":
                S = _col_scaled(S, ks)
                m = None if m is None else m * np.exp2(ks)
            yield f"{name}{' +means' if with_means else ''}", S, m


def _check_ldlt(ctx, S, m, d, alpha, fi, label):
    """returns (eta / bound, intercept error / bound)"""
    ctx.gram_import(S)
    coef, b0 = ctx.solve(alpha=alpha, fit_intercept=bool(fi))
    A, r, mL, ybar = exact_centred(S, bool(fi))
    A = A + np.eye(d, dtype=A.dtype) * alpha
    bound = 8 * (d + 1) * EPS
    if m is not None and fi:
        bound += 2 * EPS * N * np.max(np.abs(m)) ** 2 / float(np.max(np.sum(np.abs(A), axis=1)))
    eta = backward_error(A, r, coef)
    assert eta <= bound, f"{label}: D = {d}, alpha = {alpha}, fit_intercept = {fi}: eta {eta:.3e} > {bound:.3e}"
    if fi:
        ref = ybar - mL @ coef.astype(np.longdouble)
        tol = 2 * (d + 2) * EPS * (abs(float(ybar)) + float(np.sum(np.abs(mL * coef.astype(np.longdouble)))))
        err = abs(float(b0 - ref))
        assert err <= tol, f"{label}: D = {d} intercept error {err:.3e} > {tol:.3e}"
        return eta / bound, (err / tol if tol > 0 else 0.0)
    assert b0 == 0.0
    return eta / bound, 0.0


@pytest.mark.parametrize("dims", [(1, 33), (33, 65), (65, 97), (97, 129)])
def test_ldlt_backward_error_at_every_d(ctx, dims):
    worst = [0.0, 0.0]
    for d in range(*dims):
        for label, S, m in _sweep_designs(d):
            lmax = float(np.max(np.linalg.eigvalsh(exact_centred(S)[0].astype(np.float64))))
            for alpha in (0.0, 1e-3 * lmax):
                for fi in (1, 0):
                    w = _check_ldlt(ctx, S, m, d, alpha, fi, label)
                    worst = [max(worst[0], w[0]), max(worst[1], w[1])]
    print(f"\nLDL^T D in {dims}: worst eta / bound {worst[0]:.3g}, intercept {worst[1]:.3g}")


# ------------------------------------------------------------------------------------------------
# eigenvalue kernel
# ------------------------------------------------------------------------------------------------
def _block_q(*blocks):
    d = sum(b.shape[0] for b in blocks)
    Q = np.zeros((d, d))
    o = 0
    for b in blocks:
        Q[o:o + b.shape[0], o:o + b.shape[0]] = b
        o += b.shape[0]
    return Q


def _eig_designs(d):
    """(name, S) with no singular value within a factor 4 of cond * sigma_max"""
    rng = np.random.RandomState(7000 + d)
    u = rng.uniform(1.0, 2.0, d)
    out = [("eig[1,2]", designed_statistic(d, u, n=N, seed=d)[0])]
    for mult in (2, 8):
        if d >= mult:
            e = u.copy()
            e[:mult] = 1.25
            out.append((f"multiplicity {mult}", designed_statistic(d, e, n=N, seed=d)[0]))
    out.append(("multiplicity D", designed_statistic(d, np.full(d, 1.5), n=N, seed=d)[0]))
    out.append(("c I", designed_statistic(d, np.full(d, 1.5), n=N, Q=np.eye(d))[0]))
    out.append(("all columns constant", designed_statistic(d, np.zeros(d), n=N, means=_means(d, d), Q=np.eye(d))[0]))
    if d >= 2:
        e = u.copy()
        e[0] = 0.0
        Q = _block_q(np.ones((1, 1)), random_orthogonal(d - 1, d))
        out.append(("one constant column", designed_statistic(d, e, n=N, means=_means(d, d + 1), Q=Q)[0]))
    if d >= 4:
        Q = _block_q(random_orthogonal(d // 2, d), random_orthogonal(d - d // 2, d + 1))
        out.append(("block diagonal", designed_statistic(d, u, n=N, Q=Q)[0]))
    sig = np.geomspace(1.0, 1e-7, d)
    sig = np.where((sig > 2.5e-7) & (sig < 4e-6), np.where(sig < 1e-6, 1e-7, 1e-5), sig)
    out.append(("sigma 1 .. 1e-7", designed_statistic(d, sig ** 2, n=N, seed=d)[0]))
    if d >= 2:
        e = u.copy()
        e[-1] = -1e-9 * u.max()
        out.append(("one eigenvalue -1e-9 lambda_max", designed_statistic(d, e, n=N, seed=d)[0]))
    return out


def _fp64_centred(S):
    """the centred Gram as the kernels form it in fp64"""
    d = S.shape[0] - 2
    n = S[d, d]
    m = S[:d, d] * (1.0 / n)
    return S[:d, :d] - (n * m)[:, None] * m[None, :]


@pytest.mark.parametrize("dims", [(1, 65), (65, 129)])
def test_eigenvalues_at_every_d(ctx, dims):
    worst = 0.0
    for d in range(*dims):
        for name, S in _eig_designs(d):
            ctx.gram_import(S)
            sing, rank, rows = ctx.solve_eigvals(cond=1e-6)
            lam_ref = np.sort(np.maximum(np.linalg.eigvalsh(_fp64_centred(S)), 0.0))[::-1]
            lmax = float(np.max(np.abs(np.linalg.eigvalsh(_fp64_centred(S)))))
            err = float(np.max(np.abs(sing ** 2 - lam_ref)))
            tol = 8 * d * EPS * lmax
            assert err <= tol, f"{name}: D = {d}: eigenvalue error {err:.3e} > {tol:.3e}"
            worst = max(worst, err / tol if tol > 0 else 0.0)
            assert rows == N, f"{name}: D = {d}"
            assert np.all(np.diff(sing) <= 0), f"{name}: D = {d}: not descending"
            assert rank == orc.fit_from_stats(S)["rank"], f"{name}: D = {d}: rank {rank}"
    print(f"\neigenvalues D in {dims}: worst error / bound {worst:.3g}")


# ------------------------------------------------------------------------------------------------
# minimum-norm kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,kappa", [(d, k) for d in (2, 3, 16, 33, 128) for k in (1.0, 1e4, 1e8) if (d, k) != (128, 1e8)]
                         + [pytest.param(128, 1e8, marks=pytest.mark.xfail(strict=True, reason=JACOBI_XFAIL))])
def test_minimum_norm_solution_matches_the_truncated_solution(ctx, d, kappa):
    worst = worst_null = 0.0
    for dropped in (0.0, 1e-14, -1e-9):
        for n_drop in sorted({1, d // 2, d - 1}):
            kept = d - n_drop
            eigs = np.r_[np.geomspace(1.0, 1.0 / kappa, kept), np.full(n_drop, dropped)]
            S, Q, e = designed_statistic(d, eigs, n=N, seed=d + n_drop, r_perp={d - 1: 0.5, kept - 1: 0.25})
            A, r, _, _ = exact_centred(S)
            ref, rank_ref = truncated_solution(Q, e, r)
            ctx.gram_import(S)
            coef, b0, sing, rank = ctx.solve_spectral(cond=1e-6)
            sing_e, rank_e, _ = ctx.solve_eigvals(cond=1e-6)
            label = f"D = {d}, kappa_kept {kappa:g}, {n_drop} x {dropped:g}"
            assert rank == rank_e == rank_ref == kept, f"{label}: rank {rank} / eigvals {rank_e} / ref {rank_ref}"
            assert np.max(np.abs(sing[:kept] ** 2 - sing_e[:kept] ** 2)) <= 8 * d * EPS, label
            null = float(np.max(sing[kept:] ** 2))
            null_tol = 2 * JACOBI_SWEEPS * d * EPS * float(np.linalg.norm(A.astype(np.float64)))
            assert null <= null_tol, f"{label}: dropped eigenvalue {null:.3e} > {null_tol:.3e}"
            worst_null = max(worst_null, null / null_tol)
            lmin = float(np.min(eigs[:kept]))
            tol = 8 * d * EPS * (1.0 / lmin) * float(np.max(np.abs(r))) / lmin
            err = float(np.max(np.abs(coef - ref.astype(np.float64))))
            assert err <= tol, f"{label}: coefficient error {err:.3e} > {tol:.3e}"
            assert b0 == 0.0
            worst = max(worst, err / tol)
    print(f"\nminimum norm D = {d}, kappa_kept {kappa:g}: worst error / bound {worst:.3g}, "
          f"dropped eigenvalue / bound {worst_null:.3g}")


# ------------------------------------------------------------------------------------------------
# power-of-two equivariance
# ------------------------------------------------------------------------------------------------
def _all_kernels(ctx, S):
    ctx.gram_import(S)
    c, b = ctx.solve()
    cs, bs, ss, rs = ctx.solve_spectral(cond=1e-6)
    se, re, _ = ctx.solve_eigvals(cond=1e-6)
    return c, b, cs, bs, ss, rs, se, re


@pytest.mark.parametrize("d", [1, 7, 16, 33, 128])
def test_power_of_two_scalings_are_exact(ctx, d):
    rng = np.random.RandomState(d)
    S, _, _ = designed_statistic(d, np.geomspace(1.0, 1e-4, d), n=N, means=_means(d, d), ybar=1.5, seed=d)
    base = _all_kernels(ctx, S)
    t = np.ones(d + 2)
    for k in (-60, -30, 30, 60):
        t[:d] = t[d + 1] = 2.0 ** k
        t[d] = 1.0
        c, b, cs, bs, ss, rs, se, re = _all_kernels(ctx, S * np.outer(t, t))
        for name, got, want in (("LDL^T coef", c, base[0]), ("spectral coef", cs, base[2])):
            assert np.array_equal(got, want), f"D = {d}, 2^{k}: {name} not bit-identical"
        assert b == base[1] * 2.0 ** k and bs == base[3] * 2.0 ** k, f"D = {d}, 2^{k}: intercept"
        assert np.array_equal(ss, base[4] * 2.0 ** k) and np.array_equal(se, base[6] * 2.0 ** k), f"D = {d}, 2^{k}"
        assert rs == base[5] and re == base[7]
    ks = rng.randint(-8, 9, d)
    ctx.gram_import(_col_scaled(S, ks))
    c, b = ctx.solve()
    assert np.array_equal(c, base[0] * np.exp2(-ks)), f"D = {d}: column scales"
    assert b == base[1]


# ------------------------------------------------------------------------------------------------
# edge statistics
# ------------------------------------------------------------------------------------------------
def _coef_tol(S):
    """forward-error bound of items above for the statistic S: (8 (D+1) eps + centring) kappa_kept ||r|| / lambda_min,kept"""
    d = S.shape[0] - 2
    A, r, m, _ = exact_centred(S)
    lam = np.linalg.eigvalsh(A.astype(np.float64))
    lmax = max(float(lam[-1]), 0.0)
    kept = lam[np.sqrt(np.maximum(lam, 0.0)) > 1e-6 * np.sqrt(lmax)]
    if kept.size == 0:
        return 0.0
    anorm = float(np.max(np.sum(np.abs(A.astype(np.float64)), axis=1)))
    eta = 8 * (d + 1) * EPS + 2 * EPS * S[d, d] * float(np.max(np.abs(m))) ** 2 / anorm
    return eta * (lmax / kept[0]) * float(np.max(np.abs(r))) / kept[0] * 4


def _with_simt(ctx, fn):
    ctx.set_kernel(b2.KERNEL_SIMT)
    try:
        return fn()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)


@pytest.mark.parametrize("d", [1, 2, 3])
def test_smallest_d_through_every_kernel_and_the_estimator(ctx, d):
    rng = np.random.RandomState(d)
    X = rng.randint(0, 100, (3000, d)).astype(np.float32)
    y = (X @ np.arange(1, d + 1) + rng.randint(-5, 6, 3000)).astype(np.float32)
    S = orc.gram_stats(X, y)
    fo = orc.fit_from_stats(S)
    c, b, cs, bs, ss, rs, se, re = _all_kernels(ctx, S)
    tol = _coef_tol(S)
    for got in (c, cs):
        assert np.max(np.abs(got - fo["coef"])) <= tol
    assert rs == re == fo["rank"] == d
    est = _with_simt(ctx, lambda: b2.B200LinearRegression(ctx=ctx).fit(X, y))
    assert np.array_equal(est.coef_, c) and est.intercept_ == b and est.rank_ == d
    assert np.array_equal(est.singular_, se)


def test_one_row(ctx):
    X = np.array([[3.0, -1.0, 7.0]], dtype=np.float32)
    y = np.array([2.5], dtype=np.float32)
    S = orc.gram_stats(X, y)
    ctx.gram_import(S)
    with pytest.raises(np.linalg.LinAlgError):
        ctx.solve()
    coef, b0, sing, rank = ctx.solve_spectral()
    assert np.all(coef == 0.0) and b0 == 2.5 and rank == 0
    sing_e, rank_e, rows = ctx.solve_eigvals()
    assert rank_e == 0 and rows == 1 and np.all(sing_e == 0.0)
    est = _with_simt(ctx, lambda: b2.B200LinearRegression(ctx=ctx).fit(X, y))
    from sklearn.linear_model import LinearRegression
    sk = LinearRegression().fit(X.astype(np.float64), y.astype(np.float64))
    assert np.all(est.coef_ == 0.0) and est.intercept_ == 2.5 and est.rank_ == sk.rank_ == 0
    assert est.singular_.shape == sk.singular_.shape == (1,)


def test_fewer_rows_than_features_gives_sklearns_minimum_norm_solution(ctx):
    from sklearn.linear_model import LinearRegression
    rng = np.random.RandomState(50)
    X = rng.standard_normal((50, 128)).astype(np.float32)
    y = rng.standard_normal(50).astype(np.float32)
    est = _with_simt(ctx, lambda: b2.B200LinearRegression(ctx=ctx).fit(X, y))
    sk = LinearRegression().fit(X.astype(np.float64), y.astype(np.float64))
    assert est.rank_ == sk.rank_ == 49
    assert est.singular_.shape == (50,)
    np.testing.assert_allclose(est.singular_[:49], sk.singular_[:49], rtol=1e-9)
    assert np.max(np.abs(est.coef_ - sk.coef_)) <= 1e-9 * np.max(np.abs(sk.coef_))
    assert abs(est.intercept_ - sk.intercept_) <= 1e-9 * max(1.0, abs(sk.intercept_))


@pytest.mark.parametrize("n_const", [1, 6])
def test_constant_columns(ctx, n_const):
    from sklearn.linear_model import LinearRegression
    rng = np.random.RandomState(n_const)
    X = rng.randint(0, 50, (4000, 6)).astype(np.float32)
    X[:, :n_const] = np.arange(1, n_const + 1) * 2021.0
    y = (X[:, n_const:].sum(axis=1) + 7 + rng.randint(-3, 4, 4000)).astype(np.float32)
    S = orc.gram_stats(X, y)
    ctx.gram_import(S)
    with pytest.raises(np.linalg.LinAlgError):
        ctx.solve()
    est = _with_simt(ctx, lambda: b2.B200LinearRegression(ctx=ctx).fit(X, y))
    sk = LinearRegression().fit(X.astype(np.float64), y.astype(np.float64))
    assert est.rank_ == sk.rank_ == 6 - n_const
    assert np.all(est.coef_[:n_const] == 0.0)
    assert np.max(np.abs(est.coef_ - sk.coef_)) <= 1e-9
    assert abs(est.intercept_ - sk.intercept_) <= 1e-7


def test_a_row_mask_that_keeps_no_rows_raises(ctx):
    X = np.random.RandomState(0).rand(1000, 4).astype(np.float32)
    y = X.sum(axis=1)
    with pytest.raises(ValueError, match="0 sample"):
        b2.B200LinearRegression(ctx=ctx).fit(X, y, row_mask=np.zeros(1000, np.uint8))
    with pytest.raises(ValueError, match="0 sample"):
        b2.B200LinearRegression(ctx=ctx).fit(ctx.to_device(X), ctx.to_device(y),
                                             row_mask=ctx.to_device(np.zeros(1000, np.uint8)))


# ------------------------------------------------------------------------------------------------
# one rank rule in the estimator
# ------------------------------------------------------------------------------------------------
def _row_statistics():
    rng = np.random.RandomState(11)
    X = rng.randint(0, 10, (20_000, 8)).astype(np.float32)
    y = (X @ np.arange(1, 9) + rng.randint(-5, 6, 20_000)).astype(np.float32)
    dup = X.copy()
    dup[:, 5] = dup[:, 4]
    return [("well conditioned", X, y), ("integer window", *integer_window_rows()), ("duplicate column", dup, y)]


def _attrs(est):
    return est.coef_.copy(), float(est.intercept_), int(est.rank_), est.singular_.copy()


def _same(a, b, label):
    assert np.array_equal(a[0], b[0]) and a[1] == b[1], f"{label}: coef_ / intercept_ differ"
    assert a[2] == b[2] and np.array_equal(a[3], b[3]), f"{label}: rank_ / singular_ differ"


def _check_against_oracle(S, got, label):
    fo = orc.fit_from_stats(S)
    assert got[2] == fo["rank"], f"{label}: rank_ {got[2]} vs {fo['rank']}"
    tol = _coef_tol(S)
    err = float(np.max(np.abs(got[0] - fo["coef"])))
    assert err <= tol, f"{label}: coef error {err:.3e} > {tol:.3e}"


@pytest.mark.parametrize("case", range(3))
def test_every_call_path_gives_one_model(ctx, case):
    label, X, y = _row_statistics()[case]
    d = X.shape[1]
    S = orc.gram_stats(X, y)
    if label == "integer window":
        A = exact_centred(S)[0]
        assert ldlt_pivots(A).min() > 1e-12 * float(np.max(np.diag(A.astype(np.float64))))
        assert orc.fit_from_stats(S)["rank"] == d - 1

    def run():
        out = {}
        e = b2.B200LinearRegression(ctx=ctx).fit(X, y)
        out["fit"] = _attrs(e)
        assert np.array_equal(ctx.gram_export(), S), f"{label}: the statistic of the rows is not exact"
        e = b2.B200LinearRegression(ctx=ctx).fit(X, y, with_spectrum=False)
        first = (e.coef_.copy(), float(e.intercept_))
        reg = e.to_sklearn()
        assert np.array_equal(e.coef_, first[0]) and e.intercept_ == first[1], f"{label}: to_sklearn moved coef_"
        assert np.array_equal(reg.coef_, first[0])
        out["deferred"] = _attrs(e)
        e = b2.B200LinearRegression(ctx=ctx).partial_fit(X, y)
        first = (e.coef_.copy(), float(e.intercept_))
        out["partial_fit"] = _attrs(e)
        e.to_sklearn()
        assert np.array_equal(e.coef_, first[0]) and e.intercept_ == first[1]
        ctx.gram_import(S)
        out["solve_resident"] = _attrs(b2.B200LinearRegression(ctx=ctx).solve_resident(d, S))
        return out
    out = _with_simt(ctx, run)
    for k, v in out.items():
        _same(out["fit"], v, f"{label}: fit vs {k}")
    _check_against_oracle(S, out["fit"], label)


def test_designed_window_and_indefinite_statistics_through_solve_resident(ctx):
    from test_oracle_solve import window_statistics
    cases = [(name, S) for name, S, _, _ in window_statistics()]
    e = np.r_[np.geomspace(1.0, 1e-3, 31), -1e-9]
    cases.append(("indefinite", designed_statistic(32, e, n=N, means=_means(32, 3), ybar=0.5, seed=32)[0]))
    for label, S in cases:
        d = S.shape[0] - 2
        ctx.gram_import(S)
        sing, rank, _ = ctx.solve_eigvals()
        est = b2.B200LinearRegression(ctx=ctx).solve_resident(d, S)
        got = (est.coef_.copy(), float(est.intercept_), int(est.rank_), est.singular_.copy())
        assert got[2] == rank == d - 1, f"{label}: rank_ {got[2]}, eigenvalue kernel {rank}"
        assert np.array_equal(got[3], sing)
        _check_against_oracle(S, got, label)
        est.to_sklearn()
        assert np.array_equal(est.coef_, got[0]) and est.intercept_ == got[1]
