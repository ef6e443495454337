"""The designed statistics and references of tests/solve_oracle.py, checked on the CPU: the statistic has the spectrum
it was designed with, the longdouble references are as accurate as they claim, the fp64 oracle agrees with the
truncated (sklearn) solution, and the statistics the GPU tests use to separate the LDL^T pivot test from the rank rule
really lie between the two."""
import numpy as np
import pytest
from sklearn.linear_model import LinearRegression

from oracle import ols_oracle as orc
from solve_oracle import (EPS, backward_error, designed_statistic, exact_centred, integer_window_rows, ldlt_pivots,
                          refined_solve, truncated_solution)

PIVOT_TEST = 1e-12             # the LDL^T kernel refuses a pivot <= 1e-12 * max diag


def window_statistics():
    """(name, S, Q, eigs) of the designed statistics whose LDL^T pivots pass the kernel's test while sklearn's rule
    (sigma > 1e-6 sigma_max, i.e. lambda > 1e-12 lambda_max) drops one direction."""
    out = []
    for d, seed in ((16, 3), (128, 0)):
        eigs = np.ones(d)
        eigs[-1] = 2e-13
        S, Q, e = designed_statistic(d, eigs, seed=seed)
        out.append((f"d{d}", S, Q, e))
    c = np.sqrt(0.5)
    S, Q, e = designed_statistic(2, [1.0, 5e-13], Q=np.array([[c, -c], [c, c]]), seed=2)   # 1 - rho = 1e-12
    out.append(("d2", S, Q, e))
    return out


@pytest.mark.parametrize("d", [1, 2, 16, 33, 128])
def test_designed_statistic_has_the_requested_spectrum(d):
    rng = np.random.RandomState(d)
    for eigs in (rng.uniform(1, 2, d), np.geomspace(1, 1e-11, d), np.r_[np.ones(d - 1), -1e-9][-d:]):
        S, Q, e = designed_statistic(d, eigs, seed=d)
        lam = np.linalg.eigvalsh(S[:d, :d])
        assert np.max(np.abs(lam - np.sort(eigs))) <= d * EPS * np.max(np.abs(eigs))
        assert S[d, d] == 1024 and np.array_equal(S, S.T)
    means = rng.randint(-4, 5, d) / 8.0
    S, Q, e = designed_statistic(d, rng.uniform(1, 2, d), means=means, ybar=1.5, beta=np.ones(d), seed=d)
    A, r, m, ybar = exact_centred(S)
    assert np.array_equal(m.astype(np.float64), means) and float(ybar) == 1.5
    assert np.max(np.abs(A.astype(np.float64) - (Q * e) @ Q.T)) <= 4 * EPS * (2 + 1024 * 0.25)


def test_zero_means_leave_the_gram_exact():
    d = 40
    S, Q, eigs = designed_statistic(d, np.geomspace(1, 1e-6, d), seed=5)
    A, r, _, _ = exact_centred(S)
    assert np.array_equal(A.astype(np.float64), S[:d, :d])


@pytest.mark.parametrize("kappa", [1.0, 1e6, 1e11])
@pytest.mark.parametrize("d", [2, 37, 128])
def test_refined_solve_reaches_longdouble_accuracy(d, kappa):
    S, Q, eigs = designed_statistic(d, np.geomspace(1, 1 / kappa, d), seed=d + 1)
    A, r, _, _ = exact_centred(S)
    beta = refined_solve(A, r)
    assert backward_error(A, r, beta) < 1e-18
    plain = np.linalg.solve(A.astype(np.float64), r.astype(np.float64))
    assert backward_error(A, r, plain) > 1e-18                 # the fp64 solve alone cannot: the bound is not vacuous


@pytest.mark.parametrize("kappa_kept", [1.0, 1e4, 1e8])
@pytest.mark.parametrize("dropped", [0.0, 1e-14, -1e-9])
@pytest.mark.parametrize("d", [2, 16, 128])
def test_oracle_fit_is_the_truncated_solution(d, kappa_kept, dropped):
    for n_drop in sorted({1, d // 2, d - 1}):
        eigs = np.r_[np.geomspace(1, 1 / kappa_kept, d - n_drop), np.full(n_drop, dropped)]
        S, Q, e = designed_statistic(d, eigs, seed=d + n_drop, r_perp={d - 1: 0.3})
        A, r, _, _ = exact_centred(S)
        ref, rank = truncated_solution(Q, e, r)
        fo = orc.fit_from_stats(S)
        assert fo["rank"] == rank == d - n_drop
        bound = 8 * d * EPS * kappa_kept * float(np.max(np.abs(r))) * kappa_kept
        err = float(np.max(np.abs(fo["coef"] - ref.astype(np.float64))))
        assert err <= bound, f"d={d} dropped {n_drop} x {dropped}: {err:.3e} > {bound:.3e}"


@pytest.mark.parametrize("case", range(3))
def test_designed_window_passes_the_pivot_test_and_has_rank_d_minus_1(case):
    name, S, Q, eigs = window_statistics()[case]
    d = S.shape[0] - 2
    A, r, _, _ = exact_centred(S)
    piv = ldlt_pivots(A)
    assert piv.min() > 1.2 * PIVOT_TEST * np.max(np.diag(A.astype(np.float64))), name
    fo = orc.fit_from_stats(S)
    assert fo["rank"] == d - 1, name
    full = np.linalg.solve(A.astype(np.float64), r.astype(np.float64))
    assert np.max(np.abs(full - fo["coef"])) > 1e-3, name   # the two rules give different models


def test_integer_rows_lie_in_the_window():
    X, y = integer_window_rows()
    S = orc.gram_stats(X, y)
    A, r, _, _ = exact_centred(S)
    piv = ldlt_pivots(A)
    assert piv.min() > 2 * PIVOT_TEST * np.max(np.diag(A.astype(np.float64)))
    fo = orc.fit_from_stats(S)
    sk = LinearRegression().fit(X.astype(np.float64), y.astype(np.float64))
    assert fo["rank"] == sk.rank_ == 1
    np.testing.assert_allclose(fo["coef"], [0.25, 0.25], atol=1e-3)
    np.testing.assert_allclose(fo["coef"], sk.coef_, rtol=1e-9)
    full = np.linalg.solve(A.astype(np.float64), r.astype(np.float64))
    assert abs(full[0] - full[1]) > 10                      # the full solve of the same statistic
