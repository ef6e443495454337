"""The numpy restatement of the refined fit (tests/refine_oracle.py) against scikit-learn: from a perturbed statistic
it converges to the least-squares solution of the rows, with no passes it is the plain solve of that statistic, and
when the perturbation is beyond what the passes can correct the guard stops them no worse than where they started."""
import numpy as np
from sklearn.linear_model import LinearRegression, Ridge

from oracle import ols_oracle as orc
from refine_oracle import refine_fit


def _perturbed(S, rel, seed):
    """S with symmetric relative noise of size `rel` on every entry except the row count"""
    d = S.shape[0] - 2
    E = np.random.RandomState(seed).standard_normal(S.shape)
    E = 0.5 * (E + E.T)
    Sp = S * (1.0 + rel * E)
    Sp[d, d] = S[d, d]
    return Sp


def _table(n=20_000, d=16, rho=0.99, seed=0):
    X, y, _ = orc.column_table(n, d, "correlated", seed=seed, rho=rho)
    return X + 0.5, y                                         # a non-zero shift m


def test_refined_fit_converges_to_sklearn_from_a_perturbed_statistic():
    X, y = _table()
    S = orc.gram_stats(X, y)
    kappa = orc.centred_condition(S)
    sk = LinearRegression().fit(X, y)
    start = orc.fit_from_stats(_perturbed(S, 1e-5, 1))
    err0 = orc.coef_error(start["coef"], sk.coef_, S)
    out = refine_fit(X, y, _perturbed(S, 1e-5, 1), max_passes=8, tol=1e-12)
    err = orc.coef_error(out["coef"], sk.coef_, S)
    assert kappa > 500 and err0 > 1e-4, (kappa, err0)         # the perturbation alone breaks the 1e-4 contract
    assert err < 1e-9 and abs(out["intercept"] - sk.intercept_) < 1e-7, (err, out["intercept"] - sk.intercept_)
    assert out["passes"] <= 6 and out["step"] <= 1e-12, out["steps"]
    assert all(b < a for a, b in zip(out["steps"], out["steps"][1:]))


def test_ridge_and_no_intercept_converge_to_their_own_problems():
    X, y = _table(d=8, seed=3)
    S = orc.gram_stats(X, y)
    out = refine_fit(X, y, _perturbed(S, 1e-6, 2), alpha=5.0, max_passes=8, tol=1e-13)
    rd = Ridge(alpha=5.0).fit(X, y)
    assert orc.coef_error(out["coef"], rd.coef_, S) < 1e-9 and abs(out["intercept"] - rd.intercept_) < 1e-7
    out0 = refine_fit(X, y, _perturbed(S, 1e-6, 2), fit_intercept=False, max_passes=8, tol=1e-13)
    ls = np.linalg.lstsq(X, y, rcond=None)[0]
    assert orc.coef_error(out0["coef"], ls, S) < 1e-9 and out0["intercept"] == 0.0


def test_no_passes_is_the_plain_solve_of_the_statistic():
    X, y = _table(d=8, seed=4)
    Sp = _perturbed(orc.gram_stats(X, y), 1e-5, 3)
    out = refine_fit(X, y, Sp, max_passes=0)
    base = orc.fit_from_stats(Sp)
    assert np.array_equal(out["coef"], base["coef"]) and out["intercept"] == base["intercept"]
    assert out["passes"] == 0 and out["step"] == 0.0


def test_the_guard_stops_a_diverging_refinement_no_worse_than_the_start():
    X, y = _table(rho=0.999, seed=5)
    S = orc.gram_stats(X, y)
    sk = LinearRegression().fit(X, y)
    Sp = _perturbed(S, 3e-3, 6)                               # kappa ~ 8e3 x 3e-3: the passes cannot contract
    start = orc.fit_from_stats(Sp)
    out = refine_fit(X, y, Sp, max_passes=16)
    err0 = orc.coef_error(start["coef"], sk.coef_, S)
    err = orc.coef_error(out["coef"], sk.coef_, S)
    assert len(out["steps"]) < 16 and out["steps"][-1] > out["steps"][-2], out["steps"]   # the guard fired
    assert err <= err0 * (1 + 1e-12), (err, err0)
