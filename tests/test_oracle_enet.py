"""The numpy statement of b2_solve_enet_path (tests/enet_oracle.py) pinned to scikit-learn 1.9 on the CPU: its Gram
coordinate descent fed with Q, q and ||yc||^2 taken only from the raw sums of S must reproduce sklearn's
enet_path(precompute=Q, Xy=q), ElasticNet(precompute=True) and Lasso(precompute=True): coefficients, dual gaps, sweep
counts and the alpha grid."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import ElasticNet, Lasso, enet_path
from sklearn.linear_model._coordinate_descent import _alpha_grid

from enet_oracle import alpha_grid, enet_path_from_stats, gram_inputs, kkt_violation


def _rows(n, d, seed, offset=50.0, corr=0.3, sparse_beta=True):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    if corr and d > 1:
        X[:, 1:] = corr * X[:, :1] + (1 - corr) * X[:, 1:]
    X = (X + offset).astype(np.float32).astype(np.float64)
    beta = rng.uniform(-2, 2, d)
    if sparse_beta:
        beta[rng.uniform(size=d) < 0.5] = 0.0
    y = (X @ beta + rng.standard_normal(n)).astype(np.float32).astype(np.float64)
    return X, y


def _stat(X, y):
    A = np.column_stack([X, np.ones(X.shape[0]), y])
    return A.T @ A


def _sk_path(X, y, S, fit_intercept=True, **kw):
    """sklearn's Gram path on Q, q from S; y centred as the rows are (its y.y only sets the gap tolerance)."""
    Q, q, _, _, ybar, _, _ = gram_inputs(S, fit_intercept)
    Xc = X - X.mean(0) if fit_intercept else X
    yc = y - ybar if fit_intercept else y
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return enet_path(np.asfortranarray(Xc), yc, precompute=Q, Xy=q, return_n_iter=True, **kw)


def _close(o, sk, rtol=1e-8):
    alphas, coefs, gaps, iters = sk
    scale = max(float(np.max(np.abs(coefs))), 1e-12)
    np.testing.assert_allclose(o["alphas"], alphas, rtol=1e-14)
    assert float(np.max(np.abs(o["coefs"].T - coefs))) <= rtol * scale
    np.testing.assert_allclose(o["gaps"], gaps, rtol=1e-5, atol=1e-12 * max(1.0, float(np.max(np.abs(gaps)))))
    assert list(o["n_iter"]) == list(iters)


def test_alpha_grid_matches_sklearn():
    X, y = _rows(2000, 12, 1)
    S = _stat(X, y)
    Q, q, _, _, _, n, _ = gram_inputs(S)
    for l1_ratio in (1.0, 0.5, 0.1):
        for positive in (False, True):
            for eps, k in ((1e-3, 100), (1e-2, 7), (1e-3, 1)):
                ours = alpha_grid(q, n, l1_ratio, eps, k, positive)
                ref = _alpha_grid(np.zeros((int(n), 12)), np.zeros(int(n)), Xy=q, l1_ratio=l1_ratio, eps=eps,
                                  n_alphas=k, positive=positive)
                assert np.array_equal(ours, ref)
    assert np.array_equal(alpha_grid(np.zeros(3), 10.0, 1.0, 1e-3, 4), np.full(4, np.finfo(np.float64).resolution))


@pytest.mark.parametrize("l1_ratio", [1.0, 0.5, 0.1])
@pytest.mark.parametrize("positive", [False, True])
def test_path_matches_sklearn(l1_ratio, positive):
    X, y = _rows(3000, 16, 2)
    S = _stat(X, y)
    o = enet_path_from_stats(S, l1_ratio, n_alphas=30, positive=positive)
    _close(o, _sk_path(X, y, S, l1_ratio=l1_ratio, alphas=30, positive=positive))


def test_tight_tolerance_and_kkt():
    X, y = _rows(3000, 10, 3, corr=0.8)
    S = _stat(X, y)
    o = enet_path_from_stats(S, 0.5, n_alphas=12, tol=1e-10)
    _close(o, _sk_path(X, y, S, l1_ratio=0.5, alphas=12, tol=1e-10))
    for a, w in zip(o["alphas"], o["coefs"]):
        assert kkt_violation(S, w, a, 0.5) <= 1e-6


def test_without_intercept():
    X, y = _rows(2500, 8, 4, offset=3.0)
    S = _stat(X, y)
    o = enet_path_from_stats(S, 0.7, n_alphas=20, fit_intercept=False)
    _close(o, _sk_path(X, y, S, fit_intercept=False, l1_ratio=0.7, alphas=20))
    assert np.all(o["intercepts"] == 0.0)


def test_alpha_above_alpha_max_is_all_zero_in_zero_sweeps():
    X, y = _rows(1000, 6, 5)
    S = _stat(X, y)
    amax = alpha_grid(gram_inputs(S)[1], 1000.0, 1.0, n_alphas=1)[0]
    o = enet_path_from_stats(S, 1.0, alphas=[amax * 1.5, amax])
    assert np.all(o["coefs"] == 0.0) and list(o["n_iter"]) == [0, 0]
    assert np.allclose(o["intercepts"], y.mean(), rtol=1e-12)
    _close(o, _sk_path(X, y, S, l1_ratio=1.0, alphas=[amax * 1.5, amax]))


def test_max_iter_reached():
    X, y = _rows(2000, 20, 6, corr=0.95)
    S = _stat(X, y)
    o = enet_path_from_stats(S, 0.5, alphas=[0.01, 0.001], max_iter=3, tol=1e-12)
    assert list(o["n_iter"]) == [3, 3] and np.all(o["gaps"] > o["tol"])
    _close(o, _sk_path(X, y, S, l1_ratio=0.5, alphas=[0.01, 0.001], max_iter=3, tol=1e-12))


def test_warm_start_from_coef_init():
    X, y = _rows(2000, 9, 7)
    S = _stat(X, y)
    init = np.linspace(-1, 1, 9)
    o = enet_path_from_stats(S, 0.9, alphas=[0.05, 0.02], coef_init=init)
    _close(o, _sk_path(X, y, S, l1_ratio=0.9, alphas=[0.05, 0.02], coef_init=init))


def test_one_feature():
    X, y = _rows(500, 1, 8, sparse_beta=False)
    S = _stat(X, y)
    for l1_ratio in (1.0, 0.3):
        o = enet_path_from_stats(S, l1_ratio, n_alphas=10)
        _close(o, _sk_path(X, y, S, l1_ratio=l1_ratio, alphas=10))


def test_constant_column_gets_zero():
    X, y = _rows(1500, 5, 9)
    X[:, 2] = 37.25
    S = _stat(X, y)
    Q, q, _, _, _, _, live = gram_inputs(S)
    assert list(live) == [True, True, False, True, True]
    o = enet_path_from_stats(S, 0.5, n_alphas=15)
    assert np.all(o["coefs"][:, 2] == 0.0)
    keep = [0, 1, 3, 4]
    ref = enet_path_from_stats(_stat(X[:, keep], y), 0.5, n_alphas=15)
    np.testing.assert_allclose(o["alphas"], ref["alphas"], rtol=1e-14)
    assert float(np.max(np.abs(o["coefs"][:, keep] - ref["coefs"]))) <= 1e-10 * float(np.max(np.abs(ref["coefs"])))


@pytest.mark.parametrize("cls,l1_ratio", [(Lasso, 1.0), (ElasticNet, 0.5), (ElasticNet, 0.1)])
def test_estimators_match_one_alpha_paths(cls, l1_ratio):
    X, y = _rows(4000, 12, 10)
    S = _stat(X, y)
    for alpha in (0.5, 0.05):
        kw = {} if cls is Lasso else {"l1_ratio": l1_ratio}
        sk = cls(alpha=alpha, precompute=True, **kw).fit(X, y)
        o = enet_path_from_stats(S, l1_ratio, alphas=[alpha])
        scale = float(np.max(np.abs(sk.coef_)))
        assert float(np.max(np.abs(o["coefs"][0] - sk.coef_))) <= 1e-8 * scale
        assert o["n_iter"][0] == sk.n_iter_
        assert o["gaps"][0] == pytest.approx(sk.dual_gap_, rel=1e-4, abs=1e-12)
        assert o["intercepts"][0] == pytest.approx(sk.intercept_, rel=1e-9)
