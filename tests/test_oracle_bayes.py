"""The numpy statement of BayesianRidge / ARDRegression from (S, anchor) (tests/bayes_oracle.py) pinned to scikit-learn 1.9
on float64 rows; CPU only."""
import numpy as np
import pytest
from sklearn.linear_model import ARDRegression, BayesianRidge

import bayes_oracle as bo


def rows(n, d, seed, offset=3.0, noise=0.5, zero_cols=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)) * rng.uniform(0.5, 2.0, size=d) + offset
    w = rng.normal(size=d)
    if zero_cols:
        w[:zero_cols] = 0.0
    y = X @ w + 1.5 + noise * rng.normal(size=n)
    return X, y


def stat(X, y):
    Z = np.column_stack([X, np.ones(len(X)), y])
    return Z.T @ Z


def anchor(X, y, fit_intercept):
    if fit_intercept:
        w0 = np.linalg.lstsq(X - X.mean(0), y - y.mean(), rcond=None)[0]
    else:
        w0 = np.linalg.lstsq(X, y, rcond=None)[0]
    return bo.anchor_of(X, y, w0, fit_intercept)


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def check(res, sk, tol=1e-9):
    assert res["n_iter"] == sk.n_iter_
    assert rel(res["alpha"], sk.alpha_) < tol
    assert rel(res["lambda"], sk.lambda_) < tol
    assert rel(res["coef"], sk.coef_) < tol
    assert abs(res["intercept"] - sk.intercept_) <= tol * max(1.0, abs(sk.intercept_))
    if res["scores"] is not None:      # a sum of large terms of both signs
        assert rel(res["scores"], sk.scores_) < max(tol, 1e-8)


CASES = [dict(n=400, d=1), dict(n=500, d=8), dict(n=600, d=40), dict(n=30, d=40)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"n{c['n']}_d{c['d']}")
@pytest.mark.parametrize("fit_intercept", [True, False])
@pytest.mark.parametrize("compute_score", [False, True])
def test_bayes_ridge_matches_sklearn(case, fit_intercept, compute_score):
    X, y = rows(case["n"], case["d"], seed=case["d"] + 7)
    sk = BayesianRidge(fit_intercept=fit_intercept, compute_score=compute_score).fit(X, y)
    res = bo.bayes_ridge(stat(X, y), fit_intercept=fit_intercept, compute_score=compute_score,
                         anchor=anchor(X, y, fit_intercept))
    # n < d: the fit interpolates, sse is rounding noise of ||y||^2 in either computation
    tol = 1e-9 if case["n"] > case["d"] else 1e-5
    check(res, sk, tol)
    assert rel(res["sigma"], sk.sigma_) < max(tol, 1e-8)


def test_bayes_ridge_inits_and_max_iter():
    X, y = rows(300, 8, seed=3)
    kw = dict(alpha_init=2.0, lambda_init=0.1, max_iter=2, compute_score=True)
    sk = BayesianRidge(**kw).fit(X, y)
    res = bo.bayes_ridge(stat(X, y), anchor=anchor(X, y, True), **kw)
    assert sk.n_iter_ == 2
    check(res, sk)


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"n{c['n']}_d{c['d']}")
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_ard_matches_sklearn(case, fit_intercept):
    X, y = rows(case["n"], case["d"], seed=case["d"] + 11, zero_cols=case["d"] // 2)
    sk = ARDRegression(fit_intercept=fit_intercept, compute_score=True).fit(X, y)
    res = bo.ard(stat(X, y), fit_intercept=fit_intercept, compute_score=True, anchor=anchor(X, y, fit_intercept))
    tol = 1e-9 if case["n"] > case["d"] else 1e-6      # n < d: sklearn's Woodbury branch inverts another matrix
    check(res, sk, tol)
    keep = sk.lambda_ < sk.threshold_lambda
    assert rel(res["sigma"][np.ix_(keep, keep)], sk.sigma_) < 1e-6


def test_ard_prunes_features_and_all_of_them():
    X, y = rows(500, 8, seed=5, zero_cols=5)
    sk = ARDRegression(compute_score=True).fit(X, y)
    assert 0 < np.sum(sk.lambda_ >= sk.threshold_lambda) < 8
    check(bo.ard(stat(X, y), compute_score=True, anchor=anchor(X, y, True)), sk)
    sk0 = ARDRegression(threshold_lambda=1e-12).fit(X, y)
    res0 = bo.ard(stat(X, y), threshold_lambda=1e-12, anchor=anchor(X, y, True))
    assert sk0.sigma_.shape == (0, 0) and not np.any(res0["sigma"])
    check(res0, sk0)


def test_constant_column_and_constant_y():
    X, y = rows(300, 6, seed=9)
    X[:, 2] = 4.0
    for est, fn in ((BayesianRidge(), bo.bayes_ridge), (ARDRegression(), bo.ard)):
        sk = est.fit(X, y)
        check(fn(stat(X, y), anchor=anchor(X, y, True)), sk, 1e-7)
    yc = np.full(300, 2.5)
    sk = BayesianRidge().fit(X[:, [0, 1]], yc)
    res = bo.bayes_ridge(stat(X[:, [0, 1]], yc), anchor=anchor(X[:, [0, 1]], yc, True))
    assert res["n_iter"] == sk.n_iter_
    assert np.allclose(res["coef"], sk.coef_, atol=1e-12) and abs(res["intercept"] - 2.5) < 1e-12


def test_std_matches_sklearn():
    X, y = rows(400, 8, seed=1, zero_cols=4)
    for est in (BayesianRidge(), ARDRegression()):
        sk = est.fit(X, y)
        keep = getattr(sk, "lambda_", None)
        sigma = sk.sigma_
        if isinstance(sk, ARDRegression):
            keep = sk.lambda_ < sk.threshold_lambda
            sigma = np.zeros((8, 8))
            sigma[np.ix_(keep, keep)] = sk.sigma_
        ym, ys = sk.predict(X[:50], return_std=True)
        yh, yst = bo.score_std(X[:50], sk.X_offset_, sigma, 1.0 / sk.alpha_, sk.coef_, sk.intercept_)
        assert np.allclose(yh, ym, rtol=1e-12) and np.allclose(yst, ys, rtol=1e-12)


def test_anchored_sse_is_the_row_sse_and_s_alone_misses():
    """The anchor identity is exact; from S alone, with the Gram part of S perturbed by 3e-6 (the tensor-core paths'
    accuracy) on a table with ||yc||^2 / sse ~ 200, alpha_ misses by more than 1e-5, and anchored it does not."""
    rng = np.random.default_rng(0)
    n, d = 200_000, 32
    X = rng.normal(size=(n, d)) * 10
    y = X @ rng.normal(size=d) + 4.0 * rng.normal(size=n)
    S = stat(X, y)
    an = anchor(X, y, True)
    w = an[:d] + 1e-3 * rng.normal(size=d)
    A, r, m, ybar, nn, yy, _ = bo.normal_equations(S, True)
    e = (y - y.mean()) - (X - X.mean(0)) @ w
    assert abs(bo._sse(A, r, yy, nn, w, an, True) - e @ e) <= 1e-9 * (e @ e)
    sk = BayesianRidge().fit(X, y)
    P = 1 + 3e-6 * rng.uniform(-1, 1, size=S.shape)
    P[d:, d:] = 1.0                         # n, sum y and sum y^2 exact; the Gram block and X^T y perturbed
    Sp = S * (P + P.T) / 2
    alone = bo.bayes_ridge(Sp)
    anchored = bo.bayes_ridge(Sp, anchor=an)
    assert rel(alone["alpha"], sk.alpha_) > 1e-5
    assert rel(anchored["alpha"], sk.alpha_) < 1e-6
