"""The numpy leave-one-out oracle (tests/loo_oracle.py) pinned to scikit-learn's RidgeCV(store_cv_results=True), cv=None.

The oracle states what b2_ridge_loo computes; this module shows it is what RidgeCV computes, on CPU only.  Tolerances and
the worst case measured (numpy / scikit-learn 1.9, x86-64):
  * alpha_: equal, on every table.
  * best_score_ = -mse[best]: relative 1e-12 (worst 3.5e-14, the offset table without an intercept).
  * cv_results_: max |difference| / max |cv| below 1e-9 with an intercept (worst 1.8e-12, D = 40 correlated) and 1e-8
    without (worst 3.0e-10, columns offset by 100: sklearn's SVD of the uncentred rows is the less accurate side).
The grid longer than 64 alphas runs through ``estimator.merge_alpha_chunks``, the estimator's own merge of the chunks
b2_ridge_loo is called on.
"""
import importlib

import numpy as np
import pytest
from sklearn.linear_model import RidgeCV

from loo_oracle import ridge_loo

merge_alpha_chunks = importlib.import_module("bodywork_mlops_demo_b200.estimator").merge_alpha_chunks


def table(n, d, seed, offset=0.0, corr=0.0):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    if corr:
        X[:, 1:] = corr * X[:, :1] + (1 - corr) * X[:, 1:]
    X = X + offset
    y = X @ rng.uniform(-1, 1, d) + rng.standard_normal(n)
    return X, y


ALPHAS = [0.01, 0.1, 1.0, 10.0, 100.0]


def check(X, y, alphas, fit_intercept, mask=None):
    mse, cv, best = ridge_loo(X, y, alphas, mask=mask, fit_intercept=fit_intercept)
    Xs, ys = (X, y) if mask is None else (X[mask == 1], y[mask == 1])
    sk = RidgeCV(alphas=alphas, fit_intercept=fit_intercept, store_cv_results=True).fit(Xs, ys)
    assert alphas[best] == sk.alpha_
    assert -mse[best] == pytest.approx(sk.best_score_, rel=1e-12)
    tol = 1e-9 if fit_intercept else 1e-8
    assert np.max(np.abs(cv - sk.cv_results_)) <= tol * np.max(np.abs(sk.cv_results_))
    return mse, cv, best


@pytest.mark.parametrize("fit_intercept", [True, False])
@pytest.mark.parametrize("n,d,offset,corr", [(500, 8, 0.0, 0.0), (2000, 1, 5.0, 0.0), (300, 40, 3.0, 0.9),
                                             (400, 8, 100.0, 0.5)])
def test_oracle_matches_ridgecv(n, d, offset, corr, fit_intercept):
    X, y = table(n, d, n + d, offset, corr)
    check(X, y, ALPHAS, fit_intercept)


@pytest.mark.parametrize("fit_intercept", [True, False])
def test_masked_subset(fit_intercept):
    X, y = table(700, 8, 3, 2.0, 0.3)
    mask = (np.random.RandomState(4).uniform(size=700) < 0.6).astype(np.uint8)
    X[mask == 0] = np.nan                      # dropped rows never reach the arithmetic
    mse, cv, _ = check(X, y, ALPHAS, fit_intercept, mask=mask)
    assert cv.shape == (int(mask.sum()), len(ALPHAS)) and np.all(np.isfinite(mse))


def test_rank_deficient_with_alpha():
    X, y = table(400, 6, 5)
    X = np.hstack([X, X[:, :2], np.zeros((400, 1))])   # two repeated columns and a zero column
    check(X, y, ALPHAS, True)


def test_tie_goes_to_the_lowest_index():
    X, y = table(300, 4, 6)
    alphas = [5.0, 1.0, 1.0, 50.0]
    mse, _, best = ridge_loo(X, y, alphas)
    assert mse[1] == mse[2]
    sk = RidgeCV(alphas=alphas).fit(X, y)
    assert sk.alpha_ == 1.0 and best == 1


def test_grid_longer_than_one_call_merges_by_first_minimum():
    X, y = table(600, 12, 7, 1.0, 0.6)
    grid = np.logspace(-3, 4, 100)
    chunks = [(off, ridge_loo(X, y, grid[off: off + 64])[0]) for off in range(0, grid.size, 64)]
    best = merge_alpha_chunks(chunks)
    sk = RidgeCV(alphas=grid).fit(X, y)
    assert grid[best] == sk.alpha_
    assert best == ridge_loo(X, y, grid)[2]
    tied = [(0, np.array([3.0, 2.0])), (2, np.array([2.0, 5.0]))]
    assert merge_alpha_chunks(tied) == 1
