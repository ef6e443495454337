"""The numpy multi-target leave-one-out oracle (tests/loo_classes_oracle.py) pinned to scikit-learn's
RidgeClassifierCV(store_cv_results=True), cv=None, on CPU only: cv_results_, best_score_, alpha_ and the coefficients
within 1e-12 relative, for K in {2, 3, 7, 32}, both intercept modes, masks and both scorings."""
import numpy as np
import pytest
from sklearn.linear_model import RidgeClassifierCV

from loo_classes_oracle import ridge_classifier_loo

ALPHAS = [0.03, 0.3, 3.0, 30.0, 300.0]


def table(n, d, n_classes, seed, offset=0.0):
    """rows and class indices of a noisy linear argmax, every class present"""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)) + offset
    k = np.argmax(X @ rng.normal(size=(d, n_classes)) + rng.normal(0.0, 1.5, size=(n, n_classes)), axis=1)
    k[:n_classes] = np.arange(n_classes)
    return X, k


def rel(a, b):
    return np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300)


def check(X, k, n_classes, fit_intercept, scoring, mask=None, alphas=ALPHAS):
    o = ridge_classifier_loo(X, k, n_classes, alphas, mask=mask, fit_intercept=fit_intercept, scoring=scoring)
    Xs, ks = (X, k) if mask is None else (X[mask == 1], k[mask == 1])
    sk = RidgeClassifierCV(alphas=alphas, fit_intercept=fit_intercept, scoring=scoring,
                           store_cv_results=True).fit(Xs, ks)
    assert alphas[o["best"]] == sk.alpha_
    n = Xs.shape[0]
    score = o["correct"][o["best"]] / n if scoring == "accuracy" else -o["mse"][o["best"]]
    assert score == pytest.approx(sk.best_score_, rel=1e-12)
    assert o["cv"].shape == sk.cv_results_.shape
    assert rel(o["cv"], sk.cv_results_) <= 1e-12
    coef = o["coef"][0] if n_classes == 2 else o["coef"]
    assert coef.shape == sk.coef_.shape
    assert rel(coef, sk.coef_) <= 1e-12
    if fit_intercept:
        assert rel(o["intercept"], sk.intercept_) <= 1e-12
    return o, sk


@pytest.mark.parametrize("scoring", [None, "accuracy"])
@pytest.mark.parametrize("fit_intercept", [True, False])
@pytest.mark.parametrize("n_classes", [2, 3, 7, 32])
def test_oracle_matches_ridge_classifier_cv(n_classes, fit_intercept, scoring):
    X, k = table(30 * n_classes + 200, 9, n_classes, seed=n_classes, offset=0.5)
    check(X, k, n_classes, fit_intercept, scoring)


@pytest.mark.parametrize("scoring", [None, "accuracy"])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_masked_subset(fit_intercept, scoring):
    X, k = table(800, 6, 4, seed=5, offset=1.0)
    mask = (np.random.default_rng(6).uniform(size=800) < 0.6).astype(np.uint8)
    mask[:4] = 1                                     # every class kept
    X[mask == 0] = np.nan                            # dropped rows never reach the arithmetic
    o, _ = check(X, k, 4, fit_intercept, scoring, mask=mask)
    assert o["cv"].shape == (int(mask.sum()), 4, len(ALPHAS))


def test_two_classes_accuracy_scores_every_alpha_one_and_picks_the_first():
    X, k = table(300, 5, 2, seed=7)
    o, sk = check(X, k, 2, True, "accuracy", alphas=[10.0, 0.1, 1.0])
    assert np.all(o["correct"] == 300) and o["best"] == 0 and sk.best_score_ == 1.0 and sk.alpha_ == 10.0


def test_two_classes_is_the_single_target_ridge_loo():
    """T = 1: the error of the +-1 target of class 1 is RidgeCV's on y = +-1"""
    from loo_oracle import ridge_loo
    X, k = table(400, 6, 2, seed=8)
    o = ridge_classifier_loo(X, k, 2, ALPHAS)
    mse, cv, best = ridge_loo(X, np.where(k == 1, 1.0, -1.0), ALPHAS)
    assert best == o["best"] and rel(o["mse"], mse) <= 1e-13 and rel(o["cv"][:, 0, :], cv) <= 1e-12
