"""The numpy statement of b2_gram_folds + b2_solve_enet_cv (tests/enet_cv_oracle.py) pinned to scikit-learn 1.9's
LassoCV / ElasticNetCV(precompute=True) on the CPU -- the fold statistics, the paths of the summed other folds, the
held-out error from each fold's own statistic and the choice of (alpha, l1_ratio) -- and fold_ids against sklearn's
splits."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import ElasticNetCV, LassoCV
from sklearn.model_selection import KFold, RepeatedKFold, ShuffleSplit

import bodywork_mlops_demo_b200 as b2
from enet_cv_oracle import choose, enet_cv_from_stats, fold_stats, fold_sum, heldout_mse, stat
from enet_oracle import enet_path_from_stats


def _rows(n, d, seed, offset=0.5, corr=0.3):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    X[:, 1:] = corr * X[:, :1] + (1 - corr) * X[:, 1:]
    X = (X + offset).astype(np.float32).astype(np.float64)
    beta = rng.uniform(-2, 2, d)
    beta[rng.uniform(size=d) < 0.5] = 0.0
    y = (X @ beta + rng.standard_normal(n)).astype(np.float32).astype(np.float64)
    return X, y


def _sk(cls, X, y, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return cls(precompute=True, **kw).fit(X, y)


def _against(sk, X, y, ids, K, l1_ratios, alphas=None, n_alphas=100, **kw):
    fs = fold_stats(X, y, ids, K)
    o = enet_cv_from_stats(fs, l1_ratios, alphas=alphas, n_alphas=n_alphas, **kw)
    alpha, l1, li, ai = choose(o["mse"], o["alphas"], l1_ratios)
    mse = np.squeeze(o["mse"])
    assert mse.shape == sk.mse_path_.shape
    rel = float(np.max(np.abs(mse - sk.mse_path_) / np.abs(sk.mse_path_)))
    assert rel <= 1e-12, rel
    sk_alphas = np.atleast_2d(sk.alphas_)
    np.testing.assert_allclose(o["alphas"] if alphas is None else o["alphas"][:1], sk_alphas, rtol=1e-13)
    assert alpha == pytest.approx(sk.alpha_, rel=1e-13)
    assert l1 == getattr(sk, "l1_ratio_", 1.0)
    # the refit: the path of the summed statistic at (alpha_, l1_ratio_)
    ref = enet_path_from_stats(fold_sum(fs), l1, alphas=[alpha], **kw)
    scale = max(float(np.max(np.abs(sk.coef_))), 1e-12)
    assert float(np.max(np.abs(ref["coefs"][0] - sk.coef_))) <= 1e-8 * scale
    assert int(ref["n_iter"][0]) == sk.n_iter_
    return rel


def test_heldout_identity_is_the_mean_squared_residual():
    X, y = _rows(500, 7, 1)
    w, b = np.linspace(-1, 1, 7), 3.0
    for fit_b in (b, 0.0):
        assert heldout_mse(stat(X, y), w, fit_b) == pytest.approx(np.mean((X @ w + fit_b - y) ** 2), rel=1e-10)


def test_lasso_cv5():
    X, y = _rows(3001, 12, 2)
    ids, K = b2.fold_ids(3001, cv=5)
    rel = _against(_sk(LassoCV, X, y, cv=5), X, y, ids, K, [1.0])
    print(f"\nLassoCV cv=5: mse_path_ {rel:.2e}")


def test_elastic_net_cv_shuffled_folds_several_ratios():
    X, y = _rows(3001, 12, 3)
    cv = KFold(4, shuffle=True, random_state=0)
    ids, K = b2.fold_ids(3001, cv=cv)
    ratios = [0.2, 0.7, 1.0]
    rel = _against(_sk(ElasticNetCV, X, y, cv=cv, l1_ratio=ratios), X, y, ids, K, ratios)
    print(f"\nElasticNetCV KFold(4, shuffle): mse_path_ {rel:.2e}")


def test_explicit_unsorted_alphas_no_intercept_positive():
    X, y = _rows(2000, 9, 4, offset=0.0)
    ids, K = b2.fold_ids(2000, cv=3)
    user = [0.01, 0.3, 0.001, 0.05]
    srt = np.sort(user)[::-1]
    sk = _sk(ElasticNetCV, X, y, cv=3, l1_ratio=[0.5, 0.9], alphas=user, fit_intercept=False, positive=True)
    _against(sk, X, y, ids, K, [0.5, 0.9], alphas=srt, fit_intercept=False, positive=True)
    np.testing.assert_array_equal(sk.alphas_, srt)


def test_fold_ids_match_sklearn_splits():
    n = 103
    for cv in (None, 4, KFold(6), KFold(5, shuffle=True, random_state=3)):
        ids, K = b2.fold_ids(n, cv=cv)
        ref = KFold(5) if cv is None else (KFold(cv) if isinstance(cv, int) else cv)
        for k, (_, test) in enumerate(ref.split(np.zeros((n, 1)))):
            assert np.array_equal(np.flatnonzero(ids == k), np.sort(test))
        assert K == ref.get_n_splits()
    # with a row mask: the folds of the kept rows, dropped rows 255
    mask = (np.arange(n) % 3 != 0).astype(np.uint8)
    ids, K = b2.fold_ids(n, mask, 1, cv=KFold(4, shuffle=True, random_state=1))
    kept = np.flatnonzero(mask == 1)
    assert np.all(ids[mask == 0] == 255)
    for k, (_, test) in enumerate(KFold(4, shuffle=True, random_state=1).split(np.zeros((kept.size, 1)))):
        assert np.array_equal(np.flatnonzero(ids == k), np.sort(kept[test]))
    # an iterable of (train, test) works too
    splits = list(KFold(3).split(np.zeros((n, 1))))
    assert np.array_equal(b2.fold_ids(n, cv=splits)[0], b2.fold_ids(n, cv=3)[0])


def test_fold_ids_refusals():
    for cv in (ShuffleSplit(5, random_state=0), RepeatedKFold(n_splits=3, n_repeats=2, random_state=0)):
        with pytest.raises(ValueError, match="partition the kept rows"):
            b2.fold_ids(100, cv=cv)
    with pytest.raises(ValueError, match="Cannot have number of splits n_splits=5 greater than the number of samples: "
                                         "n_samples=3."):
        b2.fold_ids(10, np.array([1, 1, 1] + [0] * 7, np.uint8), 1, cv=None)
    with pytest.raises(ValueError, match="at most 254"):
        b2.fold_ids(1000, cv=255)
