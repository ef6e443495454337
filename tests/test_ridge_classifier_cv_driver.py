"""The driver of B200RidgeClassifierCV against scikit-learn 1.9's RidgeClassifierCV (cv=None), on the CPU: the estimator
runs on a numpy stand-in for the context whose calls compute, in float64 on float64 copies of the staged float32 rows,
what the kernels compute (tests/loo_classes_oracle.py for the leave-one-out pass), so every difference left is the
driver's: label staging, the chunks of at most MAX_ALPHAS alphas and their first-best merge, the scores, the shapes, the
solve's fallback and the export.  alpha_ equal, best_score_, cv_results_ and coefficients within 1e-12 relative, equal
predict and score; the refusals carry scikit-learn's messages where it has one."""
import io

import joblib
import numpy as np
import pytest
from sklearn import linear_model

import bodywork_mlops_demo_b200 as b2
from loo_classes_oracle import ridge_classifier_loo
from test_ridge_classifier_driver import NumpyClassifierContext, make_data

MAX_ALPHAS = b2.native.MAX_ALPHAS


class NumpyClassifierCVContext(NumpyClassifierContext):
    """``NumpyClassifierContext`` with the call B200RidgeClassifierCV adds, b2_ridge_classifier_loo."""

    def __init__(self):
        super().__init__()
        self.calls["loo"] = 0

    def ridge_classifier_loo(self, X, y, classes, alphas, row_mask=None, mask_keep=1, *, fit_intercept=True,
                             scoring=b2.native.LOO_SQUARED, store_cv=False):
        al = np.asarray(alphas, dtype=np.float64).ravel()
        assert 1 <= al.size <= MAX_ALPHAS
        self.calls["loo"] += 1
        n = len(np.asarray(y))
        self.gram_reset(np.asarray(X).shape[1])
        self.gram_accumulate(X, y, row_mask, mask_keep)
        d, S = self.d, self.S
        if S[d, d] == 0:
            raise ValueError("no row kept: the leave-one-out error needs at least one row")
        cs = self.class_sums(X, y, classes, S[:d, d] / S[d, d] if fit_intercept else None, row_mask=row_mask,
                             mask_keep=mask_keep)
        cl = np.asarray(classes, dtype=np.float32)
        yk = np.asarray(y, dtype=np.float32)
        k = np.array([np.flatnonzero(cl == v)[0] if np.any(cl == v) else -1 for v in yk])
        acc = scoring == b2.native.LOO_ACCURACY
        o = ridge_classifier_loo(np.asarray(X, dtype=np.float64), k, cl.size, al, mask=row_mask, keep=mask_keep,
                                 fit_intercept=fit_intercept, scoring="accuracy" if acc else None)
        cv = None
        if store_cv:
            cv = np.full((n, o["cv"].shape[1], al.size), np.nan)
            keep = np.ones(n, bool) if row_mask is None else np.asarray(row_mask) == mask_keep
            cv[keep] = o["cv"]
        out = {"mse": o["mse"], "correct": o["correct"], "best": o["best"], "kept": cs["kept"],
               "unmatched": cs["unmatched"], "nonfinite": cs["nonfinite"], "cv": cv}
        try:
            out["coef"], out["intercept"] = self.solve_classes(cs["sums"], float(al[o["best"]]), fit_intercept)
        except np.linalg.LinAlgError as exc:
            exc.result = out
            raise
        return out


def fit_pair(X, y, **kw):
    ctx = NumpyClassifierCVContext()
    ours = b2.B200RidgeClassifierCV(ctx=ctx, **kw).fit(X, y)
    ref = linear_model.RidgeClassifierCV(**kw).fit(X, y)
    return ours, ref, ctx


def rel(a, b):
    return np.max(np.abs(np.asarray(a, dtype=np.float64) - b)) / max(np.max(np.abs(b)), 1e-300)


def assert_same_model(ours, ref, X, y, tol=1e-12):
    assert ours.alpha_ == ref.alpha_ and type(ours.alpha_) is float and isinstance(ours.best_score_, float)
    assert ours.best_score_ == pytest.approx(ref.best_score_, rel=tol)
    assert ours.coef_.shape == ref.coef_.shape and np.shape(ours.intercept_) == np.shape(ref.intercept_)
    assert rel(ours.coef_, ref.coef_) <= tol
    if ref.fit_intercept:
        assert rel(ours.intercept_, ref.intercept_) <= tol
    assert ours.classes_.dtype == ref.classes_.dtype and np.array_equal(ours.classes_, ref.classes_)
    assert ours.n_features_in_ == ref.n_features_in_
    assert np.array_equal(ours.predict(X), ref.predict(X))
    assert ours.score(X, y) == ref.score(X, y)
    if ref.store_cv_results:
        assert ours.cv_results_.shape == ref.cv_results_.shape
        assert rel(ours.cv_results_, ref.cv_results_) <= tol


ALPHAS = (0.01, 0.3, 3.0, 30.0)


@pytest.mark.parametrize("scoring", [None, "accuracy"])
@pytest.mark.parametrize("fit_intercept", [True, False])
@pytest.mark.parametrize("k", [2, 3, 7, 32])
def test_fit_matches_sklearn(k, fit_intercept, scoring):
    X, y = make_data(30 * k + 150, 6, k, seed=k)
    ours, ref, ctx = fit_pair(X, y, alphas=ALPHAS, fit_intercept=fit_intercept, scoring=scoring,
                              store_cv_results=True)
    assert ctx.calls["loo"] == 1
    assert_same_model(ours, ref, X, y)


@pytest.mark.parametrize("scoring", [None, "accuracy"])
def test_grids_longer_than_one_call_merge_by_the_first_best(scoring):
    X, y = make_data(500, 5, 4, seed=31)
    grid = np.logspace(-3, 4, 150)
    ours, ref, ctx = fit_pair(X, y, alphas=grid, scoring=scoring, store_cv_results=True)
    assert ctx.calls["loo"] == 3
    assert_same_model(ours, ref, X, y)


def test_ties_across_chunks_go_to_the_lowest_index():
    X, y = make_data(400, 5, 3, seed=37)
    best = linear_model.RidgeClassifierCV(alphas=ALPHAS).fit(X, y).alpha_
    grid = np.r_[np.full(10, 1e4), best, np.full(60, 1e4), best, 1e4]   # the best alpha at 10 and at 71
    ours, ref, ctx = fit_pair(X, y, alphas=grid)
    assert ctx.calls["loo"] == 2 and ours.alpha_ == ref.alpha_ == best
    assert_same_model(ours, ref, X, y)
    # accuracy: every alpha of a two-class grid scores 1.0 and the first one wins, across chunks too
    X2, y2 = make_data(300, 4, 2, seed=41)
    ours, ref, _ = fit_pair(X2, y2, alphas=np.logspace(2, -2, 70), scoring="accuracy")
    assert ours.alpha_ == ref.alpha_ == 100.0 and ours.best_score_ == ref.best_score_ == 1.0


LABELS = {"int": np.array([0, 1, 2, 5]), "negative": np.array([-7, -3, -1, 4]), "str": np.array(["a", "bb", "c", "d"]),
          "float": np.array([-2.0, 0.0, 1.0, 3.0]), "bool": np.array([False, True])}


@pytest.mark.parametrize("kind", sorted(LABELS))
def test_label_types(kind):
    labels = LABELS[kind]
    X, y = make_data(300, 5, labels.size, seed=43, labels=labels)
    ours, ref, _ = fit_pair(X, y, alphas=ALPHAS, store_cv_results=True)
    assert_same_model(ours, ref, X, y)
    assert ours.predict(X).dtype == ref.predict(X).dtype


def test_binary_accuracy_scores_one_and_picks_the_first_alpha():
    X, y = make_data(300, 5, 2, seed=47)
    ours, ref, _ = fit_pair(X, y, alphas=(30.0, 0.01, 3.0), scoring="accuracy", store_cv_results=True)
    assert ours.best_score_ == ref.best_score_ == 1.0 and ours.alpha_ == ref.alpha_ == 30.0
    assert ours.cv_results_.shape == (300, 1, 3)
    assert_same_model(ours, ref, X, y)


@pytest.mark.parametrize("mask_keep", [0, 1])
def test_masks(mask_keep):
    X, y = make_data(500, 6, 5, seed=53)
    mask = (np.random.default_rng(2).uniform(size=500) < 0.7).astype(np.uint8)
    keep = mask == mask_keep
    ours = b2.B200RidgeClassifierCV(alphas=ALPHAS, store_cv_results=True, ctx=NumpyClassifierCVContext()).fit(
        X, y, row_mask=mask, mask_keep=mask_keep)
    ref = linear_model.RidgeClassifierCV(alphas=ALPHAS, store_cv_results=True).fit(X[keep], y[keep])
    assert_same_model(ours, ref, X[keep], y[keep])


def test_rank_deficient_grid_falls_back_to_the_eigendecomposition():
    """at a tiny alpha the factorisation refuses a duplicated column; the model then comes from the minimum-norm solve
    of B200RidgeClassifier's fallback, which predicts as the fit without the duplicate does"""
    X5, y = make_data(400, 5, 4, seed=59)
    X = np.c_[X5, X5[:, 1]]
    ours = b2.B200RidgeClassifierCV(alphas=(1e-14,), ctx=NumpyClassifierCVContext()).fit(X, y)
    reduced = linear_model.RidgeClassifier(alpha=1e-14).fit(X5, y)
    assert ours.alpha_ == 1e-14 and np.all(np.isfinite(ours.coef_))
    assert np.mean(ours.predict(X) == reduced.predict(X5)) >= 0.99
    assert np.allclose(ours.coef_[:, 1], ours.coef_[:, 5]) and np.allclose(ours.coef_[:, 1] * 2, reduced.coef_[:, 1])


def test_to_sklearn_round_trip():
    for k in (2, 5):
        X, y = make_data(300, 6, k, seed=61, labels=np.array(["x", "y", "z", "u", "v"])[:k])
        ours, ref, _ = fit_pair(X, y, alphas=ALPHAS, store_cv_results=True)
        buf = io.BytesIO()
        joblib.dump(ours.to_sklearn(), buf)
        reg = joblib.load(io.BytesIO(buf.getvalue()))
        assert type(reg) is linear_model.RidgeClassifierCV
        assert np.array_equal(reg.predict(X), ref.predict(X)) and reg.score(X, y) == ref.score(X, y)
        assert np.array_equal(reg.classes_, ref.classes_) and reg.alpha_ == ref.alpha_
        assert set(vars(reg)) == set(vars(ref))
    assert repr(b2.B200RidgeClassifierCV(alphas=(1.0, 2.0))) == "B200RidgeClassifierCV(alphas=(1.0, 2.0))"


def refusal(X, y, match, fit_kw=None, **kw):
    est = b2.B200RidgeClassifierCV(ctx=NumpyClassifierCVContext(), **kw)
    with pytest.raises(ValueError, match=match):
        est.fit(X, y, **(fit_kw or {}))


def test_refusals_carry_sklearns_messages():
    X, y = make_data(100, 3, 3, seed=67)
    for kw, yy, match in ((dict(alphas=[1.0, -1.0]), y, "must be > 0.0"),
                          ({}, np.r_[np.nan, y[1:]], "Input y contains NaN."),
                          ({}, y + 0.5, "Unknown label type")):
        refusal(X, yy, match, **kw)
        with pytest.raises(ValueError, match=match):
            linear_model.RidgeClassifierCV(**kw).fit(X, yy)


def test_refusals_name_what_is_unsupported():
    X, y = make_data(200, 3, 3, seed=71)
    refusal(X, y, "must be a finite float", alphas=[1.0, np.nan])
    refusal(X, y, "must be a finite float", alphas=[np.inf])
    refusal(X, np.zeros(200), "at least 2 classes")
    refusal(X, np.c_[y == 1, y == 2].astype(int), "multilabel")
    refusal(X, np.arange(200) % 33, "at most 32 classes")
    refusal(X, y, "k-fold grid search", cv=5)
    refusal(X, y, "scoring='f1_macro' is not supported", scoring="f1_macro")
    refusal(X, y, "class_weight", class_weight="balanced")
    refusal(X, y, "sample_weight", fit_kw=dict(sample_weight=np.ones(200)))


def test_a_class_sum_pass_that_kept_other_rows_than_the_gram_is_an_error():
    """the consistency check of B200RidgeClassifier.fit: the pass's kept rows must be the Gram's"""
    class Drifting(NumpyClassifierCVContext):
        def ridge_classifier_loo(self, *args, **kw):
            out = super().ridge_classifier_loo(*args, **kw)
            out["kept"] -= 1.0
            return out

    X, y = make_data(200, 4, 3, seed=73)
    with pytest.raises(RuntimeError, match="other labels than the label check"):
        b2.B200RidgeClassifierCV(ctx=Drifting()).fit(X, y)
