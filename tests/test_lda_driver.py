"""The driver of B200LinearDiscriminantAnalysis against scikit-learn 1.9's LinearDiscriminantAnalysis, on the CPU: the
estimator runs on a numpy stand-in for the context whose class-sum, scatter, classify, logistic-predict, softmax and
label calls compute, in float64 on float64 copies of the staged float32 rows, what the kernels compute, so every
difference left is the host code's.  coef_, intercept_, means_, priors_, xbar_, covariance_ and
explained_variance_ratio_ within 1e-10 relative, equal predict and warnings, predict_proba within 1e-9, scalings_ and
transform within 1e-10 after aligning column signs; the refusals, a joblib round trip and the export."""
import io
import warnings

import joblib
import numpy as np
import pytest
from sklearn.discriminant_analysis import LinearDiscriminantAnalysis

import bodywork_mlops_demo_b200 as b2
from test_multinomial_driver import NumpyMultinomialContext
from test_ridge_classifier_driver import NumpyClassifierContext


class NumpyLdaContext(NumpyMultinomialContext):
    """The calls B200LinearDiscriminantAnalysis makes on a ``Context``, in numpy float64."""
    _kept = staticmethod(NumpyClassifierContext._kept)
    class_sums = NumpyClassifierContext.class_sums
    classify = NumpyClassifierContext.classify

    def __init__(self):
        super().__init__()
        self.calls = {"class_sums": 0, "classify": 0, "scatter": 0}

    def class_scatter(self, X, y, classes, means, weights=None, *, row_mask=None, mask_keep=1):
        self.calls["scatter"] += 1
        Xk, yk = self._kept(X, y, row_mask, mask_keep)
        cl = np.asarray(classes, dtype=np.float32)
        w = np.ones(cl.size) if weights is None else np.asarray(weights, dtype=np.float64)
        S = np.zeros((Xk.shape[1], Xk.shape[1]))
        for k, v in enumerate(cl):
            U = Xk[yk == v] - np.asarray(means, dtype=np.float64)[k]
            S += (w[k] * U).T @ U
        S = np.triu(S) + np.triu(S, 1).T
        return {"scatter": S, "kept": float(len(yk)), "unmatched": float(np.sum(~np.isin(yk, cl))),
                "nonfinite": float(np.sum(~np.isfinite(yk)))}


def make_data(n=4000, d=5, k=3, seed=0, offset=100.0):
    """float32-representable correlated rows offset by ``offset`` (as float64) and labels of every one of k classes"""
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(d, d)) / np.sqrt(d)
    centres = rng.normal(0.0, 1.5, size=(k, d))
    t = rng.integers(0, k, size=n)
    t[:k] = np.arange(k)
    X = centres[t] + rng.normal(size=(n, d)) @ A + 0.3 * rng.normal(size=(n, d)) + offset
    return X.astype(np.float32).astype(np.float64), t


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.max(np.abs(a - b), initial=0.0) / max(np.max(np.abs(b), initial=0.0), 1e-300))


def align(ours, ref):
    """ours with each column's sign set to agree with ref's"""
    s = np.sign(np.sum(ours * ref, axis=0))
    return ours * np.where(s == 0, 1.0, s)


def fit_pair(X, y, row_mask=None, mask_keep=1, **kw):
    ctx = NumpyLdaContext()
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours = b2.B200LinearDiscriminantAnalysis(ctx=ctx, **kw).fit(X, y, row_mask, mask_keep)
    keep = slice(None) if row_mask is None else np.asarray(row_mask) == mask_keep
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref = LinearDiscriminantAnalysis(**kw).fit(X[keep], np.asarray(y)[keep])
    assert [str(w.message) for w in w_ours] == [str(w.message) for w in w_ref]
    return ours, ref, ctx


def assert_same_model(ours, ref, X, tol=1e-10):
    scale = max(np.max(np.abs(ref.coef_)), np.max(np.abs(ref.intercept_)))
    assert np.max(np.abs(ours.coef_ - ref.coef_)) / scale <= tol
    assert np.max(np.abs(ours.intercept_ - ref.intercept_)) / scale <= tol
    assert ours.coef_.shape == ref.coef_.shape and ours.intercept_.shape == ref.intercept_.shape
    assert np.array_equal(ours.classes_, ref.classes_) and ours.classes_.dtype == ref.classes_.dtype
    for name in ("means_", "priors_", "xbar_", "covariance_", "explained_variance_ratio_"):
        assert hasattr(ours, name) == hasattr(ref, name), name
        if hasattr(ref, name):
            assert rel(getattr(ours, name), getattr(ref, name)) <= tol, name
    assert ours._max_components == ref._max_components and ours._n_features_out == ref._n_features_out
    assert np.array_equal(ours.predict(X), ref.predict(X))
    assert np.max(np.abs(ours.predict_proba(X) - ref.predict_proba(X))) <= 1e-9
    assert ours.score(X, ref.predict(X)) == 1.0
    if ref.solver != "lsqr":
        c = ref._max_components if ref.solver == "eigen" else ref.scalings_.shape[1]
        assert rel(align(ours.scalings_[:, :c], ref.scalings_[:, :c]), ref.scalings_[:, :c]) <= tol
        T, Tr = ours.transform(X), ref.transform(X)
        assert T.shape == Tr.shape
        # transform is x.s - xbar.s: its error is relative to sum |x_j s_j|
        bound = np.abs(X) @ np.abs(ref.scalings_[:, : Tr.shape[1]])
        assert np.max(np.abs(align(T, Tr) - Tr) / np.maximum(bound, 1e-300), initial=0.0) <= tol


@pytest.mark.parametrize("k", [2, 3, 7, 32])
@pytest.mark.parametrize("d", [1, 5, 24])
@pytest.mark.parametrize("solver", ["svd", "lsqr", "eigen"])
def test_solvers_match_sklearn(k, d, solver):
    X, y = make_data(4000, d, k, seed=k * 31 + d)
    ours, ref, ctx = fit_pair(X, y, solver=solver)
    assert_same_model(ours, ref, X)
    assert ctx.calls["class_sums"] == 1 and ctx.calls["scatter"] == 1     # frequency priors: one scatter pass


@pytest.mark.parametrize("solver", ["svd", "lsqr", "eigen"])
@pytest.mark.parametrize("priors", ["given", "unnormalised"])
def test_priors(solver, priors):
    X, y = make_data(3000, 6, 4, seed=5)
    p = np.array([0.1, 0.2, 0.3, 0.4]) * (1.0 if priors == "given" else 3.0)
    ours, ref, ctx = fit_pair(X, y, solver=solver, priors=p, store_covariance=True)
    assert_same_model(ours, ref, X)
    assert ctx.calls["scatter"] == (1 if solver == "lsqr" else 2)


@pytest.mark.parametrize("solver", ["lsqr", "eigen"])
@pytest.mark.parametrize("shrinkage", [None, 0, 0.3, 1])
@pytest.mark.parametrize("k", [2, 5])
def test_shrinkage(solver, shrinkage, k):
    X, y = make_data(3000, 7, k, seed=11 + k)
    ours, ref, _ = fit_pair(X, y, solver=solver, shrinkage=shrinkage, priors=np.full(k, 1.0 / k))
    assert_same_model(ours, ref, X)


@pytest.mark.parametrize("solver", ["svd", "eigen"])
@pytest.mark.parametrize("n_components", [None, 1, 3])
def test_n_components_store_covariance_and_tol(solver, n_components):
    X, y = make_data(2500, 6, 5, seed=3)
    ours, ref, ctx = fit_pair(X, y, solver=solver, n_components=n_components, store_covariance=True, tol=1e-3)
    assert_same_model(ours, ref, X)
    assert ctx.calls["scatter"] == 1
    T = b2.B200LinearDiscriminantAnalysis(ctx=NumpyLdaContext(), solver=solver,
                                          n_components=n_components).fit_transform(X, y)
    Tr = LinearDiscriminantAnalysis(solver=solver, n_components=n_components).fit_transform(X, y)
    assert T.shape == Tr.shape


def test_duplicated_and_constant_columns_svd():
    X, y = make_data(4000, 5, 3, seed=9)
    X = np.c_[X, X[:, 1], np.full(len(X), 3.0)]
    ours, ref, _ = fit_pair(X, y, solver="svd", store_covariance=True)
    assert ref.scalings_.shape[1] == ours.scalings_.shape[1]
    assert_same_model(ours, ref, X)


def test_tol_cuts_the_rank_like_sklearn():
    X, y = make_data(3000, 6, 4, seed=21)
    X[:, 5] = (X[:, 4] + 0.1 * np.sign(X[:, 0] - 100)).astype(np.float32)   # one small within-class singular value
    for tol in (1e-4, 0.3):
        ours, ref, _ = fit_pair(X, y, tol=tol)
        assert ours.scalings_.shape == ref.scalings_.shape
        assert_same_model(ours, ref, X)


@pytest.mark.parametrize("kind", ["int", "float", "str", "bool", "negative"])
def test_label_types(kind):
    X, t = make_data(2000, 4, 2 if kind == "bool" else 3, seed=4)
    y = {"int": t * 7 + 1, "float": t * 2.0 - 1.0, "str": np.array(["a", "bb", "c"])[t], "bool": t.astype(bool),
         "negative": -t - 3}[kind]
    ours, ref, _ = fit_pair(X, y, solver="lsqr")
    assert_same_model(ours, ref, X)


@pytest.mark.parametrize("mask_keep", [1, 0])
def test_masks(mask_keep):
    X, y = make_data(3000, 5, 4, seed=8)
    mask = (np.arange(len(y)) % 3 != 0).astype(np.uint8)
    mask[:8] = mask_keep                    # every class among the kept rows
    for solver in ("svd", "eigen"):
        ours, ref, _ = fit_pair(X, y, mask, mask_keep, solver=solver)
        assert_same_model(ours, ref, X)


def test_predict_log_proba():
    X, y = make_data(2000, 4, 3, seed=2)
    ours, ref, _ = fit_pair(X, y)
    Xp = X.copy()
    Xp[:5] = 100.0 + 3000.0 * (X[:5] - 100.0)   # probabilities that round to 0
    a, b = ours.predict_log_proba(Xp), ref.predict_log_proba(Xp)
    floor = np.log(np.finfo(np.float64).smallest_normal)
    assert np.any(b == floor) and np.array_equal(a == floor, b == floor)
    assert np.max(np.abs(a - b)) <= 1e-9 * np.max(np.abs(b))       # log p: differences of decisions


def refusal(exc, match, X=None, y=None, **kw):
    if X is None:
        X, y = make_data(300, 3, 3, seed=1)
    with pytest.raises(exc, match=match):
        b2.B200LinearDiscriminantAnalysis(ctx=NumpyLdaContext(), **kw).fit(X, y)


def test_refusals():
    who = "B200LinearDiscriminantAnalysis"
    refusal(ValueError, f"shrinkage='auto' is not supported by {who}: the Ledoit-Wolf", solver="lsqr", shrinkage="auto")
    refusal(ValueError, f"covariance_estimator is not supported by {who}", solver="lsqr",
            covariance_estimator=object())
    refusal(NotImplementedError, r"shrinkage not supported with 'svd' solver\. \(B200", shrinkage=0.5)
    refusal(ValueError, f"The 'solver' parameter of {who} must be", solver="qr")
    refusal(ValueError, f"The 'shrinkage' parameter of {who}", solver="lsqr", shrinkage=1.5)
    refusal(ValueError, "priors must be non-negative", priors=[0.5, 0.7, -0.2])
    refusal(ValueError, "priors has 2 entries", priors=[0.5, 0.5])
    refusal(ValueError, r"n_components cannot be larger than min\(n_features, n_classes - 1\)", n_components=3)
    X, y = make_data(300, 3, 3, seed=1)
    refusal(ValueError, f"{who} needs samples of at least 2 classes", X, np.zeros(300))
    refusal(ValueError, f"{who} fits at most 32 classes", X, np.arange(300) % 33)
    refusal(ValueError, "Unknown label type", X, y + 0.5)
    refusal(ValueError, f"multilabel y .* is not supported by {who}", X, np.c_[y, y])
    refusal(ValueError, "Input y contains NaN", X, np.where(np.arange(300) == 7, np.nan, y))
    Xn = X.copy()
    Xn[4, 1] = np.inf
    refusal(ValueError, "Input X or y contains NaN", Xn, y)
    refusal(ValueError, "The number of samples must be more than the number of classes", X[:3], y[:3])
    with pytest.raises(NotImplementedError, match="transform not implemented for 'lsqr'"):
        b2.B200LinearDiscriminantAnalysis(ctx=NumpyLdaContext(), solver="lsqr").fit(X, y).transform(X)


def test_to_sklearn_and_joblib_round_trip():
    X, y = make_data(2000, 5, 4, seed=6)
    for solver in ("svd", "lsqr", "eigen"):
        ours = b2.B200LinearDiscriminantAnalysis(ctx=NumpyLdaContext(), solver=solver).fit(X, y)
        buf = io.BytesIO()
        joblib.dump(ours.to_sklearn(), buf)
        buf.seek(0)
        sk = joblib.load(buf)
        assert type(sk) is LinearDiscriminantAnalysis
        assert np.array_equal(sk.predict(X), ours.predict(X))
        assert np.max(np.abs(sk.predict_proba(X) - ours.predict_proba(X))) <= 1e-12
        if solver != "lsqr":
            assert np.max(np.abs(sk.transform(X) - ours.transform(X))) <= 1e-9 * np.max(np.abs(sk.transform(X)))
        buf = io.BytesIO()
        joblib.dump(ours, buf)
        buf.seek(0)
        again = joblib.load(buf)
        again._ctx = NumpyLdaContext()
        assert np.array_equal(again.predict(X), ours.predict(X))
