"""The driver of B200QuadraticDiscriminantAnalysis against scikit-learn 1.9's QuadraticDiscriminantAnalysis, on the CPU:
the estimator runs on a numpy stand-in for the context whose class-sum, per-class scatter and decision calls compute,
in float64 on float64 copies of the staged float32 rows, what the kernels compute, so every difference left is the host
code's.  means_, priors_, scalings_ and covariance_ within 1e-10 relative, rotations_ within 1e-10 after aligning column
signs (the data have separated eigenvalues), decisions within 1e-10 relative, equal predict and warnings, predict_proba
within 1e-9; scikit-learn's errors with its exact messages, the refusals, a joblib round trip and the export."""
import io
import re
import warnings

import joblib
import numpy as np
import pytest
from sklearn.discriminant_analysis import QuadraticDiscriminantAnalysis

import bodywork_mlops_demo_b200 as b2
from test_lda_driver import NumpyLdaContext, align, rel


class NumpyQdaContext(NumpyLdaContext):
    """The calls B200QuadraticDiscriminantAnalysis makes on a ``Context``, in numpy float64."""

    def __init__(self):
        super().__init__()
        self.calls.update(scatters=0, decision=0)

    def class_scatters(self, X, y, classes, means, *, row_mask=None, mask_keep=1):
        self.calls["scatters"] += 1
        Xk, yk = self._kept(X, y, row_mask, mask_keep)
        cl = np.asarray(classes, dtype=np.float32)
        S, nk = np.zeros((cl.size, Xk.shape[1], Xk.shape[1])), np.zeros(cl.size)
        for k, v in enumerate(cl):
            U = Xk[yk == v] - np.asarray(means, dtype=np.float64)[k]
            S[k] = np.triu(U.T @ U) + np.triu(U.T @ U, 1).T
            nk[k] = len(U)
        return {"scatters": S, "class_counts": nk, "kept": float(len(yk)),
                "unmatched": float(np.sum(~np.isin(yk, cl))), "nonfinite": float(np.sum(~np.isfinite(yk)))}

    def qda_decision(self, X, means, transforms, offsets, classes, y=None, *, row_mask=None, mask_keep=1,
                     decision=False, label=False, diff=False):
        self.calls["decision"] += 1
        X = np.asarray(X, dtype=np.float64)
        dec = np.stack([-0.5 * np.sum(((X - m) @ W) ** 2, axis=1) + c
                        for m, W, c in zip(means, transforms, offsets)], axis=1)
        cl = np.asarray(classes, dtype=np.float32)
        lab = cl[np.argmax(dec, axis=1)]
        out = {}
        if decision:
            out["decision"] = dec
        if label:
            out["label"] = lab
        if diff:
            out["diff"] = dec[:, 1] - dec[:, 0]
        if y is not None:
            keep = np.ones(len(X), bool) if row_mask is None else np.asarray(row_mask) == mask_keep
            out["kept"] = float(keep.sum())
            out["correct"] = float(np.sum(keep & (np.asarray(y, dtype=np.float32) == lab)))
        return out


def make_data(n=4000, d=5, k=3, seed=0, offset=100.0, counts=None):
    """float32-representable rows offset by ``offset`` (as float64) and labels of every one of k classes; each class has
    its own rotation and well separated variances, so its covariance has separated eigenvalues.  ``counts``: rows per
    class (default: about n / k each)."""
    rng = np.random.default_rng(seed)
    t = np.repeat(np.arange(k), counts) if counts is not None else np.r_[np.arange(k), rng.integers(0, k, size=n - k)]
    rng.shuffle(t)
    X = np.empty((len(t), d))
    centres = rng.normal(0.0, 2.0, size=(k, d))
    scales = np.geomspace(0.3, 3.0, d)
    for c in range(k):
        Q, _ = np.linalg.qr(rng.normal(size=(d, d)))
        rows = t == c
        X[rows] = centres[c] + (rng.normal(size=(rows.sum(), d)) * scales * rng.uniform(0.8, 1.25)) @ Q.T
    return (X + offset).astype(np.float32).astype(np.float64), t


def fit_pair(X, y, row_mask=None, mask_keep=1, **kw):
    ctx = NumpyQdaContext()
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours = b2.B200QuadraticDiscriminantAnalysis(ctx=ctx, **kw).fit(X, y, row_mask, mask_keep)
    keep = slice(None) if row_mask is None else np.asarray(row_mask) == mask_keep
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref = QuadraticDiscriminantAnalysis(**kw).fit(X[keep], np.asarray(y)[keep])
    assert [str(w.message) for w in w_ours] == [str(w.message) for w in w_ref]
    return ours, ref, ctx


def assert_same_model(ours, ref, X, tol=1e-10):
    assert np.array_equal(ours.classes_, ref.classes_) and ours.classes_.dtype == ref.classes_.dtype
    assert rel(ours.means_, ref.means_) <= tol
    assert rel(ours.priors_, ref.priors_) <= tol
    assert ours.n_features_in_ == ref.n_features_in_
    assert len(ours.scalings_) == len(ref.scalings_) == len(ours.rotations_) == ref.classes_.size
    for k in range(ref.classes_.size):
        assert rel(ours.scalings_[k], ref.scalings_[k]) <= tol, k
        R, Rr, s = ours.rotations_[k], ref.rotations_[k], ref.scalings_[k]
        assert rel((R * s) @ R.T, (Rr * s) @ Rr.T) <= tol, k
        if np.all(-np.diff(s) > 1e-6 * s[0]):            # separated eigenvalues: each column up to its sign
            assert rel(align(R, Rr), Rr) <= tol, k
    assert hasattr(ours, "covariance_") == hasattr(ref, "covariance_")
    if hasattr(ref, "covariance_"):
        for a, b in zip(ours.covariance_, ref.covariance_, strict=True):
            assert rel(a, b) <= tol
    assert rel(ours.decision_function(X), ref.decision_function(X)) <= tol
    assert np.array_equal(ours.predict(X), ref.predict(X))
    assert np.max(np.abs(ours.predict_proba(X) - ref.predict_proba(X))) <= 1e-9
    assert ours.score(X, ref.predict(X)) == 1.0


@pytest.mark.parametrize("k", [2, 3, 7, 32])
@pytest.mark.parametrize("d", [1, 5, 24])
@pytest.mark.parametrize("solver", ["svd", "eigen"])
def test_solvers_match_sklearn(k, d, solver):
    X, y = make_data(6000, d, k, seed=k * 31 + d)
    ours, ref, ctx = fit_pair(X, y, solver=solver)
    assert_same_model(ours, ref, X)
    assert ctx.calls["class_sums"] == 1 and ctx.calls["scatters"] == 1


@pytest.mark.parametrize("reg_param", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("k", [2, 5])
def test_reg_param(reg_param, k):
    X, y = make_data(3000, 6, k, seed=17 + k)
    ours, ref, _ = fit_pair(X, y, reg_param=reg_param, store_covariance=True)
    assert_same_model(ours, ref, X)


@pytest.mark.parametrize("shrinkage", [None, 0, 0.3, 1])
@pytest.mark.parametrize("k", [2, 5])
def test_shrinkage(shrinkage, k):
    X, y = make_data(3000, 7, k, seed=11 + k)
    ours, ref, _ = fit_pair(X, y, solver="eigen", shrinkage=shrinkage, store_covariance=True)
    assert_same_model(ours, ref, X)


@pytest.mark.parametrize("solver", ["svd", "eigen"])
def test_priors_store_covariance_and_tol(solver):
    X, y = make_data(3000, 6, 4, seed=5)
    p = np.array([0.1, 0.2, 0.3, 0.5])                  # as given: scikit-learn neither renormalises nor warns
    ours, ref, _ = fit_pair(X, y, solver=solver, priors=p, store_covariance=True, tol=1e-3)
    assert_same_model(ours, ref, X)
    assert np.array_equal(ours.priors_, p)


@pytest.mark.parametrize("kind", ["int", "float", "str", "bool", "negative"])
def test_label_types(kind):
    X, t = make_data(2000, 4, 2 if kind == "bool" else 3, seed=4)
    y = {"int": t * 7 + 1, "float": t * 2.0 - 1.0, "str": np.array(["a", "bb", "c"])[t], "bool": t.astype(bool),
         "negative": -t - 3}[kind]
    ours, ref, _ = fit_pair(X, y)
    assert_same_model(ours, ref, X)


@pytest.mark.parametrize("mask_keep", [1, 0])
def test_masks(mask_keep):
    X, y = make_data(3000, 5, 4, seed=8)
    mask = (np.arange(len(y)) % 3 != 0).astype(np.uint8)
    for solver in ("svd", "eigen"):
        ours, ref, _ = fit_pair(X, y, mask, mask_keep, solver=solver)
        assert_same_model(ours, ref, X)


def test_small_classes():
    """a class of d rows fits under svd when reg_param makes its scalings pass the rank check (as scikit-learn's d
    singular values do), and a class of 2 <= n_k <= d fits under eigen when shrinkage makes it full rank"""
    X, y = make_data(counts=[6, 300, 300], d=6, k=3, seed=12)
    ours, ref, _ = fit_pair(X, y, reg_param=0.5)
    assert_same_model(ours, ref, X)
    X, y = make_data(counts=[3, 300, 300], d=6, k=3, seed=13)
    ours, ref, _ = fit_pair(X, y, solver="eigen", shrinkage=0.4)
    assert_same_model(ours, ref, X)


def assert_same_error(X, y, **kw):
    """ours raises scikit-learn's exception type with its message"""
    with pytest.raises(Exception) as ref:
        QuadraticDiscriminantAnalysis(**kw).fit(X, y)
    with pytest.raises(type(ref.value), match=f"^{re.escape(str(ref.value))}$"):
        b2.B200QuadraticDiscriminantAnalysis(ctx=NumpyQdaContext(), **kw).fit(X, y)


def test_errors_match_sklearn():
    X, y = make_data(counts=[1, 50, 50], d=3, k=3, seed=1)
    assert_same_error(X, y)                                        # a class of one row
    assert_same_error(X, y, solver="eigen")
    X, y = make_data(counts=[40, 4, 40], d=6, k=3, seed=2)
    for reg_param in (0.0, 0.5, 1.0):                              # n_k < d under svd, whatever reg_param is
        assert_same_error(X, y, reg_param=reg_param)
    assert_same_error(X, y, solver="eigen")                        # n_k < d under eigen without shrinkage
    X, y = make_data(counts=[6, 40, 40], d=6, k=3, seed=3)
    assert_same_error(X, y)                                        # n_k = d under svd
    X, y = make_data(2000, 4, 3, seed=3)
    X = np.c_[X, X[:, 1]]                                          # rank deficient in every class
    assert_same_error(X, y)
    assert_same_error(X, y, solver="eigen")
    assert_same_error(X, y, reg_param=1e-6)
    assert_same_error(X, np.zeros(len(X)))                         # one class


def test_predict_log_proba():
    X, y = make_data(2000, 4, 3, seed=2)
    ours, ref, _ = fit_pair(X, y)
    Xp = X.copy()
    Xp[:5] = (100.0 + 30.0 * (X[:5] - 100.0)).astype(np.float32)   # probabilities far below 1e-300, staged exactly
    a, b = ours.predict_log_proba(Xp), ref.predict_log_proba(Xp)
    assert np.max(np.abs(a - b)) <= 1e-10 * np.max(np.abs(b))


def refusal(exc, match, X=None, y=None, **kw):
    if X is None:
        X, y = make_data(300, 3, 3, seed=1)
    with pytest.raises(exc, match=match):
        b2.B200QuadraticDiscriminantAnalysis(ctx=NumpyQdaContext(), **kw).fit(X, y)


def test_refusals():
    who = "B200QuadraticDiscriminantAnalysis"
    refusal(ValueError, f"shrinkage='auto' is not supported by {who}", solver="eigen", shrinkage="auto")
    refusal(ValueError, f"covariance_estimator is not supported by {who}", solver="eigen",
            covariance_estimator=object())
    refusal(NotImplementedError, r"shrinkage not supported with 'svd' solver\. \(B200", shrinkage=0.5)
    refusal(ValueError, f"The 'solver' parameter of {who} must be", solver="lsqr")
    refusal(ValueError, f"The 'shrinkage' parameter of {who}", solver="eigen", shrinkage=1.5)
    refusal(ValueError, f"The 'reg_param' parameter of {who}", reg_param=2.0)
    refusal(ValueError, f"The 'tol' parameter of {who}", tol=-1.0)
    refusal(ValueError, f"priors has 2 entries, but y holds 3 classes \\({who}\\)", priors=[0.5, 0.5])
    X, y = make_data(300, 3, 3, seed=1)
    with pytest.raises(ValueError, match=f"sample_weight is not supported by {who}"):
        b2.B200QuadraticDiscriminantAnalysis(ctx=NumpyQdaContext()).fit(X, y, sample_weight=np.ones(300))
    refusal(ValueError, f"{who} fits at most 32 classes", X, np.arange(300) % 33)
    refusal(ValueError, "Unknown label type", X, y + 0.5)
    refusal(ValueError, f"multilabel y .* is not supported by {who}", X, np.c_[y, y])
    refusal(ValueError, "Input y contains NaN", X, np.where(np.arange(300) == 7, np.nan, y))
    Xn = X.copy()
    Xn[4, 1] = np.inf
    refusal(ValueError, "Input X or y contains NaN", Xn, y)
    with pytest.raises(ValueError, match="predict_log_proba takes host rows"):
        b2.B200QuadraticDiscriminantAnalysis(ctx=NumpyQdaContext()).fit(X, y).predict_log_proba(
            b2.DeviceArray.__new__(b2.DeviceArray))


def test_to_sklearn_and_joblib_round_trip():
    X, y = make_data(2000, 5, 4, seed=6)
    for solver, kw in (("svd", {"store_covariance": True}), ("eigen", {"shrinkage": 0.2})):
        ours = b2.B200QuadraticDiscriminantAnalysis(ctx=NumpyQdaContext(), solver=solver, **kw).fit(X, y)
        buf = io.BytesIO()
        joblib.dump(ours.to_sklearn(), buf)
        buf.seek(0)
        sk = joblib.load(buf)
        assert type(sk) is QuadraticDiscriminantAnalysis
        assert np.array_equal(sk.predict(X), ours.predict(X))
        assert np.max(np.abs(sk.predict_proba(X) - ours.predict_proba(X))) <= 1e-12
        assert hasattr(sk, "covariance_") == ("store_covariance" in kw)
        buf = io.BytesIO()
        joblib.dump(ours, buf)
        buf.seek(0)
        again = joblib.load(buf)
        again._ctx = NumpyQdaContext()
        assert np.array_equal(again.predict(X), ours.predict(X))
