"""The driver of B200RidgeClassifier against scikit-learn 1.9's RidgeClassifier, on the CPU: the estimator runs on a numpy
stand-in for the context whose Gram, class-sum, solve, classify and label calls compute, in float64 on float64 copies of
the staged float32 rows, what the kernels compute, so every difference left is the driver's.  Coefficients within 1e-12
relative, equal predict, score, shapes and classes_ dtype; the refusals carry scikit-learn's messages (ours where
scikit-learn has none); the export predicts after a joblib round trip."""
import io
import warnings

import joblib
import numpy as np
import pytest
import scipy.linalg
from sklearn import linear_model

import bodywork_mlops_demo_b200 as b2


class NumpyClassifierContext:
    """The calls B200RidgeClassifier makes on a ``Context``, in numpy float64."""

    def __init__(self):
        self.calls = {"gram": 0, "class_sums": 0, "solve": 0, "classify": 0}
        self.d, self.S = 0, None

    @staticmethod
    def _kept(X, y, row_mask, mask_keep):
        X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float32)
        if row_mask is not None:
            keep = np.asarray(row_mask) == mask_keep
            X, y = X[keep], y[keep]
        return X, y

    def gram_reset(self, d):
        self.d, self.S = int(d), np.zeros((d + 2, d + 2))

    def gram_accumulate(self, X, y, row_mask=None, mask_keep=1):
        self.calls["gram"] += 1
        Xk, yk = self._kept(X, y, row_mask, mask_keep)
        Z = np.c_[Xk, np.ones(len(yk)), yk.astype(np.float64)]
        self.S = self.S + Z.T @ Z

    def gram_export(self):
        return self.S.copy()

    def class_sums(self, X, y, classes, center=None, *, row_mask=None, mask_keep=1):
        self.calls["class_sums"] += 1
        Xk, yk = self._kept(X, y, row_mask, mask_keep)
        cl = np.asarray(classes, dtype=np.float32)
        c = np.zeros(Xk.shape[1]) if center is None else np.asarray(center, dtype=np.float64)
        sums = np.zeros((cl.size, Xk.shape[1] + 1))
        for k, v in enumerate(cl):
            rows = Xk[yk == v] - c
            sums[k, :-1], sums[k, -1] = rows.sum(axis=0), len(rows)
        return {"sums": sums, "kept": float(len(yk)), "unmatched": float(np.sum(~np.isin(yk, cl))),
                "nonfinite": float(np.sum(~np.isfinite(yk)))}

    def solve_classes(self, class_sums, alpha=1.0, fit_intercept=True):
        """solve_classes_kernel's system, its right-hand sides and its pivot rule"""
        self.calls["solve"] += 1
        d, S, sums = self.d, self.S, np.asarray(class_sums)
        n = S[d, d]
        m = S[:d, d] / n if fit_intercept else np.zeros(d)
        A = S[:d, :d] - n * np.outer(m, m) + alpha * np.eye(d)
        tot, nk = sums[:, :d].sum(axis=0), sums[:, d]
        ks = [1] if sums.shape[0] == 2 else list(range(sums.shape[0]))
        R = np.stack([2 * (sums[k, :d] - nk[k] / n * tot) if fit_intercept else 2 * sums[k, :d] - tot for k in ks], 1)
        try:
            L = scipy.linalg.cholesky(A, lower=True)
        except np.linalg.LinAlgError:
            raise np.linalg.LinAlgError("pivot not positive") from None
        if np.min(np.diag(L) ** 2) <= 1e-12 * np.max(np.diag(A)):
            raise np.linalg.LinAlgError("pivot not positive")
        W = scipy.linalg.cho_solve((L, True), R)
        ybar = 2 * nk[ks] / n - 1 if fit_intercept else np.zeros(len(ks))
        return W.T, ybar - m @ W

    def solve_eigh(self, fit_intercept=True):
        d, S = self.d, self.S
        n = S[d, d]
        m = S[:d, d] / n if fit_intercept else np.zeros(d)
        lam, Q = np.linalg.eigh(S[:d, :d] - n * np.outer(m, m))
        return np.maximum(lam, 0.0), Q

    def classify(self, X, coef, intercept, classes, y=None, *, row_mask=None, mask_keep=1, decision=False,
                 label=False):
        self.calls["classify"] += 1
        W = np.atleast_2d(np.asarray(coef, dtype=np.float64))
        eta = np.asarray(X, dtype=np.float64) @ W.T + np.asarray(intercept, dtype=np.float64)
        cl = np.asarray(classes, dtype=np.float32)
        lab = cl[(eta[:, 0] > 0).astype(int)] if W.shape[0] == 1 else cl[np.argmax(eta, axis=1)]
        out = {}
        if decision:
            out["decision"] = eta
        if label:
            out["label"] = lab
        if y is not None:
            keep = np.ones(len(lab), bool) if row_mask is None else np.asarray(row_mask) == mask_keep
            out["kept"] = float(keep.sum())
            out["correct"] = float(np.sum(keep & (np.asarray(y, dtype=np.float32) == lab)))
        return out


def make_data(n, d, k, seed=0, labels=None):
    """float32-representable rows (as float64) and labels of every one of k classes, from a noisy linear argmax"""
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 1.0, size=(n, d)).astype(np.float32).astype(np.float64)
    B = rng.normal(size=(d, k))
    t = np.argmax(X @ B + rng.normal(0.0, 1.0, size=(n, k)), axis=1)
    t[:k] = np.arange(k)                       # every class present
    return X, (t if labels is None else labels[t])


def assert_close_coef(ours, ref, tol=1e-12):
    scale = max(np.max(np.abs(ref.coef_)), np.max(np.abs(ref.intercept_)), 1e-300)
    err = max(np.max(np.abs(ours.coef_ - ref.coef_)), np.max(np.abs(np.asarray(ours.intercept_) - ref.intercept_)))
    assert err / scale <= tol, f"coefficients differ by {err / scale:.3e} relative"


def fit_pair(X, y, **kw):
    ctx = NumpyClassifierContext()
    ours = b2.B200RidgeClassifier(ctx=ctx, **kw).fit(X, y)
    ref = linear_model.RidgeClassifier(**kw).fit(X, y)
    return ours, ref, ctx


def assert_same_model(ours, ref, X, y, tol=1e-12):
    assert_close_coef(ours, ref, tol)
    assert ours.coef_.shape == ref.coef_.shape and np.shape(ours.intercept_) == np.shape(ref.intercept_)
    assert type(ours.intercept_) is type(ref.intercept_)
    assert ours.classes_.dtype == ref.classes_.dtype and np.array_equal(ours.classes_, ref.classes_)
    assert ours.solver_ == ref.solver_ and ours.n_iter_ is None and ours.n_features_in_ == ref.n_features_in_
    assert np.array_equal(ours.predict(X), ref.predict(X))
    assert ours.score(X, y) == ref.score(X, y)
    dec = ours.decision_function(X)
    want = ref.decision_function(X)
    assert dec.shape == want.shape
    assert np.max(np.abs(dec - want)) <= 1e-12 * max(np.max(np.abs(want)), 1.0)


@pytest.mark.parametrize("k", [2, 3, 7, 32])
@pytest.mark.parametrize("alpha", [0.0, 1e-3, 1.0, 1e3])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_fit_matches_sklearn(k, alpha, fit_intercept):
    X, y = make_data(40 * k + 60, 6, k, seed=k)
    ours, ref, ctx = fit_pair(X, y, alpha=alpha, fit_intercept=fit_intercept)
    assert ctx.calls["gram"] == 1 and ctx.calls["class_sums"] == 1 and ctx.calls["solve"] == 1
    assert_same_model(ours, ref, X, y)


LABELS = {"int": np.array([0, 1, 2, 5]), "negative": np.array([-7, -3, -1, 4]), "str": np.array(["a", "bb", "c", "d"]),
          "float": np.array([-2.0, 0.0, 1.0, 3.0])}


@pytest.mark.parametrize("kind", sorted(LABELS))
@pytest.mark.parametrize("k", [2, 4])
def test_label_types(kind, k):
    X, y = make_data(300, 5, k, seed=3, labels=LABELS[kind][:k])
    ours, ref, _ = fit_pair(X, y, alpha=0.5)
    assert_same_model(ours, ref, X, y)


def test_bool_labels():
    X, y = make_data(200, 4, 2, seed=5, labels=np.array([False, True]))
    ours, ref, _ = fit_pair(X, y)
    assert_same_model(ours, ref, X, y)
    assert ours.predict(X).dtype == np.bool_


@pytest.mark.parametrize("mask_keep", [0, 1])
def test_masks(mask_keep):
    X, y = make_data(500, 6, 5, seed=7)
    mask = (np.random.default_rng(1).uniform(size=500) < 0.7).astype(np.uint8)
    keep = mask == mask_keep
    y = y.copy()
    y[~keep & (np.arange(500) % 3 == 0)] = 99          # a label outside the kept rows' classes, on dropped rows
    ours = b2.B200RidgeClassifier(alpha=2.0, ctx=NumpyClassifierContext()).fit(X, y, row_mask=mask, mask_keep=mask_keep)
    ref = linear_model.RidgeClassifier(alpha=2.0).fit(X[keep], y[keep])
    assert_same_model(ours, ref, X[keep], y[keep])
    assert ours.score(X, y, row_mask=mask, mask_keep=mask_keep) == ref.score(X[keep], y[keep])


def test_score_counts_labels_outside_classes_as_wrong():
    X, y = make_data(300, 4, 3, seed=11)
    ours, ref, _ = fit_pair(X, y)
    y2 = y.copy()
    y2[::4] = 17
    assert ours.score(X, y2) == ref.score(X, y2)
    assert ours.score(X, y2.astype(str)) == 0.0         # labels that do not compare with classes_


def test_rank_deficient_alpha_zero_falls_back_to_the_eigendecomposition():
    """scikit-learn's 'svd' fallback keeps singular values above an absolute 1e-15, so on a duplicated column it keeps
    the rounding-level one; the eigendecomposition drops it and returns the minimum-norm solution, which predicts as the
    fit without the duplicate does"""
    X5, y = make_data(400, 5, 4, seed=13)
    X = np.c_[X5, X5[:, 1]]
    ours, ref, _ = fit_pair(X, y, alpha=0.0)
    assert ours.solver_ == ref.solver_ == "svd"
    reduced = linear_model.RidgeClassifier(alpha=0.0).fit(X5, y)
    assert np.mean(ours.predict(X) == reduced.predict(X5)) >= 0.99
    assert np.allclose(ours.coef_[:, 1], ours.coef_[:, 5]) and np.allclose(ours.coef_[:, 1] * 2, reduced.coef_[:, 1])


def test_to_sklearn_round_trip():
    for k in (2, 5):
        X, y = make_data(300, 6, k, seed=17, labels=np.array(["x", "y", "z", "u", "v"])[:k])
        ours, ref, _ = fit_pair(X, y, alpha=3.0)
        buf = io.BytesIO()
        joblib.dump(ours.to_sklearn(), buf)
        reg = joblib.load(io.BytesIO(buf.getvalue()))
        assert type(reg) is linear_model.RidgeClassifier
        assert np.array_equal(reg.predict(X), ref.predict(X))
        assert np.array_equal(reg.classes_, ref.classes_)
        assert set(vars(reg)) == set(vars(ref))
        assert reg.score(X, y) == ref.score(X, y)


def refusal(X, y, match, fit_kw=None, **kw):
    est = b2.B200RidgeClassifier(ctx=NumpyClassifierContext(), **kw)
    with pytest.raises(ValueError, match=match):
        est.fit(X, y, **(fit_kw or {}))
    return est


def test_refusals_carry_sklearns_messages():
    X, y = make_data(100, 3, 3, seed=19)
    for kw, yy, match in ((dict(alpha=-1.0), y, "The 'alpha' parameter of RidgeClassifier must be a float in the range"),
                          (dict(solver="foo"), y, "The 'solver' parameter of RidgeClassifier must be a str among"),
                          ({}, np.r_[np.nan, y[1:]], "Input y contains NaN."),
                          ({}, y + 0.5, "Unknown label type")):
        refusal(X, yy, match, **kw)
        with pytest.raises(ValueError, match=match.split(".")[0].replace("(", r"\(")):
            linear_model.RidgeClassifier(**kw).fit(X, yy)


def test_refusals_name_what_is_unsupported():
    X, y = make_data(200, 3, 3, seed=23)
    refusal(X, np.zeros(200), "at least 2 classes")
    refusal(X, np.c_[y == 1, y == 2].astype(int), "multilabel")
    refusal(X, np.arange(200) % 33, "at most 32 classes")
    refusal(X, y, "class_weight", class_weight="balanced")
    refusal(X, y, "sample_weight", fit_kw=dict(sample_weight=np.ones(200)))
    refusal(X, y, "positive", positive=True)
    refusal(X, y, "solver='svd' is not supported", solver="svd")
    refusal(X, y, "array alpha", alpha=[1.0, 2.0, 3.0])
    refusal(X, np.full(200, 4), "at least 2 classes")
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        b2.B200RidgeClassifier(ctx=NumpyClassifierContext(), solver="cholesky").fit(X, y)


def test_32_classes_fit_and_33_are_refused():
    X, y = make_data(32 * 30, 8, 32, seed=29)
    ours, ref, _ = fit_pair(X, y, alpha=0.1)
    assert ours.coef_.shape == (32, 8)
    assert_same_model(ours, ref, X, y)
    y33 = y.copy()
    y33[-1] = 32
    refusal(X, y33, "at most 32 classes")
