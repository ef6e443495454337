"""The Newton driver of B200MultinomialLogisticRegression against scikit-learn 1.9's LogisticRegression(solver=
"newton-cholesky") with three or more classes, on the CPU: the estimator runs on a numpy stand-in for the context whose
passes (``multinomial_pass``, ``multinomial_line_search``, ``classify``, ``softmax_rows``, the label scans and, for two
classes, the binary passes) evaluate scikit-learn's own LinearModelLoss(HalfMultinomialLoss) on float64 copies of the
staged float32 rows, so every difference left is the driver's.  Equal n_iter_, the same warning categories,
coefficients within 1e-12 relative, equal predict; the refusals carry scikit-learn's messages (ours where scikit-learn
has none)."""
import warnings

import numpy as np
import pytest
from scipy.special import softmax as sp_softmax
from sklearn import linear_model
from sklearn._loss.loss import HalfMultinomialLoss
from sklearn.linear_model._linear_loss import LinearModelLoss

import bodywork_mlops_demo_b200 as b2
from test_logistic_driver import NumpyLogisticContext


class NumpyMultinomialContext(NumpyLogisticContext):
    """The multinomial passes of ``Context`` in numpy: the same unscaled sums, from scikit-learn's LinearModelLoss."""

    def __init__(self):
        super().__init__()
        self.passes.update({"mn_pass": 0, "mn_hessian": 0, "mn_ladder": 0, "classify": 0})

    @staticmethod
    def _targets(y, classes):
        """the class index of each y (-1: none), as class_of reads the fp32 labels"""
        y = np.asarray(y, dtype=np.float32)
        cl = np.asarray(classes, dtype=np.float32)
        k = np.full(y.shape, -1, dtype=np.int64)
        for c in range(cl.size):
            k[y == cl[c]] = c
        return k

    def multinomial_pass(self, X, y, classes, coef, *, row_mask=None, mask_keep=1, fit_intercept=True, hessian=True):
        self.passes["mn_pass"] += 1
        self.passes["mn_hessian"] += int(hessian)
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        n, d = Xd.shape
        K = np.size(classes)
        t = self._targets(yd, classes)
        W = np.asarray(coef, dtype=np.float64).copy()
        if not fit_intercept:
            W[:, d] = 0.0
        lml = LinearModelLoss(base_loss=HalfMultinomialLoss(n_classes=K), fit_intercept=True)
        tt = np.where(t >= 0, t, 0).astype(np.float64)
        with np.errstate(all="ignore"):
            loss = lml.loss(W, Xd, tt) * n
            grad, hess, _ = lml.gradient_hessian(W.ravel(order="F"), Xd, tt)
        raw = Xd @ W[:, :d].T + W[:, d]
        out = {"loss": float(loss), "kept": float(n), "unmatched": float(np.sum(t < 0)),
               "nonfinite": float(np.sum(~np.isfinite(yd))),
               "correct": float(np.sum(np.argmax(raw, axis=1) == t)),
               "grad": grad.reshape(K, d + 1, order="F") * n, "hessian": None}
        if hessian:
            out["hessian"] = (hess * n).reshape(d + 1, K, d + 1, K).transpose(1, 3, 0, 2).copy()
        return out

    def multinomial_line_search(self, X, y, classes, coef, step, *, n_steps=21, row_mask=None, mask_keep=1):
        self.passes["mn_ladder"] += 1
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        n, d = Xd.shape
        K = np.size(classes)
        tt = self._targets(yd, classes).astype(np.float64)
        W, S = np.asarray(coef, dtype=np.float64), np.asarray(step, dtype=np.float64)
        lml = LinearModelLoss(base_loss=HalfMultinomialLoss(n_classes=K), fit_intercept=True)
        raw = Xd @ W[:, :d].T + W[:, d]
        raw_newton = Xd @ S[:, :d].T + S[:, d]
        zero = np.zeros((K, d + 1))
        with np.errstate(all="ignore"):
            return np.array([lml.loss_gradient(zero, Xd, tt, raw_prediction=raw + 0.5 ** s * raw_newton)[0] * n
                             for s in range(n_steps)])

    def classify(self, X, coef, intercept, classes, y=None, *, row_mask=None, mask_keep=1, decision=False,
                 label=False):
        self.passes["classify"] += 1
        eta = np.asarray(X, dtype=np.float64) @ np.asarray(coef, dtype=np.float64).T + np.asarray(intercept)
        lab = np.asarray(classes, dtype=np.float32)[np.argmax(eta, axis=1)]
        out = {}
        if decision:
            out["decision"] = eta
        if label:
            out["label"] = lab
        if y is not None:
            keep = np.ones(len(lab), bool) if row_mask is None else np.asarray(row_mask) == mask_keep
            out["kept"] = float(keep.sum())
            out["correct"] = float(np.sum(keep & (np.asarray(y, np.float32) == lab)))
        return out

    def softmax_rows(self, values):
        values[:] = sp_softmax(values, axis=1)

    def label_values(self, y, row_mask=None, mask_keep=1, max_values=32):
        y = np.asarray(y, dtype=np.float32)
        if row_mask is not None:
            y = y[np.asarray(row_mask) == mask_keep]
        v = np.unique(y[np.isfinite(y)] + np.float32(0.0))
        return v[:max_values].astype(np.float32), v.size > max_values


def make_data(n=600, d=5, k=3, seed=0, collinear=False, scale=1.0):
    """float32-representable rows (returned as float64) and a target of k classes drawn from a softmax model"""
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 1.0, size=(n, d))
    if collinear:
        X[:, -1] = X[:, 0]
    X = X.astype(np.float32).astype(np.float64)
    B = rng.normal(0.0, 1.0, size=(d, k)) * scale
    P = sp_softmax(X @ B + rng.normal(0.0, 0.3, size=k), axis=1)
    t = np.array([rng.choice(k, p=p) for p in P])
    t[:k] = np.arange(k)                            # every class present
    return X, t


def fit_pair(X, y, **kw):
    ctx = NumpyMultinomialContext()
    ours = b2.B200MultinomialLogisticRegression(ctx=ctx, **kw)
    ref = linear_model.LogisticRegression(solver="newton-cholesky", **kw)
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X, y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X, y)
    return ours, ref, ctx, [w.category for w in w_ours], [w.category for w in w_ref]


def rel_err(ours, ref, centred=False):
    """the largest coefficient difference relative to the largest coefficient; centred: of the coefficients minus
    their mean over the classes, the part the probabilities depend on"""
    a, b = np.c_[ours.coef_, ours.intercept_], np.c_[ref.coef_, ref.intercept_]
    if centred:
        a, b = a - a.mean(axis=0), b - b.mean(axis=0)
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


def assert_same_model(ours, ref, X, tol=1e-12):
    assert ours.n_iter_.dtype == np.int32 and ours.n_iter_.shape == (1,)
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    assert ours.coef_.shape == ref.coef_.shape and ours.intercept_.shape == ref.intercept_.shape
    assert np.array_equal(ours.classes_, ref.classes_) and ours.classes_.dtype == ref.classes_.dtype
    err, err_c = rel_err(ours, ref), rel_err(ours, ref, centred=True)
    assert err <= tol, f"coefficients differ by {err:.3e} relative"
    assert err_c <= 1e-12, f"centred coefficients differ by {err_c:.3e} relative"
    assert np.array_equal(ours.predict(X), ref.predict(X))
    np.testing.assert_allclose(ours.predict_proba(X), ref.predict_proba(X), rtol=0, atol=1e-12)


@pytest.mark.parametrize("k", [3, 4, 7, 32])
@pytest.mark.parametrize("C", [1e-2, 1.0, 1e4, np.inf])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_newton_driver_matches_sklearn(k, C, fit_intercept):
    X, t = make_data(n=300 + 40 * k, d=6, k=k, seed=k)
    ours, ref, ctx, cat_ours, cat_ref = fit_pair(X, t, C=C, fit_intercept=fit_intercept)
    assert cat_ours == cat_ref
    if cat_ref:      # the L-BFGS-B fallback follows a path that rounding can bend: the same model class by class
        assert np.array_equal(ours.n_iter_, ref.n_iter_)
        assert np.mean(ours.predict(X) == ref.predict(X)) > 0.99
        return
    # At C = 1e4 the classes' mean weight vector, which the probabilities do not see, is held by the penalty
    # 1 / (C n) alone: a rounding difference r in the gradient moves it by about r C n (scikit-learn's own result moves
    # as much between BLAS builds), so there only the centred coefficients are held to 1e-12.
    assert_same_model(ours, ref, X, tol=1e-12 if C != 1e4 else 1e-10)
    assert ctx.passes["mn_ladder"] == ours.n_iter_[0]
    dec, ours_dec = ref.decision_function(X), ours.decision_function(X)
    np.testing.assert_allclose(ours_dec - ours_dec.mean(axis=1, keepdims=True), dec - dec.mean(axis=1, keepdims=True),
                               rtol=0, atol=1e-11 * np.max(np.abs(dec)))
    np.testing.assert_allclose(ours.predict_log_proba(X), ref.predict_log_proba(X), rtol=1e-10, atol=1e-12)
    assert ours.score(X, t) == ref.score(X, t)
    if np.isinf(C) or fit_intercept:        # the symmetric parametrisation of NewtonCholeskySolver.finalize
        np.testing.assert_allclose(ours.intercept_.sum(), 0.0, atol=1e-12 * max(1.0, np.abs(ours.intercept_).max()))


LABELS = {"int": lambda t: t, "neg": lambda t: 2 * t - 5, "float": lambda t: t + 10.0,
          "str": lambda t: np.array(["a", "b", "c", "d"])[t], "obj": lambda t: np.array(["x", 3, "z", "w"], object)[t]}


@pytest.mark.parametrize("labels", list(LABELS), ids=list(LABELS))
def test_labels_of_any_dtype(labels):
    X, t = make_data(k=4, seed=11)
    y = LABELS[labels](t)
    if labels == "obj":
        with pytest.raises(TypeError):              # scikit-learn cannot sort mixed labels either
            linear_model.LogisticRegression(solver="newton-cholesky").fit(X, y)
        return
    ours, ref, _, cat_ours, cat_ref = fit_pair(X, y, C=1.0)
    assert cat_ours == cat_ref
    assert_same_model(ours, ref, X)
    assert ours.score(X, y) == ref.score(X, y)
    y_bad = y.copy().astype(object)
    y_bad[:5] = "other"                          # labels outside classes_ count as wrong
    assert ours.score(X, y_bad) == float(np.mean(ref.predict(X) == y_bad))


def test_device_labels_through_the_label_scans():
    X, t = make_data(k=5, seed=2)
    y = np.array([-2.0, 0.0, 3.0, 7.0, 1e6], dtype=np.float32)[t]
    ctx = NumpyMultinomialContext()
    classes, n = b2.B200MultinomialLogisticRegression._device_labels(ctx, y, None, 1)
    assert n == len(y) and classes.dtype == np.float32 and list(classes) == [-2.0, 0.0, 3.0, 7.0, 1e6]


def test_warm_start_matches_sklearn():
    X, t = make_data(k=4, seed=3)
    kw = dict(warm_start=True, max_iter=2, C=10.0)
    ours = b2.B200MultinomialLogisticRegression(ctx=NumpyMultinomialContext(), **kw)
    ref = linear_model.LogisticRegression(solver="newton-cholesky", **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours.fit(X, t)
        ref.fit(X, t)
        assert rel_err(ours, ref) <= 1e-12
        ours.max_iter = ref.max_iter = 100
        ours.fit(X[:400], t[:400])
        ref.fit(X[:400], t[:400])
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    assert rel_err(ours, ref) <= 1e-12


@pytest.mark.parametrize("fit_intercept", [True, False])
def test_unpenalised_warm_start_is_moved_into_the_gauge(fit_intercept):
    X, t = make_data(k=3, seed=8)
    kw = dict(warm_start=True, C=np.inf, fit_intercept=fit_intercept)
    ours = b2.B200MultinomialLogisticRegression(ctx=NumpyMultinomialContext(), **kw)
    ref = linear_model.LogisticRegression(solver="newton-cholesky", **kw)
    ours.coef_ = ref.coef_ = np.full((3, X.shape[1]), 0.25) + np.arange(3)[:, None]
    ours.intercept_ = ref.intercept_ = np.array([1.0, -2.0, 0.5]) if fit_intercept else np.zeros(3)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours.fit(X, t)
        ref.fit(X, t)
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    assert rel_err(ours, ref) <= 1e-12


def test_masked_rows_are_the_fit_of_the_kept_rows():
    X, t = make_data(k=3, seed=5)
    y = np.array(["a", "b", "c"])[t]
    mask = (np.arange(len(t)) % 3 != 0).astype(np.uint8)
    Xn, yn = X.copy(), y.astype(object)
    Xn[mask == 0, 0] = np.nan                     # rows not kept may hold anything
    yn[mask == 0] = "q"
    ours = b2.B200MultinomialLogisticRegression(ctx=NumpyMultinomialContext()).fit(Xn, yn, row_mask=mask)
    ref = linear_model.LogisticRegression(solver="newton-cholesky").fit(X[mask == 1], y[mask == 1])
    assert np.array_equal(ours.n_iter_, ref.n_iter_) and list(ours.classes_) == list(ref.classes_)
    assert rel_err(ours, ref) <= 1e-12
    assert ours.score(Xn, yn, row_mask=mask) == ref.score(X[mask == 1], y[mask == 1])


def test_collinear_unpenalised_fit_falls_back_to_lbfgs_like_sklearn():
    X, t = make_data(k=3, seed=2, collinear=True)
    ours, ref, _, cat_ours, cat_ref = fit_pair(X, t, C=np.inf)
    assert cat_ref, "scikit-learn was expected to warn"
    assert cat_ours == cat_ref
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    assert np.array_equal(ours.predict(X), ref.predict(X))
    np.testing.assert_allclose(ours.predict_proba(X), ref.predict_proba(X), rtol=0, atol=1e-6)


def test_two_classes_take_the_binary_fit():
    X, t = make_data(k=2, seed=4)
    ours, ref, ctx, cat_ours, cat_ref = fit_pair(X, t, C=1.0)
    assert cat_ours == cat_ref
    assert ctx.passes["mn_pass"] == 0 and ctx.passes["hessian"] > 0
    assert ours.coef_.shape == (1, X.shape[1]) and ours.intercept_.shape == (1,)
    assert_same_model(ours, ref, X)
    assert ours.decision_function(X).shape == (len(t),)
    assert ours.score(X, t) == ref.score(X, t)
    binary = b2.B200LogisticRegression(ctx=NumpyLogisticContext(), C=1.0).fit(X, t)
    assert np.array_equal(binary.coef_, ours.coef_) and np.array_equal(binary.n_iter_, ours.n_iter_)


def _sk_error(fn):
    with pytest.raises(ValueError) as e:
        fn()
    return str(e.value)


def test_refusals_carry_sklearns_messages():
    X, t = make_data(k=3)
    ctx = NumpyMultinomialContext()
    sk = lambda **kw: linear_model.LogisticRegression(solver="newton-cholesky", **kw)   # noqa: E731
    ours = lambda **kw: b2.B200MultinomialLogisticRegression(ctx=ctx, **kw)             # noqa: E731
    y_nan = t.astype(np.float64)
    y_nan[4] = np.nan
    y_inf = t.astype(np.float64)
    y_inf[4] = np.inf
    for y in (np.zeros(len(t)), np.linspace(0.0, 1.0, len(t)), y_nan, y_inf):
        assert _sk_error(lambda: ours().fit(X, y)) == _sk_error(lambda: sk().fit(X, y))
    with pytest.raises(ValueError, match="at most 32 classes, y has 33"):
        ours().fit(np.repeat(X[:33], 2, axis=0), np.repeat(np.arange(33), 2))
    for C in (0, -1.0):
        assert _sk_error(lambda: ours(C=C).fit(X, t)) == _sk_error(lambda: sk(C=C).fit(X, t))
    # our own refusals name the estimator the user built
    with pytest.raises(ValueError, match="class_weight is not supported by B200MultinomialLogisticRegression"):
        ours(class_weight="balanced").fit(X, t)
    with pytest.raises(ValueError, match="l1_ratio=0.5 is not supported: B200MultinomialLogisticRegression"):
        ours(l1_ratio=0.5).fit(X, t)
    with pytest.raises(ValueError, match="B200MultinomialLogisticRegression runs scikit-learn's 'newton-cholesky'"):
        ours(solver="lbfgs").fit(X, t)
    with pytest.raises(ValueError, match="sample_weight is not supported by B200MultinomialLogisticRegression"):
        ours().fit(X, t, sample_weight=np.ones(len(t)))
    fitted = ours().fit(X, t)
    with pytest.raises(ValueError, match="but B200MultinomialLogisticRegression is expecting 5 features"):
        fitted.predict(X[:, :3])
    with pytest.raises(ValueError, match="0 sample"):
        ours().fit(X, t, row_mask=np.zeros(len(t), np.uint8))
    with pytest.raises(ValueError, match="1d array"):
        ours().fit(X, np.c_[t, t])
    Xn = X.copy()
    Xn[3, 1] = np.inf
    with pytest.raises(ValueError, match="NaN, infinity"):
        ours().fit(Xn, t)
    # device labels: the label scans give the same refusals
    for y, match in ((np.zeros(10, np.float32), "only one class: np.float32"),
                     (np.arange(40, dtype=np.float32), "at most 32 classes"),
                     (np.linspace(0, 1, 10, dtype=np.float32), "continuous"),
                     (np.r_[np.zeros(5), np.ones(4), np.nan].astype(np.float32), "NaN or infinity")):
        with pytest.raises(ValueError, match=match):
            b2.B200MultinomialLogisticRegression._device_labels(ctx, y, None, 1)


def test_to_sklearn_is_a_working_sklearn_estimator(tmp_path):
    import joblib
    X, t = make_data(k=4, seed=9)
    y = np.array(["w", "x", "y", "z"])[t]
    ours = b2.B200MultinomialLogisticRegression(ctx=NumpyMultinomialContext(), C=0.5).fit(X, y)
    path = tmp_path / "m.joblib"
    joblib.dump(ours.to_sklearn(), path)
    clf = joblib.load(path)
    assert isinstance(clf, linear_model.LogisticRegression) and clf.solver == "newton-cholesky"
    np.testing.assert_allclose(clf.predict_proba(X), ours.predict_proba(X), rtol=0, atol=1e-15)
    np.testing.assert_array_equal(clf.predict(X), ours.predict(X))
    assert clf.score(X, y) == ours.score(X, y)
