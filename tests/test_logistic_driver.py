"""The Newton driver of B200LogisticRegression against scikit-learn 1.9's binary LogisticRegression(solver=
"newton-cholesky"), on the CPU: the estimator runs on a numpy stand-in for the context whose passes (``logistic_pass``,
``logistic_line_search``, ``logistic_predict``, ``label_scan``) evaluate scikit-learn's HalfBinomialLoss on float64
copies of the staged float32 rows, so every difference left is the driver's.  Equal n_iter_, coefficients within 1e-12
relative, the same warning categories, equal predict and predict_proba within 1e-15; the refusals carry scikit-learn's
messages (ours where scikit-learn has none)."""
import warnings

import numpy as np
import pytest
from scipy.special import expit
from sklearn import linear_model
from sklearn._loss.loss import HalfBinomialLoss

import bodywork_mlops_demo_b200 as b2

LOSS = HalfBinomialLoss()


class NumpyLogisticContext:
    """The logistic passes of ``Context`` in numpy: the same unscaled sums, from scikit-learn's pointwise losses."""

    def __init__(self):
        self.passes = {"pass": 0, "hessian": 0, "ladder": 0, "predict": 0}

    @staticmethod
    def _rows(X, y, row_mask, mask_keep):
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64)
        if row_mask is not None:
            keep = np.asarray(row_mask) == mask_keep
            X, y = X[keep], y[keep]
        return X, y

    def logistic_pass(self, X, y, coef, intercept, neg_label=0.0, pos_label=1.0, *, row_mask=None, mask_keep=1,
                      fit_intercept=True, hessian=True):
        self.passes["pass"] += 1
        self.passes["hessian"] += int(hessian)
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        pos, in_range = yd == pos_label, (yd == pos_label) | (yd == neg_label)
        t = pos.astype(np.float64)
        raw = Xd @ np.asarray(coef, dtype=np.float64) + (intercept if fit_intercept else 0.0)
        with np.errstate(all="ignore"):
            pointwise = LOSS.loss(y_true=t, raw_prediction=raw)
            g, h = LOSS.gradient_hessian(y_true=t, raw_prediction=raw)
        Z = np.c_[Xd, np.ones(len(yd))]
        return {"loss": float(pointwise.sum()), "const": 0.0, "sum_y": float(t.sum()), "kept": float(len(yd)),
                "y_out_of_range": float(np.sum(~in_range)), "h_nonpos": float(np.sum(h <= 0)),
                "y_nonfinite": float(np.sum(~np.isfinite(yd))), "grad": Z.T @ g,
                "correct": float(np.sum(in_range & ((raw > 0) == pos))),
                "hessian": Z.T @ (np.abs(h)[:, None] * Z) if hessian else None}

    def logistic_line_search(self, X, y, coef, intercept, step, step_intercept, neg_label=0.0, pos_label=1.0, *,
                             n_steps=21, row_mask=None, mask_keep=1):
        """the loss of loss_gradient, which scikit-learn's line search evaluates"""
        self.passes["ladder"] += 1
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        t = (yd == pos_label).astype(np.float64)
        raw = Xd @ np.asarray(coef, dtype=np.float64) + intercept
        raw_newton = Xd @ np.asarray(step, dtype=np.float64) + step_intercept
        with np.errstate(all="ignore"):
            return np.array([LOSS.loss_gradient(y_true=t, raw_prediction=raw + 0.5 ** k * raw_newton)[0].sum()
                             for k in range(n_steps)])

    def logistic_predict(self, X, coef, intercept, neg_label=0.0, pos_label=1.0, *, decision=False, proba=False,
                         label=False):
        self.passes["predict"] += 1
        eta = np.asarray(X, dtype=np.float64) @ np.asarray(coef, dtype=np.float64) + intercept
        out = {}
        if decision:
            out["decision"] = eta
        if proba:
            p = expit(eta)
            out["proba"] = np.stack([1 - p, p], axis=1)
        if label:
            out["label"] = np.where(eta > 0, pos_label, neg_label).astype(np.float32)
        return out

    def label_scan(self, y, row_mask=None, mask_keep=1):
        y = np.asarray(y, dtype=np.float32)
        if row_mask is not None:
            y = y[np.asarray(row_mask) == mask_keep]
        fin = y[np.isfinite(y)]
        lo, hi = (float(fin.min()), float(fin.max())) if fin.size else (np.nan, np.nan)
        return {"kept": float(y.size), "nonfinite": float(np.sum(~np.isfinite(y))),
                "nonintegral": float(np.sum(fin != np.rint(fin))), "min": lo, "max": hi,
                "n_min": float(np.sum(y == lo)), "n_max": float(np.sum(y == hi))}


LABELS = {"01": np.array([0, 1]), "pm1": np.array([-1, 1]), "37": np.array([3, 7]),
          "str": np.array(["no", "yes"]), "bool": np.array([False, True])}


def make_data(n=400, d=6, seed=0, collinear=False, scale=1.0):
    """float32-representable rows (returned as float64) and a {0, 1} target drawn from a logistic model"""
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 1.0, size=(n, d))
    if collinear:
        X[:, -1] = X[:, 0]
    X = X.astype(np.float32).astype(np.float64)
    beta = rng.uniform(-1.0, 1.0, size=d) * scale
    t = (rng.uniform(size=n) < expit(X @ beta + 0.3)).astype(np.int64)
    return X, t


def assert_close_coef(ours, ref, tol=1e-12):
    scale = max(np.max(np.abs(ref.coef_)), np.max(np.abs(ref.intercept_)), 1e-300)
    err = max(np.max(np.abs(ours.coef_ - ref.coef_)), np.max(np.abs(ours.intercept_ - ref.intercept_))) / scale
    assert err <= tol, f"coefficients differ by {err:.3e} relative"


def fit_pair(X, y, **kw):
    ctx = NumpyLogisticContext()
    ours = b2.B200LogisticRegression(ctx=ctx, **kw)
    ref = linear_model.LogisticRegression(solver="newton-cholesky", **kw)
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X, y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X, y)
    return ours, ref, ctx, [w.category for w in w_ours], [w.category for w in w_ref]


def assert_same_model(ours, ref, X):
    assert ours.n_iter_.dtype == np.int32 and ours.n_iter_.shape == (1,)
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    assert ours.coef_.shape == ref.coef_.shape and ours.intercept_.shape == ref.intercept_.shape
    assert np.array_equal(ours.classes_, ref.classes_) and ours.classes_.dtype == ref.classes_.dtype
    assert_close_coef(ours, ref)
    assert np.array_equal(ours.predict(X), ref.predict(X))
    np.testing.assert_allclose(ours.predict_proba(X), ref.predict_proba(X), rtol=0, atol=1e-15)


@pytest.mark.parametrize("C", [1e-2, 1.0, 1e4, np.inf])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_newton_driver_matches_sklearn(C, fit_intercept):
    X, t = make_data()
    ours, ref, ctx, cat_ours, cat_ref = fit_pair(X, t, C=C, fit_intercept=fit_intercept)
    assert cat_ours == cat_ref
    assert_same_model(ours, ref, X)
    if not cat_ref:   # a Newton fit without fallback: the first Hessian pass, then a ladder and a pass per iteration
        assert ctx.passes["ladder"] == ours.n_iter_[0]
    dec = ref.decision_function(X)
    np.testing.assert_allclose(ours.decision_function(X), dec, rtol=0, atol=1e-12 * np.max(np.abs(dec)))
    np.testing.assert_allclose(ours.predict_log_proba(X), ref.predict_log_proba(X), rtol=1e-12)
    assert ours.score(X, t) == ref.score(X, t)


@pytest.mark.parametrize("labels", list(LABELS), ids=list(LABELS))
def test_labels_of_any_dtype(labels):
    X, t = make_data(seed=1)
    y = LABELS[labels][t]
    ours, ref, _, cat_ours, cat_ref = fit_pair(X, y, C=1.0)
    assert cat_ours == cat_ref
    assert_same_model(ours, ref, X)
    assert ours.score(X, y) == ref.score(X, y)
    y_bad = y.copy().astype(object)
    y_bad[:5] = "other"                          # labels outside classes_ count as wrong
    assert ours.score(X, y_bad) == float(np.mean(ref.predict(X) == y_bad))


def test_device_labels_through_the_label_scan():
    X, t = make_data(seed=2)
    y = np.array([-2.0, 5.0], dtype=np.float32)[t]
    ctx = NumpyLogisticContext()
    ours = b2.B200LogisticRegression(ctx=ctx)
    classes, n = ours._device_labels(ctx, y, None, 1)
    assert n == len(y) and classes.dtype == np.float32 and list(classes) == [-2.0, 5.0]
    ref = linear_model.LogisticRegression(solver="newton-cholesky").fit(X, y)
    assert np.array_equal(ref.classes_, classes)


def test_warm_start_matches_sklearn():
    X, t = make_data(seed=3)
    ours = b2.B200LogisticRegression(ctx=NumpyLogisticContext(), warm_start=True, max_iter=2, C=10.0)
    ref = linear_model.LogisticRegression(solver="newton-cholesky", warm_start=True, max_iter=2, C=10.0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours.fit(X, t)
        ref.fit(X, t)
        ours.max_iter = ref.max_iter = 100
        ours.fit(X[:300], t[:300])
        ref.fit(X[:300], t[:300])
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    assert_close_coef(ours, ref)


def test_masked_rows_are_the_fit_of_the_kept_rows():
    X, t = make_data(seed=5)
    y = np.array(["a", "b"])[t]
    mask = (np.arange(len(t)) % 3 != 0).astype(np.uint8)
    Xn, yn = X.copy(), y.astype(object)
    Xn[mask == 0, 0] = np.nan                     # rows not kept may hold anything
    yn[mask == 0] = "c"
    ours = b2.B200LogisticRegression(ctx=NumpyLogisticContext()).fit(Xn, yn, row_mask=mask)
    ref = linear_model.LogisticRegression(solver="newton-cholesky").fit(X[mask == 1], y[mask == 1])
    assert np.array_equal(ours.n_iter_, ref.n_iter_) and list(ours.classes_) == list(ref.classes_)
    assert_close_coef(ours, ref)
    assert ours.score(Xn, yn, row_mask=mask) == ref.score(X[mask == 1], y[mask == 1])


@pytest.mark.parametrize("case", ["collinear", "separable"])
def test_unpenalised_hard_cases_warn_and_fall_back_like_sklearn(case):
    if case == "collinear":
        X, t = make_data(collinear=True, seed=2)
    else:
        X, t = make_data(seed=6, scale=40.0)        # nearly separable: the unpenalised optimum runs away
    ours, ref, _, cat_ours, cat_ref = fit_pair(X, t, C=np.inf)
    assert cat_ref, "scikit-learn was expected to warn"
    assert cat_ours == cat_ref
    assert np.array_equal(ours.n_iter_, ref.n_iter_)
    assert np.array_equal(ours.predict(X), ref.predict(X))
    np.testing.assert_allclose(ours.predict_proba(X), ref.predict_proba(X), rtol=0, atol=1e-6)


def _sk_error(fn):
    with pytest.raises(ValueError) as e:
        fn()
    return str(e.value)


def test_refusals_carry_sklearns_messages():
    X, t = make_data()
    ctx = NumpyLogisticContext()
    sk = lambda **kw: linear_model.LogisticRegression(solver="newton-cholesky", **kw)   # noqa: E731
    ours = lambda **kw: b2.B200LogisticRegression(ctx=ctx, **kw)                        # noqa: E731
    cases = [np.zeros(len(t)), np.arange(len(t)) % 3, np.linspace(0.0, 1.0, len(t))]
    y_nan = t.astype(np.float64)
    y_nan[4] = np.nan
    y_inf = t.astype(np.float64)
    y_inf[4] = np.inf
    cases += [y_nan, y_inf]
    for y in cases:
        msg_ref = _sk_error(lambda: sk().fit(X, y)) if not np.array_equal(y, np.arange(len(t)) % 3) else None
        msg = _sk_error(lambda: ours().fit(X, y))
        if msg_ref is None:
            assert "multinomial fits are not supported" in msg
        else:
            assert msg == msg_ref
    for C in (0, -1.0):
        assert _sk_error(lambda: ours(C=C).fit(X, t)) == _sk_error(lambda: sk(C=C).fit(X, t))
    with pytest.raises(ValueError, match="class_weight"):
        ours(class_weight="balanced").fit(X, t)
    with pytest.raises(ValueError, match="l1_ratio"):
        ours(l1_ratio=0.5).fit(X, t)
    with pytest.raises(ValueError, match="newton-cholesky"):
        ours(solver="lbfgs").fit(X, t)
    with pytest.raises(ValueError, match="sample_weight"):
        ours().fit(X, t, sample_weight=np.ones(len(t)))
    with pytest.raises(ValueError, match="0 sample"):
        ours().fit(X, t, row_mask=np.zeros(len(t), np.uint8))
    Xn = X.copy()
    Xn[3, 1] = np.inf
    with pytest.raises(ValueError, match="NaN, infinity"):
        ours().fit(Xn, t)
    # device labels: the label scan's counts give the same refusals
    st = NumpyLogisticContext()
    for y, match in ((np.zeros(10, np.float32), "only one class: np.float32"),
                     (np.arange(10, dtype=np.float32) % 3, "multinomial"),
                     (np.linspace(0, 1, 10, dtype=np.float32), "continuous"),
                     (np.r_[np.zeros(5), np.ones(4), np.nan].astype(np.float32), "NaN or infinity")):
        with pytest.raises(ValueError, match=match):
            b2.B200LogisticRegression._device_labels(st, y, None, 1)


def test_to_sklearn_is_a_working_sklearn_estimator(tmp_path):
    import joblib
    X, t = make_data()
    y = np.array(["no", "yes"])[t]
    ours = b2.B200LogisticRegression(ctx=NumpyLogisticContext(), C=0.5).fit(X, y)
    path = tmp_path / "m.joblib"
    joblib.dump(ours.to_sklearn(), path)
    clf = joblib.load(path)
    assert isinstance(clf, linear_model.LogisticRegression) and clf.solver == "newton-cholesky"
    np.testing.assert_array_equal(clf.predict_proba(X), ours.predict_proba(X))
    np.testing.assert_array_equal(clf.predict(X), ours.predict(X))
    assert clf.score(X, y) == ours.score(X, y)
