"""The trust-region Newton driver of B200LinearSVC and B200LinearSVR against scikit-learn 1.9's LinearSVC / LinearSVR
with liblinear's primal solver, on the CPU: the estimators run on a numpy stand-in for the context whose ``svm_pass``
restates b2_svm_pass on float64 copies of the staged float32 rows, including the change of the Hessian between the
accepted and the trial point, so every difference left is the driver's.  Equal n_iter_ and warnings, coefficients within
1e-12 relative, the Hessian carried by updates equal to a fresh sum over the active rows at every accepted iteration;
the refusals and the export."""
import io
import warnings

import joblib
import numpy as np
import pytest
from sklearn import svm
from sklearn.exceptions import ConvergenceWarning

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import estimator as est
from test_multinomial_driver import NumpyMultinomialContext


def _active(eta, y, loss, param):
    if loss == b2.native.SVM_SQUARED_HINGE:
        t = np.where(y == param, 1.0, -1.0)
        return 1.0 - t * eta > 0.0
    return np.abs(eta - y) > param


class NumpySvmContext(NumpyMultinomialContext):
    """``svm_pass`` in numpy: the same unscaled sums as b2_svm_pass, eta at both points by the same arithmetic"""

    def __init__(self):
        super().__init__()
        self.passes.update({"svm": 0, "svm_hessian": 0, "svm_changed": 0})
        self.rows = None

    def svm_pass(self, X, y, coef, intercept, *, loss, param, coef_from=None, intercept_from=0.0, row_mask=None,
                 mask_keep=1, fit_intercept=True, hessian=True):
        self.passes["svm"] += 1
        self.passes["svm_hessian"] += int(hessian)
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        self.rows = (Xd, yd)
        n, d = Xd.shape
        Z = np.hstack([Xd, np.ones((n, 1))])
        b = intercept if fit_intercept else 0.0
        eta = Xd @ np.asarray(coef, dtype=np.float64) + b
        act = _active(eta, yd, loss, param)
        if coef_from is None:
            act_f = np.zeros(n, bool)
        else:
            eta_f = Xd @ np.asarray(coef_from, dtype=np.float64) + (intercept_from if fit_intercept else 0.0)
            act_f = _active(eta_f, yd, loss, param)
        if loss == b2.native.SVM_SQUARED_HINGE:
            t = np.where(yd == param, 1.0, -1.0)
            lo, g = (1.0 - t * eta) ** 2, eta - t
        else:
            r = eta - yd
            g = np.where(r > param, r - param, r + param)
            lo = g * g
        sigma = act.astype(float) - act_f.astype(float)
        self.passes["svm_changed"] += int(np.sum(sigma != 0))
        out = {"loss": float(np.sum(lo[act])), "kept": float(n), "active": float(act.sum()),
               "entering": float(np.sum(act & ~act_f)), "leaving": float(np.sum(act_f & ~act)),
               "positive": float(np.sum(yd == param)) if loss == b2.native.SVM_SQUARED_HINGE else 0.0,
               "y_nonfinite": float(np.sum(~np.isfinite(yd))), "grad": Z.T @ np.where(act, g, 0.0),
               "dhessian": (Z * sigma[:, None]).T @ Z if hessian else None}
        return out

    def classify(self, X, coef, intercept, classes, y=None, *, row_mask=None, mask_keep=1, decision=False,
                 label=False):
        """b2_classify: one target picks classes[1] where eta > 0"""
        W = np.atleast_2d(np.asarray(coef, dtype=np.float64))
        if W.shape[0] > 1:
            return super().classify(X, coef, intercept, classes, y, row_mask=row_mask, mask_keep=mask_keep,
                                    decision=decision, label=label)
        eta = np.asarray(X, dtype=np.float64) @ W.T + np.asarray(intercept)
        lab = np.asarray(classes, dtype=np.float32)[(eta[:, 0] > 0).astype(int)]
        out = {"decision": eta} if decision else {}
        if label:
            out["label"] = lab
        if y is not None:
            keep = np.ones(len(lab), bool) if row_mask is None else np.asarray(row_mask) == mask_keep
            out["kept"] = float(keep.sum())
            out["correct"] = float(np.sum(keep & (np.asarray(y, np.float32) == lab)))
        return out

    def glm_predict(self, X, coef, intercept, *, link):
        assert link == b2.native.GLM_IDENTITY
        return np.asarray(X, dtype=np.float64) @ np.asarray(coef, dtype=np.float64) + intercept

    def glm_pass(self, X, y, coef, intercept, *, link, power, row_mask=None, mask_keep=1, fit_intercept=True,
                 hessian=True):
        assert link == b2.native.GLM_IDENTITY and power == 0.0 and not hessian
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        r = Xd @ np.asarray(coef, dtype=np.float64) + intercept - yd
        return {"loss": 0.5 * float(r @ r), "kept": float(yd.size), "sum_y": float(yd.sum()),
                "y_nonfinite": float(np.sum(~np.isfinite(yd)))}


def make_rows(n=400, d=6, seed=0, k=2, noise=0.5):
    """float32-representable rows (as float64) and k classes from a noisy linear score"""
    rng = np.random.default_rng(seed)
    X = (rng.normal(0.0, 1.0, size=(n, d)) + rng.normal(0.0, 0.5, size=d)).astype(np.float32).astype(np.float64)
    S = X @ rng.normal(0.0, 1.0, size=(d, k)) + rng.normal(0.0, noise, size=(n, k))
    t = np.argmax(S, axis=1)
    t[:k] = np.arange(k)
    return X, t


def _fit_both(ours, ref, X, y, **fit_kw):
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X, y, **fit_kw)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X if "row_mask" not in fit_kw else X[fit_kw["row_mask"] == 1],
                y if "row_mask" not in fit_kw else y[fit_kw["row_mask"] == 1])
    return [w.category for w in w_ours], [w.category for w in w_ref]


def _close(a, b, rtol=1e-12):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.max(np.abs(a - b)) <= rtol * max(np.max(np.abs(b)), 1e-300), (a, b)


@pytest.mark.parametrize("k", [2, 3, 10, 32])
@pytest.mark.parametrize("C", [1e-3, 1.0, 100.0])
def test_linear_svc_matches_sklearn(k, C):
    X, t = make_rows(n=60 * k, d=5, seed=k, k=k)
    ctx = NumpySvmContext()
    ours = b2.B200LinearSVC(C=C, ctx=ctx)
    ref = svm.LinearSVC(C=C, dual=False)
    w_ours, w_ref = _fit_both(ours, ref, X, t)
    assert w_ours == w_ref
    assert ours.n_iter_ == ref.n_iter_
    _close(ours.coef_, ref.coef_)
    _close(ours.intercept_, ref.intercept_)
    np.testing.assert_array_equal(ours.classes_, ref.classes_)
    np.testing.assert_array_equal(ours.predict(X), ref.predict(X))
    assert ours.score(X, t) == ref.score(X, t)
    _close(ours.decision_function(X), ref.decision_function(X), 1e-11)
    # one Gram pass: every later class starts without the Hessian
    assert ctx.passes["svm_hessian"] == ctx.passes["svm"] - (k - 1 if k > 2 else 0)


@pytest.mark.parametrize("scaling", [0.5, 1.0, 3.0])
@pytest.mark.parametrize("fit_intercept", [True, False])
@pytest.mark.parametrize("k", [2, 5])
def test_linear_svc_intercept_modes(scaling, fit_intercept, k):
    X, t = make_rows(n=300, d=4, seed=7, k=k)
    ours = b2.B200LinearSVC(C=1.0, fit_intercept=fit_intercept, intercept_scaling=scaling, ctx=NumpySvmContext())
    ref = svm.LinearSVC(C=1.0, dual=False, fit_intercept=fit_intercept, intercept_scaling=scaling)
    w_ours, w_ref = _fit_both(ours, ref, X, t)
    assert w_ours == w_ref and ours.n_iter_ == ref.n_iter_
    _close(ours.coef_, ref.coef_)
    _close(ours.intercept_, ref.intercept_)


LABELS = {"int": np.array([3, 7, 11]), "str": np.array(["a", "b", "c"]), "bool": np.array([False, True]),
          "float": np.array([-1.0, 0.0, 2.0]), "neg": np.array([-2, -1])}


@pytest.mark.parametrize("name", sorted(LABELS))
def test_linear_svc_label_dtypes_and_mask(name):
    vals = LABELS[name]
    X, t = make_rows(n=240, d=3, seed=3, k=vals.size)
    y = vals[t]
    mask = (np.arange(240) % 4 != 1).astype(np.uint8)
    ours = b2.B200LinearSVC(ctx=NumpySvmContext())
    ref = svm.LinearSVC(dual=False)
    _fit_both(ours, ref, X, y, row_mask=mask)
    assert ours.n_iter_ == ref.n_iter_
    _close(ours.coef_, ref.coef_)
    np.testing.assert_array_equal(ours.classes_, ref.classes_)
    np.testing.assert_array_equal(ours.predict(X), ref.predict(X))


def test_linear_svc_max_iter_warning():
    X, t = make_rows(n=200, d=5, seed=11, k=3)
    ours = b2.B200LinearSVC(C=100.0, max_iter=2, ctx=NumpySvmContext())
    ref = svm.LinearSVC(C=100.0, dual=False, max_iter=2)
    w_ours, w_ref = _fit_both(ours, ref, X, t)
    assert ConvergenceWarning in w_ref and w_ours == w_ref
    assert ours.n_iter_ == ref.n_iter_ == 2
    _close(ours.coef_, ref.coef_)


@pytest.mark.parametrize("epsilon", [0.0, 0.5])
@pytest.mark.parametrize("C", [1e-3, 1.0, 100.0])
@pytest.mark.parametrize("fit_intercept,scaling", [(True, 1.0), (True, 3.0), (False, 1.0)])
def test_linear_svr_matches_sklearn(epsilon, C, fit_intercept, scaling):
    rng = np.random.default_rng(5)
    X = rng.normal(0.0, 1.0, size=(300, 6)).astype(np.float32).astype(np.float64)
    y = (X @ rng.normal(0.0, 1.0, size=6) + 1.5 + rng.normal(0.0, 0.7, size=300)).astype(np.float32)
    ours = b2.B200LinearSVR(epsilon=epsilon, C=C, loss="squared_epsilon_insensitive", fit_intercept=fit_intercept,
                            intercept_scaling=scaling, ctx=NumpySvmContext())
    ref = svm.LinearSVR(epsilon=epsilon, C=C, loss="squared_epsilon_insensitive", dual=False,
                        fit_intercept=fit_intercept, intercept_scaling=scaling)
    w_ours, w_ref = _fit_both(ours, ref, X, y.astype(np.float64))
    assert w_ours == w_ref and ours.n_iter_ == ref.n_iter_
    _close(ours.coef_, ref.coef_)
    _close(ours.intercept_, ref.intercept_)
    _close(ours.predict(X), ref.predict(X), 1e-11)


def test_carried_hessian_equals_fresh_sum(monkeypatch):
    """at every accepted iteration the Hessian sum carried by +- updates is the sum over the rows active there"""
    checked = []
    accept = est._SvmProblem.accept

    def checking_accept(self):
        g = accept(self)
        ctx = checking_accept.ctx
        Xd, yd = ctx.rows
        Z = np.hstack([Xd, np.ones((Xd.shape[0], 1))])
        c, _ = self.coef(self.w)
        b = self.scale * self.w[self.d] if self.fi else 0.0
        act = _active(Xd @ c + b, yd, checking_accept.loss, checking_accept.param)
        fresh = Z[act].T @ Z[act]
        assert np.max(np.abs(self.H - fresh)) <= 1e-12 * np.max(np.abs(fresh))
        checked.append(1)
        return g

    monkeypatch.setattr(est._SvmProblem, "accept", checking_accept)
    X, t = make_rows(n=500, d=6, seed=2, k=2)
    checking_accept.ctx = NumpySvmContext()
    checking_accept.loss, checking_accept.param = b2.native.SVM_SQUARED_HINGE, 1.0
    b2.B200LinearSVC(C=10.0, intercept_scaling=2.0, ctx=checking_accept.ctx).fit(X, t)
    n_svc = len(checked)
    y = (X @ np.arange(6.0) + np.random.default_rng(0).normal(size=500)).astype(np.float32)
    checking_accept.ctx = NumpySvmContext()
    checking_accept.loss, checking_accept.param = b2.native.SVM_SQUARED_EPSILON, 0.5
    b2.B200LinearSVR(epsilon=0.5, loss="squared_epsilon_insensitive", ctx=checking_accept.ctx).fit(X, y)
    assert n_svc >= 3 and len(checked) > n_svc


def test_refusals():
    X, t = make_rows(n=50, d=3, k=2)
    ctx = NumpySvmContext()
    cases = [
        (dict(loss="hinge"), "loss='hinge' is not supported"),
        (dict(penalty="l1"), "penalty='l1' is not supported"),
        (dict(dual=True), "dual=True is not supported"),
        (dict(multi_class="crammer_singer"), "crammer_singer"),
        (dict(class_weight="balanced"), "class_weight is not supported"),
        (dict(C=0.0), "The 'C' parameter of LinearSVC"),
        (dict(intercept_scaling=0.0), "Intercept scaling is 0.0 but needs to be greater than 0"),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg.replace("(", r"\(")):
            b2.B200LinearSVC(ctx=ctx, **kw).fit(X, t)
    with pytest.raises(ValueError, match="sample_weight is not supported"):
        b2.B200LinearSVC(ctx=ctx).fit(X, t, sample_weight=np.ones(50))
    with pytest.raises(ValueError, match="the data contains only one class"):
        b2.B200LinearSVC(ctx=ctx).fit(X, np.zeros(50, int))
    with pytest.raises(ValueError, match="at most 32 classes"):
        b2.B200LinearSVC(ctx=ctx).fit(np.tile(X, (1, 1))[:40], np.arange(40))
    with pytest.raises(ValueError, match="Input y contains NaN"):
        b2.B200LinearSVC(ctx=ctx).fit(X, np.where(t == 0, np.nan, 1.0))
    Xn = X.copy()
    Xn[3, 1] = np.inf
    with pytest.raises(ValueError, match="contains NaN, infinity"):
        b2.B200LinearSVC(ctx=ctx).fit(Xn, t)
    with pytest.raises(ValueError, match="dual='auto' selects liblinear's dual solver"):
        b2.B200LinearSVC(ctx=ctx).fit(X[:2], t[:2])
    b2.B200LinearSVC(ctx=ctx, dual=False).fit(np.vstack([X[:2]] * 1), t[:2])   # dual=False: the primal solver
    y = X[:, 0].astype(np.float32)
    with pytest.raises(ValueError, match="loss='epsilon_insensitive' is not supported"):
        b2.B200LinearSVR(ctx=ctx).fit(X, y)
    sq = dict(loss="squared_epsilon_insensitive", ctx=ctx)
    with pytest.raises(ValueError, match="dual=True is not supported"):
        b2.B200LinearSVR(dual=True, **sq).fit(X, y)
    with pytest.raises(ValueError, match="The 'epsilon' parameter of LinearSVR"):
        b2.B200LinearSVR(epsilon=-1.0, **sq).fit(X, y)
    with pytest.raises(ValueError, match="sample_weight is not supported"):
        b2.B200LinearSVR(**sq).fit(X, y, sample_weight=np.ones(50))
    with pytest.raises(ValueError, match="contains NaN, infinity"):
        b2.B200LinearSVR(**sq).fit(X, np.where(y > 0, np.inf, y))


def test_to_sklearn_round_trip():
    X, t = make_rows(n=200, d=4, seed=9, k=3)
    ours = b2.B200LinearSVC(C=0.5, ctx=NumpySvmContext()).fit(X, t)
    buf = io.BytesIO()
    joblib.dump(ours.to_sklearn(), buf)
    buf.seek(0)
    sk = joblib.load(buf)
    assert isinstance(sk, svm.LinearSVC) and sk.n_iter_ == ours.n_iter_
    np.testing.assert_array_equal(sk.predict(X), ours.predict(X))
    y = (X @ np.ones(4)).astype(np.float32)
    r = b2.B200LinearSVR(loss="squared_epsilon_insensitive", ctx=NumpySvmContext()).fit(X, y)
    buf = io.BytesIO()
    joblib.dump(r.to_sklearn(), buf)
    buf.seek(0)
    skr = joblib.load(buf)
    assert isinstance(skr, svm.LinearSVR)
    np.testing.assert_allclose(skr.predict(X), r.predict(X), rtol=1e-12)
    assert abs(r.score(X, y) - skr.score(X, y)) < 1e-9
