"""The Newton driver of B200PoissonRegressor / B200GammaRegressor / B200TweedieRegressor against scikit-learn 1.9's
``solver="newton-cholesky"``, on the CPU: the estimators run on a numpy stand-in for the context whose three passes
(``glm_pass``, ``glm_line_search``, ``glm_predict``) evaluate scikit-learn's own losses on float64 copies of the staged
float32 rows, so every difference left is the driver's.  Equal n_iter_, coefficients within 1e-12 relative, the same
warning categories on a collinear alpha = 0 case that ends in the L-BFGS fallback."""
import warnings

import numpy as np
import pytest
from sklearn import linear_model
from sklearn._loss.loss import HalfGammaLoss, HalfPoissonLoss, HalfTweedieLoss, HalfTweedieLossIdentity

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native


class NumpyGLMContext:
    """The GLM passes of ``Context`` in numpy: the same unscaled sums, from scikit-learn's pointwise losses."""

    def __init__(self):
        self.passes = {"pass": 0, "hessian": 0, "ladder": 0}

    @staticmethod
    def _loss(link, power):
        if link == native.GLM_IDENTITY:
            return HalfTweedieLossIdentity(power=power)
        return {1.0: HalfPoissonLoss(), 2.0: HalfGammaLoss()}.get(power, HalfTweedieLoss(power=power))

    @staticmethod
    def _rows(X, y, row_mask, mask_keep):
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64)
        if row_mask is not None:
            keep = np.asarray(row_mask) == mask_keep
            X, y = X[keep], y[keep]
        return X, y

    def glm_pass(self, X, y, coef, intercept, *, link, power, row_mask=None, mask_keep=1, fit_intercept=True,
                 hessian=True):
        self.passes["pass"] += 1
        self.passes["hessian"] += int(hessian)
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        loss = self._loss(link, power)
        raw = Xd @ np.asarray(coef, dtype=np.float64) + (intercept if fit_intercept else 0.0)
        with np.errstate(all="ignore"):
            pointwise = loss.loss(y_true=yd, raw_prediction=raw)
            g, h = loss.gradient_hessian(y_true=yd, raw_prediction=raw)
            const = loss.constant_to_optimal_zero(yd)
        iv = loss.interval_y_true          # in_y_true_range's test, row by row
        in_range = (yd >= iv.low if iv.low_inclusive else yd > iv.low) & \
            (yd <= iv.high if iv.high_inclusive else yd < iv.high)
        Z = np.c_[Xd, np.ones(len(yd))]
        return {"loss": float(pointwise.sum()), "const": float(const.sum()), "sum_y": float(yd.sum()),
                "kept": float(len(yd)), "y_out_of_range": float(np.sum(~in_range)), "h_nonpos": float(np.sum(h <= 0)),
                "y_nonfinite": float(np.sum(~np.isfinite(yd))), "grad": Z.T @ g,
                "hessian": Z.T @ (np.abs(h)[:, None] * Z) if hessian else None}

    def glm_line_search(self, X, y, coef, intercept, step, step_intercept, *, link, power, n_steps=21, row_mask=None,
                        mask_keep=1):
        self.passes["ladder"] += 1
        Xd, yd = self._rows(X, y, row_mask, mask_keep)
        loss = self._loss(link, power)
        raw = Xd @ np.asarray(coef, dtype=np.float64) + intercept
        raw_newton = Xd @ np.asarray(step, dtype=np.float64) + step_intercept
        with np.errstate(all="ignore"):
            return np.array([loss.loss(y_true=yd, raw_prediction=raw + 0.5 ** k * raw_newton).sum()
                             for k in range(n_steps)])

    def glm_predict(self, X, coef, intercept, *, link):
        eta = np.asarray(X, dtype=np.float64) @ np.asarray(coef, dtype=np.float64) + intercept
        return np.exp(eta) if link == native.GLM_LOG else eta


# (label, ours, scikit-learn's, extra constructor arguments, target family)
CASES = [
    ("identity p=0", b2.B200TweedieRegressor, linear_model.TweedieRegressor, dict(power=0.0), "normal"),
    ("log p=0", b2.B200TweedieRegressor, linear_model.TweedieRegressor, dict(power=0.0, link="log"), "lognormal"),
    ("poisson", b2.B200PoissonRegressor, linear_model.PoissonRegressor, {}, "poisson"),
    ("tweedie p=1", b2.B200TweedieRegressor, linear_model.TweedieRegressor, dict(power=1.0, link="log"), "poisson"),
    ("tweedie p=1.5", b2.B200TweedieRegressor, linear_model.TweedieRegressor, dict(power=1.5), "compound"),
    ("gamma", b2.B200GammaRegressor, linear_model.GammaRegressor, {}, "gamma"),
    ("tweedie p=3", b2.B200TweedieRegressor, linear_model.TweedieRegressor, dict(power=3.0), "gamma"),
]


def make_data(family, n=400, d=6, seed=0, collinear=False):
    """float32-representable rows and targets (what the estimators stage), returned as float64"""
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 0.5, size=(n, d))
    if collinear:
        X[:, -1] = X[:, 0]
    X = X.astype(np.float32).astype(np.float64)
    beta = rng.uniform(-0.4, 0.4, size=d)
    eta = X @ beta + 0.3
    mu = np.exp(eta)
    if family == "normal":
        y = eta + rng.normal(0.0, 0.3, size=n)
    elif family == "lognormal":
        y = mu + rng.normal(0.0, 0.2, size=n)
    elif family == "poisson":
        y = rng.poisson(mu).astype(np.float64)
    elif family == "compound":
        y = rng.poisson(mu) * rng.gamma(2.0, 0.5, size=n)
    else:
        y = rng.gamma(2.0, mu / 2.0)
    return X, y.astype(np.float32).astype(np.float64)


def assert_close_coef(ours, ref, tol=1e-12):
    scale = max(np.max(np.abs(ref.coef_)), abs(ref.intercept_), 1e-300)
    err = max(np.max(np.abs(ours.coef_ - ref.coef_)), abs(ours.intercept_ - ref.intercept_)) / scale
    assert err <= tol, f"coefficients differ by {err:.3e} relative"


def fit_pair(ours_cls, sk_cls, extra, X, y, **kw):
    ctx = NumpyGLMContext()
    ours = ours_cls(ctx=ctx, **extra, **kw)
    ref = sk_cls(solver="newton-cholesky", **extra, **kw)
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X, y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X, y)
    return ours, ref, ctx, [w.category for w in w_ours], [w.category for w in w_ref]


@pytest.mark.parametrize("label,ours_cls,sk_cls,extra,family", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("alpha", [0.0, 1e-3, 1.0])
@pytest.mark.parametrize("fit_intercept", [True, False])
def test_newton_driver_matches_sklearn(label, ours_cls, sk_cls, extra, family, alpha, fit_intercept):
    X, y = make_data(family)
    ours, ref, ctx, cat_ours, cat_ref = fit_pair(ours_cls, sk_cls, extra, X, y, alpha=alpha,
                                                 fit_intercept=fit_intercept)
    assert ours.n_iter_ == ref.n_iter_
    assert cat_ours == cat_ref
    assert_close_coef(ours, ref)
    assert isinstance(ours.intercept_, type(ref.intercept_)) or not fit_intercept
    if not cat_ref:   # a Newton fit without fallback: two passes per iteration, the ladder and the next Hessian pass
        assert ctx.passes["ladder"] == ours.n_iter_
    np.testing.assert_allclose(ours.predict(X), ref.predict(X), rtol=1e-12)
    assert abs(ours.score(X, y) - ref.score(X, y)) <= 1e-12


@pytest.mark.parametrize("label,ours_cls,sk_cls,extra,family", CASES, ids=[c[0] for c in CASES])
def test_warm_start_matches_sklearn(label, ours_cls, sk_cls, extra, family):
    X, y = make_data(family, seed=3)
    ctx = NumpyGLMContext()
    ours = ours_cls(ctx=ctx, warm_start=True, max_iter=2, alpha=1e-3, **extra)
    ref = sk_cls(solver="newton-cholesky", warm_start=True, max_iter=2, alpha=1e-3, **extra)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours.fit(X, y)
        ref.fit(X, y)
        ours.max_iter = ref.max_iter = 100
        ours.fit(X[:300], y[:300])
        ref.fit(X[:300], y[:300])
    assert ours.n_iter_ == ref.n_iter_
    assert_close_coef(ours, ref)


@pytest.mark.parametrize("label,ours_cls,sk_cls,extra,family", CASES, ids=[c[0] for c in CASES])
def test_masked_rows_are_the_fit_of_the_kept_rows(label, ours_cls, sk_cls, extra, family):
    X, y = make_data(family, seed=5)
    mask = (np.arange(len(y)) % 3 != 0).astype(np.uint8)
    Xn = X.copy()
    Xn[mask == 0, 0] = np.nan                     # rows not kept may hold anything
    ours = ours_cls(ctx=NumpyGLMContext(), alpha=1e-3, **extra).fit(Xn, y, row_mask=mask)
    ref = sk_cls(solver="newton-cholesky", alpha=1e-3, **extra).fit(X[mask == 1], y[mask == 1])
    assert ours.n_iter_ == ref.n_iter_
    assert_close_coef(ours, ref)


def test_collinear_unpenalised_fit_falls_back_to_lbfgs_with_sklearns_warnings():
    X, y = make_data("poisson", collinear=True, seed=2)
    ours, ref, _, cat_ours, cat_ref = fit_pair(b2.B200PoissonRegressor, linear_model.PoissonRegressor, {}, X, y,
                                               alpha=0.0)
    import scipy.linalg
    assert scipy.linalg.LinAlgWarning in cat_ref, cat_ref
    assert cat_ours == cat_ref
    assert ours.n_iter_ == ref.n_iter_
    np.testing.assert_allclose(ours.predict(X), ref.predict(X), rtol=1e-6)


def test_unconverged_fit_warns_like_sklearn():
    X, y = make_data("gamma", seed=4)
    ours, ref, _, cat_ours, cat_ref = fit_pair(b2.B200GammaRegressor, linear_model.GammaRegressor, {}, X, y,
                                               alpha=0.0, max_iter=1, tol=1e-12)
    assert cat_ours == cat_ref and len(cat_ref) == 1
    assert ours.n_iter_ == ref.n_iter_ == 1
    assert_close_coef(ours, ref)


def test_refusals():
    X, y = make_data("poisson")
    ctx = NumpyGLMContext()
    with pytest.raises(ValueError, match="sample_weight"):
        b2.B200PoissonRegressor(ctx=ctx).fit(X, y, sample_weight=np.ones(len(y)))
    with pytest.raises(ValueError, match="lbfgs"):
        b2.B200PoissonRegressor(ctx=ctx, solver="lbfgs").fit(X, y)
    with pytest.raises(ValueError, match="power 0 only"):
        b2.B200TweedieRegressor(ctx=ctx, power=1.5, link="identity").fit(X, y)
    with pytest.raises(ValueError, match="power 0 only"):
        b2.B200TweedieRegressor(ctx=ctx, power=-1.0).fit(X, y)
    with pytest.raises(ValueError, match="0 sample"):
        b2.B200PoissonRegressor(ctx=ctx).fit(X, y, row_mask=np.zeros(len(y), np.uint8))
    Xn = X.copy()
    Xn[3, 1] = np.inf
    with pytest.raises(ValueError, match="NaN, infinity"):
        b2.B200PoissonRegressor(ctx=ctx).fit(Xn, y)
    with pytest.raises(ValueError, match="out of the valid range of the loss 'HalfPoissonLoss'"):
        b2.B200PoissonRegressor(ctx=ctx).fit(X, y - 100.0)
    with pytest.raises(ValueError, match="out of the valid range of the loss 'HalfGammaLoss'"):
        b2.B200GammaRegressor(ctx=ctx).fit(X, np.where(y > 0, y, 0.0) * 0.0)


def test_to_sklearn_is_a_working_sklearn_estimator(tmp_path):
    import joblib
    X, y = make_data("compound")
    ours = b2.B200TweedieRegressor(ctx=NumpyGLMContext(), power=1.5, alpha=0.1).fit(X, y)
    path = tmp_path / "m.joblib"
    joblib.dump(ours.to_sklearn(), path)
    reg = joblib.load(path)
    assert isinstance(reg, linear_model.TweedieRegressor) and reg.solver == "newton-cholesky"
    np.testing.assert_array_equal(reg.predict(X), ours.predict(X))
    assert abs(reg.score(X, y) - ours.score(X, y)) <= 1e-12
