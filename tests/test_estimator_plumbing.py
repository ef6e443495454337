"""The host plumbing every estimator shares, on the CPU: each public estimator (and enet_path / lasso_path) runs on a
recording stand-in for ``Context`` whose device arrays are ``native.DeviceArray`` instances that allocate nothing and
count their ``free()`` calls.  Checked: the wrong-width refusal of predict / score on host and on device rows, the
too-few-rows, non-finite and sample_weight refusals word for word, that every buffer a fit uploads (float64 rows of
65 536 or more with their targets and mask, fold ids and host labels beside device rows) is freed exactly once after
the fit and when the stand-in fails in the middle of it, that warnings point at the caller's line, and the attribute
names and types ``to_sklearn()`` sets."""
import warnings

import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native

D = 4


class FakeArray(native.DeviceArray):
    """A DeviceArray holding its values on the host: no allocation, ``free()`` counted."""

    def __init__(self, ctx, shape, kind, host=None):
        self.ctx, self.shape, self.kind = ctx, tuple(int(s) for s in shape), kind
        self.nbytes = int(np.prod(self.shape, dtype=np.int64)) * self._ITEM[kind]
        self.ptr = 1
        self.host = np.zeros(self.shape, self._NP[kind]) if host is None else np.array(host, self._NP[kind])
        self.frees = 0

    def to_host(self):
        return self.host.copy()

    def free(self):
        self.frees += 1
        self.ptr = None

    def __del__(self):
        pass


def _host(a):
    return a.host if isinstance(a, FakeArray) else np.asarray(a)


class StandIn:
    """Context's entry points with the shapes and types the library returns.  Rows holding NaN give NaN results (as
    the statistic does on the GPU); a fit's passes report a gradient of ``grad`` per kept row (0: converged at once);
    with ``fail`` every entry point but an upload raises.  ``uploads``: the buffers it made."""
    _h = None
    _UPLOADS = ("to_device", "upload_columns", "empty")

    def __init__(self, fail=False, grad=0.0, step=0.0):
        self.uploads, self.fail, self.grad, self.step = [], fail, grad, step
        self.d, self.serial, self.rows, self.nan = 0, 0, 0, False

    def __getattribute__(self, name):
        attr = object.__getattribute__(self, name)
        if callable(attr) and not name.startswith("_") and name not in StandIn._UPLOADS \
                and object.__getattribute__(self, "fail"):
            raise RuntimeError(f"stand-in failure in {name}")
        return attr

    def _rows(self, X, row_mask=None, mask_keep=1):
        self.d = X.shape[1]
        self.nan = not np.all(np.isfinite(_host(X).astype(np.float64)))
        m = None if row_mask is None else _host(row_mask).ravel() == mask_keep
        self.rows = X.shape[0] if m is None else int(m.sum())
        return self.rows

    def _coef(self):
        return np.full(self.d, np.nan if self.nan else 0.1)

    def _out(self, X, shape, kind):
        return FakeArray(self, shape, kind) if isinstance(X, FakeArray) else np.zeros(shape, FakeArray._NP[kind])

    # -- buffers
    def to_device(self, host, kind=None):
        kind = kind or {np.dtype(np.float32): "f32", np.dtype(np.uint8): "u8", np.dtype(np.float64): "f64"}[host.dtype]
        a = FakeArray(self, host.shape, kind, host)
        self.uploads.append(a)
        return a

    def upload_columns(self, columns):
        return self.to_device(np.stack(columns, axis=1).astype(np.float32))

    def empty(self, shape, kind):
        a = FakeArray(self, shape, kind)
        self.uploads.append(a)
        return a

    # -- the statistic and its solves
    def gram_reset(self, d):
        self.d = d

    def gram_accumulate(self, X, y, row_mask=None, mask_keep=1):
        self._rows(X, row_mask, mask_keep)

    def gram_export(self):
        S = np.eye(self.d + 2)
        S[self.d, self.d] = self.rows
        return S

    def fit(self, X, y, row_mask=None, mask_keep=1, alpha=0.0, fit_intercept=True):
        self._rows(X, row_mask, mask_keep)
        return self._coef(), 0.5

    def fit_refined(self, X, y, row_mask=None, mask_keep=1, alpha=0.0, fit_intercept=True, max_passes=2, tol=1e-10):
        coef, b0 = self.fit(X, y, row_mask, mask_keep)
        return coef, b0, 1, self.step

    def solve_eigvals(self, cond=1e-6, fit_intercept=True):
        return np.linspace(2.0, 1.0, self.d), self.d, self.rows

    def solve_spectral(self, cond=1e-6, fit_intercept=True):
        return self._coef(), 0.5, np.linspace(2.0, 1.0, self.d), self.d

    def ridge_loo(self, X, y, alphas, row_mask=None, mask_keep=1, fit_intercept=True, store_cv=False):
        if self._rows(X, row_mask, mask_keep) == 0:
            raise RuntimeError("b2_ridge_loo failed (code -1): no row kept")
        cv = self._out(X, (X.shape[0], len(alphas)), "f64") if store_cv else None
        return np.linspace(1.0, 2.0, len(alphas)), 0, self._coef(), 0.5, cv

    def _path(self, k, max_iter):
        return {"alphas": np.linspace(1.0, 0.1, k), "coefs": np.tile(self._coef(), (k, 1)), "intercepts": np.zeros(k),
                "gaps": np.ones(k), "n_iter": np.full(k, max_iter, np.int32), "tol": 1e-6}

    def solve_enet_path(self, l1_ratio=1.0, alphas=None, n_alphas=100, eps=1e-3, max_iter=1000, tol=1e-4,
                        positive=False, coef_init=None, fit_intercept=True):
        if self.rows == 0:
            raise ValueError("b2_solve_enet_path: no row kept")
        return self._path(n_alphas if alphas is None else len(alphas), max_iter)

    def gram_folds(self, X, y, fold_of_row, n_folds):
        self._rows(X)
        S = np.tile(np.eye(self.d + 2), (n_folds, 1, 1))
        S[:, self.d, self.d] = S[:, self.d + 1, self.d + 1] = 10.0
        return S

    def solve_enet_cv(self, n_folds, l1_ratios=(1.0,), alphas=None, n_alphas=100, eps=1e-3, max_iter=1000, tol=1e-4,
                      positive=False, fit_intercept=True):
        L, A, K = len(l1_ratios), n_alphas, n_folds
        return {"alphas": np.tile(np.linspace(1.0, 0.1, A), (L, 1)), "mse": np.full((L, A, K), np.nan if self.nan else 1.0),
                "n_iter": np.full((L, K, A), max_iter, np.int32), "gaps": np.ones((L, K, A))}

    def residual_moments(self, X, y, coef, intercept, row_mask=None, mask_keep=1, fit_intercept=True):
        return np.zeros(self.d + 2)

    def solve_bayes_ridge(self, *args, **kw):
        return {"coef": self._coef(), "intercept": 0.5, "alpha": 2.0, "lambda": 1.0, "n_iter": 3, "scores": None,
                "sigma": np.eye(self.d)}

    def solve_ard(self, *args, **kw):
        return dict(self.solve_bayes_ridge(), **{"lambda": np.ones(self.d)})

    def score(self, X, coef, intercept, y=None, row_mask=None, mask_keep=1, want_yhat=True, out=None):
        if np.asarray(coef).size != X.shape[1]:                      # the binding's own check
            raise RuntimeError(f"coef has {np.asarray(coef).size} entries, X has {X.shape[1]} columns")
        return self._out(X, (X.shape[0],), "f32"), None

    def score_std(self, X, mean, sigma, noise_var, coef, intercept, want_yhat=True):
        return self._out(X, (X.shape[0],), "f64"), self._out(X, (X.shape[0],), "f64")

    # -- the Newton passes
    def _pass(self, X, y, row_mask, mask_keep, hessian):
        n = self._rows(X, row_mask, mask_keep)
        loss = np.nan if self.nan else float(n)
        return {"loss": loss, "const": 0.0, "sum_y": float(n), "kept": float(n), "y_out_of_range": 0.0,
                "h_nonpos": 0.0, "y_nonfinite": 0.0, "grad": np.full(self.d + 1, self.grad * n), "correct": float(n),
                "hessian": np.eye(self.d + 1) * n if hessian else None}

    def glm_pass(self, X, y, coef, intercept, *, link=0, power=1.0, row_mask=None, mask_keep=1, fit_intercept=True,
                 hessian=True):
        return self._pass(X, y, row_mask, mask_keep, hessian)

    def logistic_pass(self, X, y, coef, intercept, neg_label=0.0, pos_label=1.0, *, row_mask=None, mask_keep=1,
                      fit_intercept=True, hessian=True):
        return self._pass(X, y, row_mask, mask_keep, hessian)

    def glm_line_search(self, *args, n_steps=21, **kw):
        return np.full(n_steps, -1e6)

    logistic_line_search = glm_line_search

    def glm_predict(self, X, coef, intercept, *, link=0):
        return self._out(X, (X.shape[0],), "f64")

    def logistic_predict(self, X, coef, intercept, neg_label=0.0, pos_label=1.0, *, decision=False, proba=False,
                         label=False):
        out = {"decision": self._out(X, (X.shape[0],), "f64"), "proba": self._out(X, (X.shape[0], 2), "f64"),
               "label": self._out(X, (X.shape[0],), "f32")}
        return {k: v for k, v in out.items() if {"decision": decision, "proba": proba, "label": label}[k]}

    def label_scan(self, y, row_mask=None, mask_keep=1):
        v = _host(y) if row_mask is None else _host(y)[_host(row_mask) == mask_keep]
        return {"kept": float(v.size), "nonfinite": 0.0, "nonintegral": 0.0, "min": float(v.min(initial=0.0)),
                "max": float(v.max(initial=0.0)), "n_min": float(np.sum(v == v.min(initial=0.0))),
                "n_max": float(np.sum(v == v.max(initial=0.0)))}


# (class, constructor arguments, targets, the fitted attributes to_sklearn sets and their types)
F, I, A, F64 = float, int, np.ndarray, np.float64
CASES = [
    (b2.B200LinearRegression, {}, "real",
     dict(coef_=A, intercept_=F64, rank_=I, singular_=A, n_features_in_=I)),
    (b2.B200RidgeCV, {"store_cv_results": True}, "real",
     dict(alpha_=F, best_score_=F, coef_=A, intercept_=F64, n_features_in_=I, cv_results_=A)),
    (b2.B200ElasticNet, {"alpha": 0.1}, "real",
     dict(coef_=A, intercept_=F64, dual_gap_=F64, n_iter_=I, n_features_in_=I)),
    (b2.B200Lasso, {"alpha": 0.1}, "real", dict(coef_=A, intercept_=F64, dual_gap_=F64, n_iter_=I, n_features_in_=I)),
    (b2.B200ElasticNetCV, {"cv": 2}, "real",
     dict(alpha_=F, l1_ratio_=F, alphas_=A, mse_path_=A, coef_=A, intercept_=F64, dual_gap_=F64, n_iter_=I,
          n_features_in_=I)),
    (b2.B200LassoCV, {"cv": 2}, "real",
     dict(alpha_=F, alphas_=A, mse_path_=A, coef_=A, intercept_=F64, dual_gap_=F64, n_iter_=I, n_features_in_=I)),
    (b2.B200BayesianRidge, {}, "real",
     dict(coef_=A, intercept_=F64, alpha_=F64, lambda_=F64, sigma_=A, scores_=list, n_iter_=I, X_offset_=A,
          X_scale_=A, n_features_in_=I)),
    (b2.B200ARDRegression, {}, "real",
     dict(coef_=A, intercept_=F64, alpha_=F64, lambda_=A, sigma_=A, scores_=list, n_iter_=I, X_offset_=A,
          X_scale_=A, n_features_in_=I)),
    (b2.B200PoissonRegressor, {}, "count", dict(coef_=A, intercept_=F64, n_iter_=I, n_features_in_=I)),
    (b2.B200GammaRegressor, {}, "count", dict(coef_=A, intercept_=F64, n_iter_=I, n_features_in_=I)),
    (b2.B200TweedieRegressor, {"power": 1.5}, "count", dict(coef_=A, intercept_=F64, n_iter_=I, n_features_in_=I)),
    (b2.B200LogisticRegression, {}, "label",
     dict(coef_=A, intercept_=A, classes_=A, n_iter_=A, n_features_in_=I)),
]
IDS = [c[0].__name__ for c in CASES]
SCORED = (b2.B200PoissonRegressor, b2.B200GammaRegressor, b2.B200TweedieRegressor, b2.B200LogisticRegression)


def data(kind, n=60, d=D, dtype=np.float32, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(dtype)
    y = {"real": rng.normal(size=n), "count": rng.uniform(0.5, 2.0, size=n),
         "label": (np.arange(n) % 2).astype(np.int64)}[kind]
    return X, y


def fitted(cls, kw, kind, ctx=None):
    ctx = ctx or StandIn()
    X, y = data(kind)
    return cls(ctx=ctx, **kw).fit(X, y), ctx


def on_device(ctx, a, kind="f32"):
    return FakeArray(ctx, a.shape, kind, a)


@pytest.mark.parametrize("cls,kw,kind,attrs", CASES, ids=IDS)
@pytest.mark.parametrize("where", ["host", "device"])
def test_wrong_width_is_refused_with_sklearns_message(cls, kw, kind, attrs, where):
    est, ctx = fitted(cls, kw, kind)
    X, y = data(kind, d=D + 1)
    Xw = X if where == "host" else on_device(ctx, X)
    msg = f"X has {D + 1} features, but {cls.__name__} is expecting {D} features as input."
    with pytest.raises(ValueError) as e:
        est.predict(Xw)
    assert str(e.value) == msg
    if cls in SCORED:
        yw = y if where == "host" else on_device(ctx, y.astype(np.float32))
        with pytest.raises(ValueError) as e:
            est.score(Xw, yw)
        assert str(e.value) == msg


def _refusal(fn):
    with pytest.raises(ValueError) as e:
        fn()
    return str(e.value)


@pytest.mark.parametrize("cls,kw,kind,attrs", CASES, ids=IDS)
def test_refusals_carry_their_messages_verbatim(cls, kw, kind, attrs):
    X, y = data(kind)
    name = cls.__name__
    none = np.zeros(len(y), np.uint8)
    if cls in (b2.B200ElasticNetCV, b2.B200LassoCV):
        few = "Cannot have number of splits n_splits=2 greater than the number of samples: n_samples=0."
    elif cls is b2.B200LogisticRegression:
        few = f"Found array with 0 sample(s) (shape=(0,)) while a minimum of 1 is required by {name}."
    else:
        need = 2 if cls is b2.B200ARDRegression else 1
        few = f"Found array with 0 sample(s) (shape=(0, {D})) while a minimum of {need} is required by {name}."
    assert _refusal(lambda: cls(ctx=StandIn(), **kw).fit(X, y, row_mask=none)) == few
    if cls is b2.B200ARDRegression:
        one = (np.arange(len(y)) == 3).astype(np.uint8)
        assert _refusal(lambda: cls(ctx=StandIn(), **kw).fit(X, y, row_mask=one)) == \
            f"Found array with 1 sample(s) (shape=(1, {D})) while a minimum of 2 is required by {name}."
    Xn = X.copy()
    Xn[2, 1] = np.nan
    assert _refusal(lambda: cls(ctx=StandIn(), **kw).fit(Xn, y)) == \
        "Input X or y contains NaN, infinity or a value too large for dtype('float32')."
    if "sample_weight" in cls.fit.__code__.co_varnames:
        assert _refusal(lambda: cls(ctx=StandIn(), **kw).fit(X, y, sample_weight=np.ones(len(y)))) == \
            f"sample_weight is not supported by {name}: every kept row has weight 1"
    if cls in SCORED:
        est, _ = fitted(cls, kw, kind)
        shape = "(0,)" if cls is b2.B200LogisticRegression else f"(0, {D})"
        assert _refusal(lambda: est.score(X, y, row_mask=none)) == \
            f"Found array with 0 sample(s) (shape={shape}) while a minimum of 1 is required."


@pytest.mark.parametrize("fn", [b2.enet_path, b2.lasso_path])
def test_path_refusal(fn):
    X, y = data("real")
    assert _refusal(lambda: fn(X, y, row_mask=np.zeros(len(y), np.uint8), ctx=StandIn())) == \
        f"Found array with 0 sample(s) (shape=(0, {D})) while a minimum of 1 is required by enet_path."


def _upload_cases(cls, kind):
    """(label, X, y, row_mask, the number of buffers the fit uploads) for the staging paths that upload"""
    X64, y64 = data(kind, n=65_536, dtype=np.float64)
    mask = (np.arange(65_536) % 3 != 0).astype(np.uint8)
    out = [("float64 rows", X64, y64, None, 2), ("float64 rows and host mask", X64, y64, mask, 3)]
    if cls in (b2.B200ElasticNetCV, b2.B200LassoCV):
        out = [(label, X, y, m, k + 1) for label, X, y, m, k in out]          # and the fold ids beside device rows
    return out


@pytest.mark.parametrize("cls,kw,kind,attrs", CASES, ids=IDS)
@pytest.mark.parametrize("fail", [False, True], ids=["fit", "failing"])
def test_every_upload_is_freed_once(cls, kw, kind, attrs, fail):
    cases = _upload_cases(cls, kind)
    if cls is b2.B200LogisticRegression:
        X, y = data(kind)
        cases.append(("host labels beside device rows", "device", y, None, 1))
    for label, X, y, mask, n_uploads in cases:
        ctx = StandIn(fail=fail)
        if isinstance(X, str):
            X = on_device(ctx, data(kind)[0])
        est = cls(ctx=ctx, **kw)
        if fail:
            with pytest.raises(RuntimeError, match="stand-in failure"):
                est.fit(X, y, row_mask=mask)
        else:
            est.fit(X, y, row_mask=mask)
        assert len(ctx.uploads) == n_uploads, label
        assert [a.frees for a in ctx.uploads] == [1] * n_uploads, label
        if cls is b2.B200LogisticRegression and not fail and label.startswith("host labels"):
            ctx.uploads.clear()
            est.score(X, y)
            assert [a.frees for a in ctx.uploads] == [1], label


@pytest.mark.parametrize("fn", [b2.enet_path, b2.lasso_path])
@pytest.mark.parametrize("fail", [False, True], ids=["fit", "failing"])
def test_path_uploads_are_freed_once(fn, fail):
    X64, y64 = data("real", n=65_536, dtype=np.float64)
    ctx = StandIn(fail=fail)
    mask = np.ones(65_536, np.uint8)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if fail:
            with pytest.raises(RuntimeError, match="stand-in failure"):
                fn(X64, y64, row_mask=mask, ctx=ctx)
        else:
            fn(X64, y64, row_mask=mask, ctx=ctx)
    assert [a.frees for a in ctx.uploads] == [1, 1, 1]


# the estimators whose fits warn on the stand-in, and how to make them; LassoCV and lasso_path warn from the line of
# their wrapper around ElasticNetCV.fit / enet_path, so only the wrapped calls are checked
WARNING_CASES = [
    (b2.B200LinearRegression, {"refine": 1}, dict(step=1e-3)),
    (b2.B200ElasticNet, {"alpha": 0.1}, {}),
    (b2.B200Lasso, {"alpha": 0.1}, {}),
    (b2.B200ElasticNetCV, {"cv": 2}, {}),
    (b2.B200PoissonRegressor, {"max_iter": 1}, dict(grad=1.0)),
    (b2.B200TweedieRegressor, {"max_iter": 1, "power": 1.5}, dict(grad=1.0)),
    (b2.B200LogisticRegression, {"max_iter": 1}, dict(grad=1.0)),
]


@pytest.mark.parametrize("cls,kw,standin", WARNING_CASES, ids=[c[0].__name__ for c in WARNING_CASES])
def test_warnings_point_at_the_callers_line(cls, kw, standin):
    X, y = data("label" if cls is b2.B200LogisticRegression else "count")
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        cls(ctx=StandIn(**standin), **kw).fit(X, y)
    assert caught
    assert all(w.filename == __file__ for w in caught), [(w.filename, w.lineno) for w in caught]


def test_path_warnings_point_at_the_callers_line():
    X, y = data("real")
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        b2.enet_path(X, y, alphas=3, ctx=StandIn())
    assert len(caught) == 3 and all(w.filename == __file__ for w in caught)


@pytest.mark.parametrize("cls,kw,kind,attrs", CASES, ids=IDS)
def test_to_sklearn_sets_the_fitted_attributes(cls, kw, kind, attrs):
    from sklearn import linear_model
    est, _ = fitted(cls, kw, kind)
    reg = est.to_sklearn()
    assert type(reg) is getattr(linear_model, cls.__name__[4:])
    fitted_names = {k for k in vars(reg) if k.endswith("_") and not k.startswith("_")}
    assert fitted_names == set(attrs)
    assert {k: type(getattr(reg, k)) for k in attrs} == attrs
    for k in attrs:
        v = getattr(reg, k)
        if isinstance(v, np.ndarray):
            assert v is not getattr(est, k) and np.array_equal(v, getattr(est, k))
    if isinstance(est, b2.B200PoissonRegressor) or cls is b2.B200TweedieRegressor:
        assert type(reg._base_loss) is type(reg._get_loss())
