"""Estimator-protocol mirror of what stage_1 uses from scikit-learn.

``B200LinearRegression`` keeps the constructor / ``fit`` / ``predict`` / attribute contract of
``sklearn.linear_model.LinearRegression`` as the reference uses it
(stage_1_train_model.py:105-107: ``LinearRegression(fit_intercept=True)``, ``.fit(X_train, y_train)``,
``.predict(X_test)``), with the arithmetic on the H100 through libb2gram.so.  ``alpha`` adds the
ridge term (alpha = 0 == the reference).

``to_sklearn()`` returns a genuine ``sklearn.linear_model.LinearRegression`` carrying our
coefficients: stage_2_serve_model.py:65,78,79 un-pickles the model with only sklearn / numpy /
joblib importable, calls ``.predict`` and ``str(model)`` -- a custom class could not be loaded there.
"""
from __future__ import annotations

import contextlib
import warnings
from typing import Optional

import numpy as np

from . import _native as native

_shared_ctx: Optional[native.Context] = None


def default_context() -> native.Context:
    global _shared_ctx
    if _shared_ctx is None or _shared_ctx._h is None:
        _shared_ctx = native.Context(0)
    return _shared_ctx


_REFINE_TOL = 1e-10             # the refined fit's step tolerance (max_j |dcoef_j| sigma_j / sigma_y)
_F64_UPLOAD_LIMIT = 64 << 30     # float64 host rows larger than this (as fp32, bytes) are converted and streamed block-wise


def _as_f32_matrix(X) -> np.ndarray:
    X = np.asarray(X)
    if X.ndim == 1:
        X = X.reshape(-1, 1)
    if X.ndim != 2:
        raise ValueError(f"Expected 2D array, got {X.ndim}D array instead")
    if X.shape[1] > native.MAX_D:
        raise ValueError(f"at most {native.MAX_D} features are supported, got {X.shape[1]}")
    return np.ascontiguousarray(X, dtype=np.float32)


# ---- the refusals and messages every estimator shares: scikit-learn's wording, which tests and users match on ---------
_NAN_MESSAGE = "Input X or y contains NaN, infinity or a value too large for dtype('float32')."


def _too_few_rows(shape, need: int = 1, by: Optional[str] = None) -> ValueError:
    """check_array's refusal of an input with fewer than ``need`` rows; ``shape``: the kept rows' (n, d) or (n,)."""
    shape = tuple(int(s) for s in shape)
    return ValueError(f"Found array with {shape[0]} sample(s) (shape={shape}) while a minimum of {need} is required"
                      + (f" by {by}." if by else "."))


def _check_finite(*values) -> None:
    """check_array's refusal of non-finite input, which the GPU paths see in what the rows produce (the statistic, the
    solution, the loss)."""
    if not all(np.all(np.isfinite(v)) for v in values):
        raise ValueError(_NAN_MESSAGE)


def _refuse_sample_weight(sample_weight, who: str) -> None:
    if sample_weight is not None:
        raise ValueError(f"sample_weight is not supported by {who}: every kept row has weight 1")


def _check_selection(selection) -> None:
    if selection == "random":
        raise ValueError("selection='random' is not supported: the GPU solver runs sklearn's cyclic order only")
    if selection != "cyclic":
        raise ValueError("selection should be either random or cyclic.")


def _alpha_grid(alphas):
    """(alphas sorted descending, their count), or (None, n) for sklearn's grid of n alphas when ``alphas`` is an int."""
    if isinstance(alphas, (int, np.integer)) and not isinstance(alphas, bool):
        if int(alphas) < 1:
            raise ValueError(f"alphas must be >= 1 when given as an integer, got {int(alphas)}")
        return None, int(alphas)
    al = np.sort(np.asarray(alphas, dtype=np.float64).ravel())[::-1]
    return al, al.size


@contextlib.contextmanager
def _stage_rows(ctx: native.Context, X, y, row_mask):
    """(X, y, row_mask) in a form the context's fit entry points take, for the body of the ``with``: a ``DeviceArray``
    as it is, float64 host rows (65 536 or more) converted on the way up by ``upload_columns`` and resident until the
    ``with`` ends (on success and on error), any other host rows as contiguous float32."""
    owned = []
    try:
        Xh = None if isinstance(X, native.DeviceArray) else np.asarray(X)
        if Xh is not None and Xh.ndim == 2 and Xh.dtype == np.float64 and 0 < Xh.shape[1] <= native.MAX_D \
                and Xh.shape[0] >= 65_536 and Xh.size * 4 <= _F64_UPLOAD_LIMIT:
            # what scikit-learn users hand over: float64 rows.  numpy's astype(float32) is one thread; b2_upload_columns
            # converts with the host threads of the bounce ring beside the H2D copies and leaves the rows resident
            if np.asarray(y).size != Xh.shape[0]:
                raise ValueError(f"Found input variables with inconsistent numbers of samples: "
                                 f"[{Xh.shape[0]}, {np.asarray(y).size}]")
            X = ctx.upload_columns([Xh[:, j] for j in range(Xh.shape[1])])
            owned.append(X)
            y = ctx.to_device(np.ascontiguousarray(np.asarray(y).ravel(), dtype=np.float32))
            owned.append(y)
            if row_mask is not None and not isinstance(row_mask, native.DeviceArray):
                row_mask = ctx.to_device(np.ascontiguousarray(row_mask, dtype=np.uint8))
                owned.append(row_mask)
        elif Xh is not None:
            X = _as_f32_matrix(X)
            y = np.ascontiguousarray(np.asarray(y).ravel(), dtype=np.float32)
            if y.shape[0] != X.shape[0]:
                raise ValueError(f"Found input variables with inconsistent numbers of samples: "
                                 f"[{X.shape[0]}, {y.shape[0]}]")
        yield X, y, row_mask
    finally:
        for a in owned:
            a.free()


@contextlib.contextmanager
def _on_device(ctx: native.Context, host: np.ndarray):
    """``host`` copied to the device for the body of the ``with``."""
    a = ctx.to_device(host)
    try:
        yield a
    finally:
        a.free()


class _B200Estimator:
    """What every estimator shares: its context, the width check of the rows it predicts on, the linear ``predict``
    and the export to scikit-learn.  ``_sk_name``: the scikit-learn class restated (in ``sklearn._sk_module``);
    ``_sk_attrs``: the fitted attributes ``to_sklearn`` copies onto it."""
    _sk_module, _sk_name = "linear_model", ""
    _sk_attrs: tuple = ()

    @property
    def ctx(self) -> native.Context:
        return self._ctx if self._ctx is not None else default_context()

    def _checked_rows(self, X):
        """host rows as contiguous float32, device rows as they are; either must have ``n_features_in_`` columns."""
        X = X if isinstance(X, native.DeviceArray) else _as_f32_matrix(X)
        if X.shape[1] != self.n_features_in_:
            raise ValueError(f"X has {X.shape[1]} features, but {type(self).__name__} is expecting "
                             f"{self.n_features_in_} features as input.")
        return X

    def predict(self, X):
        """X coef_ + intercept_: float64 for host rows, an f32 ``DeviceArray`` for device rows."""
        ctx = self.ctx
        X = self._checked_rows(X)
        yhat, _ = ctx.score(X, self.coef_, float(self.intercept_))
        return yhat if isinstance(X, native.DeviceArray) else yhat.astype(np.float64)

    def _sk_prepare(self, reg) -> None:
        """whatever the export needs beyond copying ``_sk_attrs``"""

    def to_sklearn(self):
        """A real scikit-learn estimator with the attributes ``fit`` would have set (joblib-dumpable; its own
        ``predict`` works)."""
        import importlib
        reg = getattr(importlib.import_module(f"sklearn.{self._sk_module}"), self._sk_name)(**self._sk_params())
        self._sk_prepare(reg)
        for name in self._sk_attrs:
            v = getattr(self, name)
            setattr(reg, name, v.copy() if isinstance(v, np.ndarray) else v)
        return reg


class B200LinearRegression(_B200Estimator):
    """The statistic S = [X 1 y]^T [X 1 y] of a fit lives in the (shared) context while the fit runs; whatever an
    estimator needs of it later -- the next ``partial_fit``, a deferred ``singular_`` / ``rank_`` -- is kept per
    estimator (``_S``) or guarded by the context's serial number, so two estimators on one context never see each
    other's rows."""
    _sk_name = "LinearRegression"
    _sk_attrs = ("coef_", "intercept_", "rank_", "singular_", "n_features_in_")

    def __init__(self, *, fit_intercept: bool = True, alpha: float = 0.0, tol: float = 1e-6,
                 ctx: Optional[native.Context] = None, refine: int = 0):
        self.fit_intercept = fit_intercept
        self.alpha = float(alpha)
        self.tol = tol
        # refine > 0: fit() adds up to `refine` residual passes over the same rows (b2_fit_refined), which take the
        # tensor-core fit to the fp64 least-squares solution on correlated features; 0 keeps the plain fit
        self.refine = int(refine)
        self._ctx = ctx
        self._S: Optional[np.ndarray] = None     # this estimator's statistic (set by partial_fit / deferred attributes)
        self._serial = -1                        # ctx.serial right after this estimator's last fit

    # -- fit -------------------------------------------------------------------------------------
    def _set_solution(self, coef, b0, d: int) -> None:
        _check_finite(coef, b0)
        self.coef_ = coef
        self.intercept_ = np.float64(b0 if self.fit_intercept else 0.0)
        self.n_features_in_ = int(d)

    def _spectrum(self, d: int) -> int:
        """singular_ / rank_ of the statistic resident in the context (eigenvalues only, b2_solve_eigvals); returns the
        number of rows in the statistic."""
        sing, rank, rows = self.ctx.solve_eigvals(cond=self.tol, fit_intercept=self.fit_intercept)
        if rows == 0:
            raise _too_few_rows((0, d), by="B200LinearRegression")
        self.singular_ = sing[: min(rows, d)]
        self.rank_ = int(rank)
        return rows

    def _solve_statistic(self, d: int, solve, with_spectrum: bool) -> None:
        """The model of the statistic that ``solve()`` leaves resident in the context; ``solve`` returns the LDL^T
        solution (coef, intercept) or raises ``LinAlgError`` when a pivot is not positive.

        One rank rule, whichever call produced the statistic: with alpha = 0 the eigenvalue kernel's rank_ decides, and
        the minimum-norm solution gelsd would return (b2_solve_spectral) replaces the LDL^T solution when
        rank_ < min(rows, D) -- the factorisation accepts pivots down to 1e-12 of the largest diagonal entry, while
        sklearn's cond = 1e-6 on the singular values drops eigenvalues below 1e-12 of the largest, so a statistic can
        pass the first test and still be rank deficient.  With alpha > 0 the ridge solution stands and the spectrum
        is computed only if ``with_spectrum``; a statistic the factorisation refuses always gets the minimum-norm
        solution."""
        try:
            coef, b0 = solve()
        except np.linalg.LinAlgError:
            coef, b0 = None, 0.0
        if coef is None or self.alpha == 0.0 or with_spectrum:
            rows = self._spectrum(d)
            if coef is None or (self.alpha == 0.0 and self.rank_ < min(rows, d)):
                coef, b0, _, _ = self.ctx.solve_spectral(cond=self.tol, fit_intercept=self.fit_intercept)
        self._set_solution(coef, b0, d)

    def _drop_spectrum(self) -> None:
        for name in ("singular_", "rank_"):
            if hasattr(self, name):
                delattr(self, name)

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, with_spectrum: bool = True) -> "B200LinearRegression":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16).
        ``row_mask`` (uint8 per row) restricts the fit to rows equal to ``mask_keep``.
        ``with_spectrum=False`` defers ``singular_`` / ``rank_`` (computed on first use, e.g. by ``to_sklearn``) when
        alpha > 0; with alpha = 0 the spectrum decides between the LDL^T and the minimum-norm solution, so it is always
        computed.  Wherever the spectrum is computed, a fit that keeps no rows (e.g. through ``row_mask``) raises
        ``ValueError``, as sklearn does for 0 samples."""
        ctx = self.ctx
        with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
            d = X.shape[1]
            self._S = None
            self._drop_spectrum()

            def solve():
                if self.refine == 0:
                    return ctx.fit(X, y, row_mask, mask_keep, alpha=self.alpha, fit_intercept=self.fit_intercept)
                self.n_refine_passes_, self.refine_step_ = 0, 0.0      # the min-norm fallback stays unrefined
                coef, b0, passes, step = ctx.fit_refined(X, y, row_mask, mask_keep, alpha=self.alpha,
                                                         fit_intercept=self.fit_intercept, max_passes=self.refine,
                                                         tol=_REFINE_TOL)
                self.n_refine_passes_, self.refine_step_ = passes, step
                if step > _REFINE_TOL:
                    warnings.warn(f"refined fit stopped at step {step:.3e} after {passes} kept correction(s) "
                                  f"(tolerance {_REFINE_TOL:.0e}): more passes may help, or the features are too "
                                  "ill-conditioned for the Gram path's precision", RuntimeWarning, stacklevel=4)
                return coef, b0
            self._solve_statistic(d, solve, with_spectrum)
        self._serial = ctx.serial
        return self

    def _no_refine(self, what: str) -> None:
        if self.refine > 0:
            raise ValueError(f"{what} solves from a statistic and has no rows to re-read: refine must be 0 "
                             f"(got refine={self.refine})")

    def partial_fit(self, X, y, with_spectrum: bool = False) -> "B200LinearRegression":
        """Fold one more tranche into THIS estimator's running statistic and re-solve (incremental daily refit)."""
        self._no_refine("partial_fit")
        ctx = self.ctx
        Xh = X if isinstance(X, native.DeviceArray) else _as_f32_matrix(X)
        d = Xh.shape[1]
        if not isinstance(Xh, native.DeviceArray):
            y = np.ascontiguousarray(np.asarray(y).ravel(), dtype=np.float32)
        if self._S is not None and self._S.shape[0] == d + 2:
            ctx.gram_import(self._S)
        elif hasattr(self, "coef_") and self._serial == ctx.serial and ctx.d == d:
            pass                       # the statistic of this estimator's last fit is still resident
        else:
            ctx.gram_reset(d)          # first tranche of this estimator
        ctx.gram_accumulate(Xh, y)
        self._drop_spectrum()
        self._solve_statistic(d, lambda: ctx.solve(alpha=self.alpha, fit_intercept=self.fit_intercept), with_spectrum)
        self._S = ctx.gram_export()
        self._serial = ctx.serial
        return self

    def solve_resident(self, d: int, S: Optional[np.ndarray] = None) -> "B200LinearRegression":
        """Solve from the statistic currently resident in the context (after gram_import / gram_accumulate calls made
        by the caller, e.g. IncrementalTrainer); ``S``: the caller's host copy of it, kept for deferred attributes."""
        self._no_refine("solve_resident")
        ctx = self.ctx
        self._drop_spectrum()
        self._S = S
        self._solve_statistic(d, lambda: ctx.solve(alpha=self.alpha, fit_intercept=self.fit_intercept), False)
        self._serial = ctx.serial
        return self

    def _ensure_spectrum(self) -> None:
        if hasattr(self, "rank_"):
            return
        ctx = self.ctx
        if self._S is not None:
            ctx.gram_import(self._S)
        elif self._serial != ctx.serial:
            raise RuntimeError("singular_ / rank_ were deferred (with_spectrum=False) and the statistic of this fit is no "
                               "longer resident in the context: refit, or fit with with_spectrum=True")
        self._spectrum(self.n_features_in_)
        self._serial = ctx.serial

    # -- artefact ----------------------------------------------------------------------------------------
    def _sk_params(self) -> dict:
        return dict(fit_intercept=self.fit_intercept)

    def _sk_prepare(self, reg) -> None:
        self._ensure_spectrum()

    def __repr__(self) -> str:
        args = ([f"alpha={self.alpha}"] if self.alpha != 0.0 else []) + ([f"refine={self.refine}"] if self.refine else [])
        return f"B200LinearRegression({', '.join(args)})"


def _check_alphas(alphas) -> np.ndarray:
    """sklearn RidgeCV's validation of the grid (same wording)."""
    al = np.asarray(alphas, dtype=np.float64).ravel()
    if al.size == 0:
        raise ValueError("alphas must be a non-empty array-like of floats > 0.0")
    for i, a in enumerate(al):
        if not np.isfinite(a):
            raise ValueError(f"alphas[{i}] == {a}, must be a finite float > 0.0.")
        if a <= 0.0:
            raise ValueError(f"alphas[{i}] == {a}, must be > 0.0.")
    return al


def merge_alpha_chunks(chunks):
    """The first-minimum rule of sklearn's RidgeCV over a grid searched in chunks of at most MAX_ALPHAS alphas:
    ``chunks`` is a list of (offset, mse of the chunk); returns the global index of the first smallest mse."""
    best, best_mse = 0, None
    for off, mse in chunks:
        for k, v in enumerate(np.asarray(mse, dtype=np.float64)):
            if best_mse is None or v < best_mse:
                best, best_mse = off + k, v
    return best


class B200RidgeCV(_B200Estimator):
    """``sklearn.linear_model.RidgeCV(alphas, fit_intercept=..., store_cv_results=...)`` with its default ``cv=None``:
    the alpha with the smallest exact leave-one-out squared error, found on the H100 by ``b2_ridge_loo`` (Gram,
    eigendecomposition and one fp64 pass over the rows per chunk of up to MAX_ALPHAS alphas).  Ties go to the lowest
    index, as in sklearn.  ``to_sklearn()`` returns a genuine RidgeCV carrying the fitted attributes."""
    _sk_name = "RidgeCV"

    def __init__(self, alphas=(0.1, 1.0, 10.0), *, fit_intercept: bool = True, store_cv_results: bool = False,
                 ctx: Optional[native.Context] = None):
        self.alphas = alphas
        self.fit_intercept = fit_intercept
        self.store_cv_results = store_cv_results
        self._ctx = ctx

    def fit(self, X, y, row_mask=None, mask_keep: int = 1) -> "B200RidgeCV":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``.  Sets alpha_, best_score_, coef_, intercept_,
        n_features_in_ and, with store_cv_results, cv_results_ of shape (rows kept, n_alphas)."""
        al = _check_alphas(self.alphas)
        ctx = self.ctx
        with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
            d = X.shape[1]
            chunks, cvs, sols = [], [], []
            for off in range(0, al.size, native.MAX_ALPHAS):
                part = al[off: off + native.MAX_ALPHAS]
                try:
                    mse, best, coef, b0, cv = ctx.ridge_loo(X, y, part, row_mask, mask_keep,
                                                            fit_intercept=self.fit_intercept,
                                                            store_cv=self.store_cv_results)
                except RuntimeError as exc:
                    if "no row kept" in str(exc):
                        raise _too_few_rows((0, d), by="B200RidgeCV") from None
                    raise
                chunks.append((off, mse))
                sols.append((off + best, coef, b0))
                if cv is not None:
                    cvs.append(cv.to_host() if isinstance(cv, native.DeviceArray) else cv)
                    if isinstance(cv, native.DeviceArray):
                        cv.free()
        best = merge_alpha_chunks(chunks)
        mse_all = np.concatenate([m for _, m in chunks])
        coef, b0 = next((c, b) for i, c, b in sols if i == best)
        _check_finite(coef, b0, mse_all[best])
        self.alpha_ = float(al[best])
        self.best_score_ = float(-mse_all[best])
        self.coef_ = coef
        self.intercept_ = np.float64(b0 if self.fit_intercept else 0.0)
        self.n_features_in_ = int(d)
        if self.store_cv_results:
            cv = np.concatenate(cvs, axis=1)
            keep = ~np.isnan(cv[:, 0]) if cv.shape[0] else np.zeros(0, bool)
            self.cv_results_ = cv[keep]
        return self

    @property
    def _sk_attrs(self) -> tuple:
        return ("alpha_", "best_score_", "coef_", "intercept_", "n_features_in_") \
            + (("cv_results_",) if self.store_cv_results else ())

    def _sk_params(self) -> dict:
        return dict(alphas=np.asarray(self.alphas, dtype=np.float64), fit_intercept=self.fit_intercept,
                    store_cv_results=self.store_cv_results)

    def __repr__(self) -> str:
        return f"B200RidgeCV(alphas={self.alphas!r})"


# ---- ElasticNet / Lasso: coordinate descent on the fp64 Gram (b2_solve_enet_path, DESIGN.md section 7) -----------------
_MESSAGE_CONV = ("Objective did not converge. You might want to increase the number of iterations, check the scale of the "
                 "features or consider increasing regularisation.")
_MESSAGE_RIDGE = ("Linear regression models with a zero l1 penalization strength are more efficiently fitted using one of "
                  "the solvers implemented in sklearn.linear_model.Ridge/RidgeCV instead.")


def _gram_of_rows(ctx: native.Context, X, y, row_mask, mask_keep: int) -> int:
    """S of the rows (b2_gram_reset + b2_gram_accumulate: the Gram dispatch every fit uses) left resident; returns D."""
    with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
        ctx.gram_reset(X.shape[1])
        ctx.gram_accumulate(X, y, row_mask, mask_keep)
    return X.shape[1]


def _solve_path(ctx: native.Context, d: int, who: str, **kw) -> dict:
    try:
        return ctx.solve_enet_path(**kw)
    except ValueError as exc:
        if "no row kept" in str(exc):
            raise _too_few_rows((0, d), by=who) from None
        raise


def _warn_unconverged(ctx: native.Context, res: dict, l1_ratio: float, max_iter: int, n: Optional[float] = None) -> None:
    """sklearn's ConvergenceWarning for every alpha that ran out of sweeps above the gap tolerance (its wording, with the
    gap and tolerance on cd_fast's scale: n times the dual_gaps scale).  ``n``: the rows of the path's statistic, None for
    the resident one."""
    late = [i for i in range(res["gaps"].size) if res["n_iter"][i] >= max_iter and res["gaps"][i] > res["tol"]]
    if not late:
        return
    from sklearn.exceptions import ConvergenceWarning
    n = float(ctx.gram_export()[-2, -2]) if n is None else float(n)
    for i in late:
        message = _MESSAGE_CONV + f" Duality gap: {res['gaps'][i] * n:.6e}, tolerance: {res['tol'] * n:.3e}"
        if res["alphas"][i] * l1_ratio * n < np.finfo(np.float64).eps:
            message += "\n" + _MESSAGE_RIDGE
        warnings.warn(message, ConvergenceWarning, stacklevel=3)


class B200ElasticNet(_B200Estimator):
    """``sklearn.linear_model.ElasticNet`` (cyclic selection) fitted on the H100: the rows go through the Gram kernels
    once, then ``b2_solve_enet_path`` runs sklearn's Gram coordinate descent (``precompute=True``) for the one alpha on
    one SM.  Sets coef_, intercept_, dual_gap_, n_iter_ and n_features_in_; ``to_sklearn()`` returns a genuine
    ElasticNet carrying them (``precompute=True``: the Gram solver this fit restates)."""
    _sk_name = "ElasticNet"
    _sk_attrs = ("coef_", "intercept_", "dual_gap_", "n_iter_", "n_features_in_")

    def __init__(self, alpha: float = 1.0, *, l1_ratio: float = 0.5, fit_intercept: bool = True, max_iter: int = 1000,
                 tol: float = 1e-4, positive: bool = False, warm_start: bool = False, selection: str = "cyclic",
                 ctx: Optional[native.Context] = None):
        self.alpha = alpha
        self.l1_ratio = l1_ratio
        self.fit_intercept = fit_intercept
        self.max_iter = max_iter
        self.tol = tol
        self.positive = positive
        self.warm_start = warm_start
        self.selection = selection
        self._ctx = ctx

    def fit(self, X, y, row_mask=None, mask_keep: int = 1):
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``."""
        _check_selection(self.selection)
        if not (np.isfinite(self.alpha) and self.alpha >= 0):
            raise ValueError(f"alpha must be a finite float >= 0, got {self.alpha!r}")
        ctx = self.ctx
        d = _gram_of_rows(ctx, X, y, row_mask, mask_keep)
        coef_init = None
        if self.warm_start and getattr(self, "coef_", None) is not None and np.asarray(self.coef_).size == d:
            coef_init = self.coef_
        res = _solve_path(ctx, d, f"B200{self._sk_name}", l1_ratio=self.l1_ratio, alphas=[float(self.alpha)],
                          max_iter=self.max_iter, tol=self.tol, positive=self.positive, coef_init=coef_init,
                          fit_intercept=self.fit_intercept)
        coef, b0 = res["coefs"][0], float(res["intercepts"][0])
        _check_finite(coef, b0)
        _warn_unconverged(ctx, res, self.l1_ratio, self.max_iter)
        self.coef_ = coef.copy()
        self.intercept_ = np.float64(b0 if self.fit_intercept else 0.0)
        self.dual_gap_ = np.float64(res["gaps"][0])
        self.n_iter_ = int(res["n_iter"][0])
        self.n_features_in_ = int(d)
        return self

    def _sk_params(self) -> dict:
        return dict(alpha=self.alpha, l1_ratio=self.l1_ratio, fit_intercept=self.fit_intercept, precompute=True,
                    max_iter=self.max_iter, tol=self.tol, positive=self.positive, warm_start=self.warm_start,
                    selection=self.selection)

    def __repr__(self) -> str:
        return f"B200{self._sk_name}(alpha={self.alpha}, l1_ratio={self.l1_ratio})"


class B200Lasso(B200ElasticNet):
    """``sklearn.linear_model.Lasso``: B200ElasticNet with l1_ratio = 1."""
    _sk_name = "Lasso"

    def __init__(self, alpha: float = 1.0, *, fit_intercept: bool = True, max_iter: int = 1000, tol: float = 1e-4,
                 positive: bool = False, warm_start: bool = False, selection: str = "cyclic",
                 ctx: Optional[native.Context] = None):
        super().__init__(alpha, l1_ratio=1.0, fit_intercept=fit_intercept, max_iter=max_iter, tol=tol,
                         positive=positive, warm_start=warm_start, selection=selection, ctx=ctx)

    def _sk_params(self) -> dict:
        p = super()._sk_params()
        del p["l1_ratio"]
        return p

    def __repr__(self) -> str:
        return f"B200Lasso(alpha={self.alpha})"


def enet_path(X, y, *, l1_ratio=0.5, eps=1e-3, alphas=100, coef_init=None, return_n_iter=False, positive=False,
              fit_intercept=False, max_iter=1000, tol=1e-4, row_mask=None, mask_keep=1, ctx=None):
    """sklearn 1.9's ``enet_path`` on the H100: one Gram pass over the rows, then the whole path in one launch.
    ``alphas``: an int (the size of sklearn's grid from alpha_max down to alpha_max * eps) or an array (sorted
    descending, as sklearn does).  Returns (alphas, coefs of shape (D, n_alphas), dual_gaps), plus n_iters with
    ``return_n_iter``.  ``fit_intercept=False`` (sklearn's path does not centre) solves on the raw rows; with
    ``fit_intercept=True`` the path runs on the centred Gram and the intercepts of every alpha are appended to the
    returned tuple."""
    ctx = ctx if ctx is not None else default_context()
    al, n_alphas = _alpha_grid(alphas)
    d = _gram_of_rows(ctx, X, y, row_mask, mask_keep)
    res = _solve_path(ctx, d, "enet_path", l1_ratio=l1_ratio, alphas=al, n_alphas=n_alphas, eps=eps,
                      max_iter=max_iter, tol=tol, positive=positive, coef_init=coef_init, fit_intercept=fit_intercept)
    _warn_unconverged(ctx, res, l1_ratio, max_iter)
    out = (res["alphas"], res["coefs"].T.copy(), res["gaps"])
    if return_n_iter:
        out += ([int(k) for k in res["n_iter"]],)
    if fit_intercept:
        out += (res["intercepts"],)
    return out


def lasso_path(X, y, *, eps=1e-3, alphas=100, coef_init=None, return_n_iter=False, positive=False,
               fit_intercept=False, max_iter=1000, tol=1e-4, row_mask=None, mask_keep=1, ctx=None):
    """sklearn 1.9's ``lasso_path``: ``enet_path`` with l1_ratio = 1."""
    return enet_path(X, y, l1_ratio=1.0, eps=eps, alphas=alphas, coef_init=coef_init, return_n_iter=return_n_iter,
                     positive=positive, fit_intercept=fit_intercept, max_iter=max_iter, tol=tol, row_mask=row_mask,
                     mask_keep=mask_keep, ctx=ctx)


# ---- LassoCV / ElasticNetCV: every fold's statistic in one pass, every path in one launch (DESIGN.md section 8) ----------
_MAX_FOLDS = 254
_DROPPED = 255
_CV_RESTRICTION = ("cv must be None, an int, or a splitter / iterable of (train, test) whose test sets partition the "
                   "kept rows and whose train sets are the complements of their test sets (KFold, shuffled or not); "
                   "ShuffleSplit, RepeatedKFold and other overlapping or partial splits are not supported")


def fold_ids(n_rows: int, row_mask=None, mask_keep: int = 1, cv=None):
    """(ids, n_folds): the fold of every row as uint8 (host), dropped rows 255 -- scikit-learn's folds of the kept rows
    numbered 0, 1, ... in order.  ``cv``: None (5), an int k (KFold(k) without shuffling: contiguous folds, the first
    n % k one row longer) or a splitter / iterable of (train, test) over the kept rows whose test sets partition them
    and whose train sets are their complements.  A device ``row_mask`` is copied down (n bytes)."""
    n_rows = int(n_rows)
    if row_mask is None:
        kept = None
        m = n_rows
    else:
        mask = row_mask.to_host() if isinstance(row_mask, native.DeviceArray) else np.asarray(row_mask)
        kept = np.flatnonzero(mask.ravel() == mask_keep)
        m = kept.size
    ids = np.full(n_rows, _DROPPED, dtype=np.uint8)
    sel = slice(None) if kept is None else kept
    if cv is None or (isinstance(cv, (int, np.integer)) and not isinstance(cv, bool)):
        k = 5 if cv is None else int(cv)
        if k < 2:
            raise ValueError(f"k-fold cross-validation requires at least one train/test split by setting n_splits=2 "
                             f"or more, got n_splits={k}.")
        if k > _MAX_FOLDS:
            raise ValueError(f"at most {_MAX_FOLDS} folds are supported, got {k}")
        if m < k:
            raise ValueError(f"Cannot have number of splits n_splits={k} greater than the number of samples: "
                             f"n_samples={m}.")
        sizes = np.full(k, m // k, dtype=np.int64)
        sizes[: m % k] += 1
        ids[sel] = np.repeat(np.arange(k, dtype=np.uint8), sizes)
        return ids, k
    splits = list(cv.split(np.zeros((m, 1)))) if hasattr(cv, "split") else list(cv)
    k = len(splits)
    if k > _MAX_FOLDS:
        raise ValueError(f"at most {_MAX_FOLDS} folds are supported, got {k}")
    if k < 2:
        raise ValueError(_CV_RESTRICTION)
    fold = np.full(m, -1, dtype=np.int64)
    for j, (train, test) in enumerate(splits):
        test = np.asarray(test, dtype=np.int64).ravel()
        if test.size == 0 or np.any(test < 0) or np.any(test >= m) or np.any(fold[test] != -1):
            raise ValueError(_CV_RESTRICTION)
        fold[test] = j
    if np.any(fold < 0):
        raise ValueError(_CV_RESTRICTION)
    for j, (train, test) in enumerate(splits):
        train = np.asarray(train, dtype=np.int64).ravel()
        if train.size != m - np.asarray(test).size or np.any(train < 0) or np.any(train >= m) \
                or np.any(fold[train] == j) or np.unique(train).size != train.size:
            raise ValueError(_CV_RESTRICTION)
    ids[sel] = fold.astype(np.uint8)
    return ids, k


def _fold_tolerances(fold_S: np.ndarray, tol: float, fit_intercept: bool):
    """(rows, tol y_norm2 / n) of each fold's training statistic T_k (the other folds, added in fold order)."""
    K = fold_S.shape[0]
    d = fold_S.shape[1] - 2
    rows, tols = np.empty(K), np.empty(K)
    for k in range(K):
        T = np.zeros_like(fold_S[0])
        for j in range(K):
            if j != k:
                T = T + fold_S[j]
        n = T[d, d]
        ybar = T[d, d + 1] / n if fit_intercept else 0.0
        rows[k], tols[k] = n, tol * (T[d + 1, d + 1] - n * ybar * ybar) / n
    return rows, tols


class B200ElasticNetCV(_B200Estimator):
    """``sklearn.linear_model.ElasticNetCV`` (Gram solver, cyclic selection) on the H100: one pass over the rows gives
    the statistic of every fold (``b2_gram_folds``), one launch runs the path of every (l1_ratio, fold) on the sum of
    the other folds and forms its held-out error from the fold's own statistic (``b2_solve_enet_cv``), and the refit at
    the chosen (alpha, l1_ratio) runs on the summed statistic (``b2_solve_enet_path``).  Sets sklearn's attributes;
    ``to_sklearn()`` returns a genuine ElasticNetCV carrying them (``precompute=True``: the Gram solver this fit
    restates)."""
    _sk_name = "ElasticNetCV"
    _sk_attrs = ("alpha_", "l1_ratio_", "alphas_", "mse_path_", "coef_", "intercept_", "dual_gap_", "n_iter_",
                 "n_features_in_")

    def __init__(self, *, l1_ratio=0.5, eps: float = 1e-3, alphas=100, fit_intercept: bool = True, precompute="auto",
                 max_iter: int = 1000, tol: float = 1e-4, cv=None, positive: bool = False, selection: str = "cyclic",
                 ctx: Optional[native.Context] = None):
        self.l1_ratio = l1_ratio
        self.eps = eps
        self.alphas = alphas
        self.fit_intercept = fit_intercept
        self.precompute = precompute         # accepted for sklearn's signature: the solver always uses the Gram
        self.max_iter = max_iter
        self.tol = tol
        self.cv = cv
        self.positive = positive
        self.selection = selection
        self._ctx = ctx

    def _l1_ratios(self) -> np.ndarray:
        return np.atleast_1d(np.asarray(self.l1_ratio, dtype=np.float64)).ravel()

    def fit(self, X, y, row_mask=None, mask_keep: int = 1):
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit and the folds to rows equal to ``mask_keep``."""
        _check_selection(self.selection)
        l1 = self._l1_ratios()
        al, n_alphas = _alpha_grid(self.alphas)
        if al is None and np.any(l1 == 0.0):
            raise ValueError("Automatic alpha grid generation is not supported for l1_ratio=0. Please supply a "
                             "grid by providing your estimator with the appropriate `alphas=` argument.")
        ctx = self.ctx
        with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
            d = X.shape[1]
            ids, K = fold_ids(X.shape[0], row_mask, mask_keep, self.cv)
            with _on_device(ctx, ids) if isinstance(X, native.DeviceArray) else contextlib.nullcontext(ids) as ids:
                fold_S = ctx.gram_folds(X, y, ids, K)
        res = ctx.solve_enet_cv(K, l1, alphas=al, n_alphas=n_alphas, eps=self.eps, max_iter=self.max_iter,
                                tol=self.tol, positive=self.positive, fit_intercept=self.fit_intercept)
        _check_finite(res["mse"])
        rows, tols = _fold_tolerances(fold_S, self.tol, self.fit_intercept)
        for li in range(l1.size):
            for k in range(K):
                _warn_unconverged(ctx, {"gaps": res["gaps"][li, k], "n_iter": res["n_iter"][li, k], "tol": tols[k],
                                        "alphas": res["alphas"][li]}, float(l1[li]), self.max_iter, n=rows[k])
        # sklearn: the mean over folds, the first minimum per l1_ratio, a later l1_ratio only when strictly better
        mean_mse = np.mean(np.moveaxis(res["mse"], 2, 1), axis=1)
        best_mse, best = np.inf, (0, 0)
        for li in range(l1.size):
            i = int(np.argmin(mean_mse[li]))
            if mean_mse[li, i] < best_mse:
                best_mse, best = mean_mse[li, i], (li, i)
        best_l1, best_alpha = float(l1[best[0]]), float(res["alphas"][best[0], best[1]])
        ref = _solve_path(ctx, d, f"B200{self._sk_name}", l1_ratio=best_l1, alphas=[best_alpha],
                          max_iter=self.max_iter, tol=self.tol, positive=self.positive,
                          fit_intercept=self.fit_intercept)
        coef, b0 = ref["coefs"][0], float(ref["intercepts"][0])
        _check_finite(coef, b0)
        _warn_unconverged(ctx, ref, best_l1, self.max_iter)
        self.alpha_ = best_alpha
        self.l1_ratio_ = best_l1
        self.alphas_ = (res["alphas"][0] if l1.size == 1 else res["alphas"]) if al is None else al.copy()
        self.mse_path_ = np.squeeze(res["mse"])
        self.coef_ = coef.copy()
        self.intercept_ = np.float64(b0 if self.fit_intercept else 0.0)
        self.dual_gap_ = np.float64(ref["gaps"][0])
        self.n_iter_ = int(ref["n_iter"][0])
        self.n_features_in_ = int(d)
        return self

    def _sk_params(self) -> dict:
        cv = self.cv
        if cv is not None and not isinstance(cv, (int, np.integer)) and not hasattr(cv, "split") \
                and not isinstance(cv, (list, tuple)):
            cv = None                          # a one-shot iterator has been consumed by fit
        return dict(l1_ratio=self.l1_ratio, eps=self.eps, alphas=self.alphas, fit_intercept=self.fit_intercept,
                    precompute=True, max_iter=self.max_iter, tol=self.tol, cv=cv, positive=self.positive,
                    selection=self.selection)

    def __repr__(self) -> str:
        return f"B200{self._sk_name}(l1_ratio={self.l1_ratio}, cv={self.cv!r})"


class B200LassoCV(B200ElasticNetCV):
    """``sklearn.linear_model.LassoCV``: B200ElasticNetCV with l1_ratio = 1 (no ``l1_ratio_``)."""
    _sk_name = "LassoCV"
    _sk_attrs = tuple(a for a in B200ElasticNetCV._sk_attrs if a != "l1_ratio_")

    def __init__(self, *, eps: float = 1e-3, alphas=100, fit_intercept: bool = True, precompute="auto",
                 max_iter: int = 1000, tol: float = 1e-4, cv=None, positive: bool = False, selection: str = "cyclic",
                 ctx: Optional[native.Context] = None):
        super().__init__(l1_ratio=1.0, eps=eps, alphas=alphas, fit_intercept=fit_intercept, precompute=precompute,
                         max_iter=max_iter, tol=tol, cv=cv, positive=positive, selection=selection, ctx=ctx)

    def fit(self, X, y, row_mask=None, mask_keep: int = 1):
        super().fit(X, y, row_mask, mask_keep)
        del self.l1_ratio_
        return self

    def _sk_params(self) -> dict:
        p = super()._sk_params()
        del p["l1_ratio"]
        return p

    def __repr__(self) -> str:
        return f"B200LassoCV(cv={self.cv!r})"


# ---- BayesianRidge / ARDRegression: evidence maximisation on the fp64 Gram (DESIGN.md section 9) -------------------------
class _B200Bayes(_B200Estimator):
    """What BayesianRidge and ARDRegression share: a fit is the Gram pass with the least-squares solution w0 (``ctx.fit``;
    the minimum-norm solution when the factorisation refuses), one fp64 pass over the same rows for the anchor
    (``residual_moments`` at w0, which makes the residual sum of squares of every iteration exact), then one solve on the
    resident statistic.  ``predict(X, return_std=True)`` is one fp64 tensor-core pass (``score_std``)."""
    _sk_attrs = ("coef_", "intercept_", "alpha_", "lambda_", "sigma_", "scores_", "n_iter_", "X_offset_", "X_scale_",
                 "n_features_in_")

    def _solve(self, ctx: native.Context, anchor) -> dict:
        raise NotImplementedError

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, sample_weight=None):
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``."""
        _refuse_sample_weight(sample_weight, f"B200{self._sk_name}")
        ctx = self.ctx
        with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
            d = X.shape[1]
            try:
                w0, b0 = ctx.fit(X, y, row_mask, mask_keep, 0.0, fit_intercept=self.fit_intercept)
            except np.linalg.LinAlgError:
                w0, b0, _, _ = ctx.solve_spectral(1e-12, fit_intercept=self.fit_intercept)
            moments = ctx.residual_moments(X, y, w0, b0, row_mask, mask_keep, fit_intercept=self.fit_intercept)
        S = ctx.gram_export()
        n = S[d, d]
        need = 2 if self._sk_name == "ARDRegression" else 1
        if not n >= need:
            raise _too_few_rows((n, d), need, by=f"B200{self._sk_name}")
        res = self._solve(ctx, np.concatenate([w0, moments]))
        _check_finite(res["coef"], res["intercept"], res["alpha"])
        self.coef_ = res["coef"]
        self.intercept_ = np.float64(res["intercept"] if self.fit_intercept else 0.0)
        self.alpha_ = np.float64(res["alpha"])
        self.n_iter_ = int(res["n_iter"])
        self.X_offset_ = S[:d, d] / n if self.fit_intercept else np.zeros(d)
        self.X_scale_ = np.ones(d)
        self.n_features_in_ = int(d)
        self.scores_ = np.asarray(res["scores"]) if self.compute_score else []
        self._set_posterior(res)
        return self

    def _full_sigma(self) -> np.ndarray:
        return self.sigma_

    def predict(self, X, return_std: bool = False):
        """The linear prediction; with ``return_std`` (yhat, ystd) from one fp64 pass, float64 for host rows and f64
        ``DeviceArray``s for device rows."""
        if not return_std:
            return super().predict(X)
        ctx = self.ctx
        return ctx.score_std(self._checked_rows(X), self.X_offset_, self._full_sigma(), 1.0 / float(self.alpha_),
                             self.coef_, float(self.intercept_))


class B200BayesianRidge(_B200Bayes):
    """``sklearn.linear_model.BayesianRidge`` fitted on the H100: ``b2_solve_bayes_ridge`` runs scikit-learn 1.9's
    iteration in the eigenbasis of the fp64 centred Gram.  Sets coef_, intercept_, alpha_, lambda_, sigma_, scores_ (with
    compute_score), n_iter_, X_offset_, X_scale_ and n_features_in_.  copy_X and verbose have no effect."""
    _sk_name = "BayesianRidge"

    def __init__(self, *, max_iter: int = 300, tol: float = 1e-3, alpha_1: float = 1e-6, alpha_2: float = 1e-6,
                 lambda_1: float = 1e-6, lambda_2: float = 1e-6, alpha_init=None, lambda_init=None,
                 compute_score: bool = False, fit_intercept: bool = True, copy_X: bool = True, verbose: bool = False,
                 ctx: Optional[native.Context] = None):
        self.max_iter = max_iter
        self.tol = tol
        self.alpha_1 = alpha_1
        self.alpha_2 = alpha_2
        self.lambda_1 = lambda_1
        self.lambda_2 = lambda_2
        self.alpha_init = alpha_init
        self.lambda_init = lambda_init
        self.compute_score = compute_score
        self.fit_intercept = fit_intercept
        self.copy_X = copy_X
        self.verbose = verbose
        self._ctx = ctx

    def _solve(self, ctx, anchor):
        return ctx.solve_bayes_ridge(self.alpha_1, self.alpha_2, self.lambda_1, self.lambda_2, self.alpha_init,
                                     self.lambda_init, max_iter=self.max_iter, tol=self.tol, anchor=anchor,
                                     compute_score=self.compute_score, fit_intercept=self.fit_intercept)

    def _set_posterior(self, res: dict) -> None:
        self.lambda_ = np.float64(res["lambda"])
        self.sigma_ = res["sigma"]

    def _sk_params(self) -> dict:
        return dict(max_iter=self.max_iter, tol=self.tol, alpha_1=self.alpha_1, alpha_2=self.alpha_2,
                    lambda_1=self.lambda_1, lambda_2=self.lambda_2, alpha_init=self.alpha_init,
                    lambda_init=self.lambda_init, compute_score=self.compute_score, fit_intercept=self.fit_intercept,
                    copy_X=self.copy_X, verbose=self.verbose)

    def __repr__(self) -> str:
        return "B200BayesianRidge()"


class B200ARDRegression(_B200Bayes):
    """``sklearn.linear_model.ARDRegression`` fitted on the H100: ``b2_solve_ard`` runs scikit-learn 1.9's iteration,
    pruning included, in one single-SM launch on the fp64 statistic.  Sets sklearn's attributes; sigma_ is kept x kept
    ((0, 0) when every feature is pruned).  copy_X and verbose have no effect."""
    _sk_name = "ARDRegression"

    def __init__(self, *, max_iter: int = 300, tol: float = 1e-3, alpha_1: float = 1e-6, alpha_2: float = 1e-6,
                 lambda_1: float = 1e-6, lambda_2: float = 1e-6, compute_score: bool = False,
                 threshold_lambda: float = 1e4, fit_intercept: bool = True, copy_X: bool = True, verbose: bool = False,
                 ctx: Optional[native.Context] = None):
        self.max_iter = max_iter
        self.tol = tol
        self.alpha_1 = alpha_1
        self.alpha_2 = alpha_2
        self.lambda_1 = lambda_1
        self.lambda_2 = lambda_2
        self.compute_score = compute_score
        self.threshold_lambda = threshold_lambda
        self.fit_intercept = fit_intercept
        self.copy_X = copy_X
        self.verbose = verbose
        self._ctx = ctx

    def _solve(self, ctx, anchor):
        return ctx.solve_ard(self.alpha_1, self.alpha_2, self.lambda_1, self.lambda_2,
                             threshold_lambda=self.threshold_lambda, max_iter=self.max_iter, tol=self.tol,
                             anchor=anchor, compute_score=self.compute_score, fit_intercept=self.fit_intercept)

    def _set_posterior(self, res: dict) -> None:
        self.lambda_ = np.asarray(res["lambda"], dtype=np.float64)
        keep = self.lambda_ < self.threshold_lambda
        self.sigma_ = res["sigma"][np.ix_(keep, keep)].copy()

    def _full_sigma(self) -> np.ndarray:
        keep = self.lambda_ < self.threshold_lambda
        full = np.zeros((self.n_features_in_, self.n_features_in_))
        full[np.ix_(keep, keep)] = self.sigma_
        return full

    def _sk_params(self) -> dict:
        return dict(max_iter=self.max_iter, tol=self.tol, alpha_1=self.alpha_1, alpha_2=self.alpha_2,
                    lambda_1=self.lambda_1, lambda_2=self.lambda_2, compute_score=self.compute_score,
                    threshold_lambda=self.threshold_lambda, fit_intercept=self.fit_intercept, copy_X=self.copy_X,
                    verbose=self.verbose)

    def __repr__(self) -> str:
        return "B200ARDRegression()"


# ---- PoissonRegressor / GammaRegressor / TweedieRegressor: Newton fits on GPU passes (DESIGN.md section 10) ------------
class _B200GLM(_B200Estimator):
    """What the three generalised linear regressors share: scikit-learn 1.9's ``_GeneralizedLinearRegressor.fit`` with
    ``solver="newton-cholesky"``, its ``NewtonSolver.solve`` restated on the host around GPU passes over the rows.  Each
    Newton iteration is one pass for the loss, gradient and fp64 Hessian (``glm_pass``) and one pass for all 21 candidate
    steps of the backtracking line search (``glm_line_search``); the (D + 1)^2 Newton solve, the Armijo rule and the
    convergence tests run on the host as scikit-learn runs them.  A singular Hessian, a Hessian with many non-positive
    pointwise values, a step that is not a descent direction or a failed line search hand over to L-BFGS-B on GPU
    loss-and-gradient passes, with scikit-learn's warnings.

    The fit is the float64 fit of the stored fp32 / bf16 values: it matches scikit-learn run on float64 copies of those
    values (scikit-learn computes float32 input in float32).  ``B200LogisticRegression`` runs the same ``fit`` with its
    own hooks."""
    _sk_attrs = ("coef_", "intercept_", "n_iter_", "n_features_in_")

    def _link_power(self):
        """(link, power, the name of scikit-learn's loss class)"""
        raise NotImplementedError

    def _sk_params(self) -> dict:
        return dict(alpha=self.alpha, fit_intercept=self.fit_intercept, solver=self.solver, max_iter=self.max_iter,
                    tol=self.tol, warm_start=self.warm_start, verbose=self.verbose)

    def _check_params(self):
        if self.solver != "newton-cholesky":
            raise ValueError(f"solver={self.solver!r} is not supported: B200{self._sk_name} runs scikit-learn's "
                             "'newton-cholesky' solver (L-BFGS-B runs only as its fallback)")
        if not (np.isfinite(self.alpha) and self.alpha >= 0):
            raise ValueError(f"The 'alpha' parameter of {self._sk_name} must be a float in the range [0.0, inf). "
                             f"Got {self.alpha!r} instead.")
        if isinstance(self.max_iter, bool) or not isinstance(self.max_iter, (int, np.integer)) or self.max_iter < 1:
            raise ValueError(f"The 'max_iter' parameter of {self._sk_name} must be an int in the range [1, inf). "
                             f"Got {self.max_iter!r} instead.")
        if not (np.isfinite(self.tol) and self.tol > 0):
            raise ValueError(f"The 'tol' parameter of {self._sk_name} must be a float in the range (0.0, inf). "
                             f"Got {self.tol!r} instead.")
        return self._link_power()

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, sample_weight=None):
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``.  Sets coef_, intercept_, n_iter_ and
        n_features_in_."""
        _refuse_sample_weight(sample_weight, type(self).__name__)
        model = self._check_params()
        with self._stage_targets(X, y, row_mask, mask_keep) as (X, y, row_mask, labels):
            d = X.shape[1]
            run, line_search = self._passes(X, y, row_mask, mask_keep, model, labels)
            coef, n_iter = self._newton(d, self._l2(labels), lambda: self._start(d, run, model, labels), run,
                                        line_search, **self._layout(d, labels))
        self._store(coef, n_iter, d, labels)
        return self

    # -- the hooks of fit: (X, y, row_mask, labels) staged; the pass pair; the start; the L2 strength; the attributes --
    @contextlib.contextmanager
    def _stage_targets(self, X, y, row_mask, mask_keep):
        with _stage_rows(self.ctx, X, y, row_mask) as rows:
            yield rows + (None,)

    def _passes(self, X, y, row_mask, mask_keep, model, labels):
        """(run(coef, hessian), line_search(coef, step)) as ``_newton`` takes them"""
        ctx, fi, d = self.ctx, bool(self.fit_intercept), X.shape[1]
        link, power, _ = model

        def run(c, hessian):
            return ctx.glm_pass(X, y, c[:d], float(c[d]) if fi else 0.0, link=link, power=power, row_mask=row_mask,
                                mask_keep=mask_keep, fit_intercept=fi, hessian=hessian)

        def line_search(c, step):
            return ctx.glm_line_search(X, y, c[:d], float(c[d]) if fi else 0.0, step[:d],
                                       float(step[d]) if fi else 0.0, link=link, power=power,
                                       n_steps=native.GLM_STEPS, row_mask=row_mask, mask_keep=mask_keep)
        return run, line_search

    def _start(self, d, run, model, labels):
        """the first pass checks y; the intercept starts at link(mean y)"""
        link, _, loss_name = model
        coef, warm = self._start_coef(d)
        first = run(coef, warm)
        n = first["kept"]
        if n == 0:
            raise _too_few_rows((0, d), by=f"B200{self._sk_name}")
        if first["y_nonfinite"] > 0:
            raise ValueError(_NAN_MESSAGE)
        _check_finite(first["loss"], first["grad"])
        if first["y_out_of_range"] > 0:
            raise ValueError(f"Some value(s) of y are out of the valid range of the loss {loss_name!r}.")
        if warm:
            return coef, first, n
        if self.fit_intercept:
            ybar = first["sum_y"] / n
            coef[-1] = np.log(ybar) if link == native.GLM_LOG else ybar
        return coef, run(coef, True), n

    def _l2(self, labels) -> float:
        return float(self.alpha)

    def _layout(self, d, labels) -> dict:
        """the coefficient layout ``_newton`` takes beyond one row [w, b] (its defaults)"""
        return {}

    def _store(self, coef, n_iter, d, labels) -> None:
        if self.fit_intercept:
            self.coef_, self.intercept_ = coef[:-1].copy(), np.float64(coef[-1])
        else:
            self.coef_, self.intercept_ = coef.copy(), 0.0
        self.n_iter_ = int(n_iter)
        self.n_features_in_ = int(d)

    def _start_coef(self, d):
        """(the starting coefficients with the intercept last, zeros unless warm_start finds a fit; warm)"""
        fi = bool(self.fit_intercept)
        warm = bool(self.warm_start) and getattr(self, "coef_", None) is not None
        if not warm:
            return np.zeros(d + int(fi)), False
        coef = np.asarray(self.coef_, dtype=np.float64).ravel().copy()
        if coef.size != d:
            raise ValueError(f"X has {d} features, but the warm start coef_ has {coef.size}")
        if fi:
            coef = np.concatenate([coef, [float(np.ravel(self.intercept_)[0])]])
        return coef, True

    def _newton(self, d, alpha, start, run, line_search, n_classes=1, free=None):
        """NewtonSolver.solve (NewtonCholeskySolver) step by step on the caller's passes: start() -> (coef, the pass
        with the Hessian at coef, the kept rows), run(coef, hessian) -> the pass sums at coef, line_search(coef, step)
        -> the loss sums of the 21 ladder steps.  The coefficients are scikit-learn's: n_classes rows [w, b] raveled
        with the classes of one feature contiguous (order "F"), so the weights come first; the pass's "grad" holds the
        n_classes rows of sum g [x 1] and its "hessian" is in the same order.  free: None, or the coefficients the Newton
        step solves for, the others held where they are (NewtonCholeskySolver's gauge of an overparametrised multinomial
        fit).  Returns (coef, n_iter)."""
        import scipy.linalg
        import scipy.optimize
        from sklearn.exceptions import ConvergenceWarning
        from sklearn.utils.optimize import _check_optimize_result
        fi, tol, max_iter = bool(self.fit_intercept), float(self.tol), int(self.max_iter)
        n_dof = d + int(fi)
        n_w = n_classes * d                       # the weights, before the intercepts

        def loss_of(c, loss_sum):                 # LinearModelLoss.loss: mean loss + alpha / 2 |w|^2
            w = c[:n_w]
            return float(loss_sum / n) + float(0.5 * alpha * (w @ w))

        def grad_of(c, s):                        # LinearModelLoss.gradient
            G = np.reshape(s["grad"], (n_classes, -1))
            W = np.reshape(c, (n_classes, n_dof), order="F")
            g = np.empty((n_classes, n_dof))
            g[:, :d] = G[:, :d] / n + alpha * W[:, :d]
            if fi:
                g[:, d] = G[:, d] / n
            return g.ravel(order="F")

        coef, cur, n = start()
        loss_value = loss_of(coef, cur["loss"])

        beta, sigma = 0.5, 0.00048828125
        eps = 16 * np.finfo(np.float64).eps
        iteration, converged, fallback = 1, False, False
        while iteration <= max_iter and not converged:
            fallback = False
            gradient = grad_of(coef, cur)
            # inner_solve
            if cur["h_nonpos"] / n > 0.25:
                warnings.warn(f"The inner solver of NewtonCholeskySolver detected a pointwise hessian with many negative "
                              f"values at iteration #{iteration}. It will now resort to lbfgs instead.",
                              ConvergenceWarning, stacklevel=3)
                fallback = True
                break
            hessian = cur["hessian"] / n
            if not fi:
                hessian = hessian[:n_w, :n_w].copy()
            hessian[np.arange(n_w), np.arange(n_w)] += alpha
            if free is None:
                h_free, g_free = hessian, gradient
            else:                                 # the held coefficients leave the gradient and the Hessian
                held = np.setdiff1d(np.arange(gradient.size), free)
                gradient[held] = 0
                hessian[held, :] = 0
                hessian[:, held] = 0
                h_free, g_free = hessian[np.ix_(free, free)], gradient[free]
            try:
                with warnings.catch_warnings():
                    warnings.simplefilter("error", scipy.linalg.LinAlgWarning)
                    coef_newton = scipy.linalg.solve(h_free, -g_free, check_finite=False, assume_a="sym")
                    if free is not None:
                        coef_newton, step_free = np.zeros(gradient.size), coef_newton
                        coef_newton[free] = step_free
                    gradient_times_newton = gradient @ coef_newton
                    if gradient_times_newton > 0:
                        fallback = True
                        break
            except (np.linalg.LinAlgError, scipy.linalg.LinAlgWarning) as e:
                warnings.warn("The inner solver of NewtonCholeskySolver stumbled upon a singular or very ill-conditioned "
                              f"Hessian matrix at iteration {iteration}. It will now resort to lbfgs instead.\n"
                              "Further options are to use another solver or to avoid such situation in the first place. "
                              "Possible remedies are removing collinear features of X or increasing the penalization "
                              "strengths.\nThe original Linear Algebra message was:\n" + str(e),
                              scipy.linalg.LinAlgWarning, stacklevel=3)
                fallback = True
                break
            # line search: every candidate step from one pass
            ladder = line_search(coef, coef_newton)
            armijo_term = sigma * gradient_times_newton
            coef_old, loss_value_old, gradient_old = coef, loss_value, gradient
            sum_abs_grad_old = -1
            t = 1
            for i in range(native.GLM_STEPS):
                coef = coef_old + t * coef_newton
                loss_value = loss_of(coef, ladder[i])
                loss_improvement = loss_value - loss_value_old
                if loss_improvement <= t * armijo_term:
                    break
                if np.abs(loss_improvement) <= np.abs(loss_value_old * eps):
                    if sum_abs_grad_old < 0:
                        sum_abs_grad_old = scipy.linalg.norm(gradient_old, ord=1)
                    if scipy.linalg.norm(grad_of(coef, run(coef, False)), ord=1) < sum_abs_grad_old:
                        break
                t *= beta
            else:
                warnings.warn(f"Line search of Newton solver NewtonCholeskySolver at iteration #{iteration} did not "
                              "converge after 21 line search refinement iterations. It will now resort to lbfgs "
                              "instead.", ConvergenceWarning, stacklevel=3)
                fallback = True
                break
            # convergence: the gradient at the new coefficients comes with the next iteration's Hessian
            cur = run(coef, iteration < max_iter)
            if np.max(np.abs(grad_of(coef, cur))) <= tol:
                if 0.5 * (coef_newton @ hessian @ coef_newton) <= tol:
                    converged = True
            iteration += 1

        if not converged:
            if fallback:
                def fun(c):
                    s = run(c, False)
                    return loss_of(c, s["loss"]), grad_of(c, s)
                maxiter = max_iter - iteration
                opt_res = scipy.optimize.minimize(fun, coef, method="L-BFGS-B", jac=True,
                                                  options={"maxiter": maxiter, "maxls": 50, "gtol": tol,
                                                           "ftol": 64 * np.finfo(np.float64).eps})
                iteration += _check_optimize_result("lbfgs", opt_res, max_iter=maxiter)
                coef = opt_res.x
            else:
                warnings.warn(f"Newton solver did not converge after {iteration - 1} iterations.", ConvergenceWarning,
                              stacklevel=3)
        return coef, iteration - 1

    def predict(self, X):
        """mu = exp(X coef_ + intercept_) (log link) or X coef_ + intercept_ in fp64: float64 for host rows, an f64
        ``DeviceArray`` for device rows."""
        link = self._link_power()[0]
        return self.ctx.glm_predict(self._checked_rows(X), self.coef_, float(self.intercept_), link=link)

    def score(self, X, y, row_mask=None, mask_keep: int = 1):
        """D^2, the fraction of deviance explained (scikit-learn's ``score``): one pass at the model and one at the
        intercept-only model link(mean y), both over the kept rows."""
        link, power, loss_name = self._link_power()
        ctx = self.ctx
        with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
            d = self._checked_rows(X).shape[1]
            kw = dict(link=link, power=power, row_mask=row_mask, mask_keep=mask_keep, hessian=False)
            model = ctx.glm_pass(X, y, self.coef_, float(self.intercept_), **kw)
            n = model["kept"]
            if n == 0:
                raise _too_few_rows((0, d))
            if model["y_nonfinite"] > 0:
                raise ValueError(_NAN_MESSAGE)
            if model["y_out_of_range"] > 0:
                raise ValueError(f"Some value(s) of y are out of the valid range of the loss {loss_name!r}.")
            ybar = model["sum_y"] / n
            y_mean = np.log(ybar) if link == native.GLM_LOG else ybar
            null = ctx.glm_pass(X, y, np.zeros(d), float(y_mean), **kw)
        constant = model["const"] / n
        deviance, deviance_null = model["loss"] / n, null["loss"] / n
        return float(1 - (deviance + constant) / (deviance_null + constant))

    def _sk_prepare(self, reg) -> None:
        reg._base_loss = reg._get_loss()          # scikit-learn's fit sets it; its predict and score read it

    def __repr__(self) -> str:
        return f"B200{self._sk_name}(alpha={self.alpha})"


class B200PoissonRegressor(_B200GLM):
    """``sklearn.linear_model.PoissonRegressor(solver="newton-cholesky")`` fitted on the H100: HalfPoissonLoss with the
    log link.  verbose is accepted and has no effect."""
    _sk_name = "PoissonRegressor"

    def __init__(self, *, alpha: float = 1.0, fit_intercept: bool = True, solver: str = "newton-cholesky",
                 max_iter: int = 100, tol: float = 1e-4, warm_start: bool = False, verbose: int = 0,
                 ctx: Optional[native.Context] = None):
        self.alpha = alpha
        self.fit_intercept = fit_intercept
        self.solver = solver
        self.max_iter = max_iter
        self.tol = tol
        self.warm_start = warm_start
        self.verbose = verbose
        self._ctx = ctx

    def _link_power(self):
        return native.GLM_LOG, 1.0, "HalfPoissonLoss"


class B200GammaRegressor(B200PoissonRegressor):
    """``sklearn.linear_model.GammaRegressor(solver="newton-cholesky")`` fitted on the H100: HalfGammaLoss with the log
    link.  verbose is accepted and has no effect."""
    _sk_name = "GammaRegressor"

    def _link_power(self):
        return native.GLM_LOG, 2.0, "HalfGammaLoss"


class B200TweedieRegressor(_B200GLM):
    """``sklearn.linear_model.TweedieRegressor(power, link, solver="newton-cholesky")`` fitted on the H100:
    HalfTweedieLoss (log link) at any power, HalfTweedieLossIdentity (identity link, the default for power <= 0) at power
    0 only.  verbose is accepted and has no effect."""
    _sk_name = "TweedieRegressor"

    def __init__(self, *, power: float = 0.0, alpha: float = 1.0, fit_intercept: bool = True, link: str = "auto",
                 solver: str = "newton-cholesky", max_iter: int = 100, tol: float = 1e-4, warm_start: bool = False,
                 verbose: int = 0, ctx: Optional[native.Context] = None):
        self.power = power
        self.alpha = alpha
        self.fit_intercept = fit_intercept
        self.link = link
        self.solver = solver
        self.max_iter = max_iter
        self.tol = tol
        self.warm_start = warm_start
        self.verbose = verbose
        self._ctx = ctx

    def _link_power(self):
        power = float(self.power)
        if not np.isfinite(power):
            raise ValueError(f"The 'power' parameter of TweedieRegressor must be a finite float. Got {self.power!r}.")
        if self.link not in ("auto", "identity", "log"):
            raise ValueError(f"The 'link' parameter of TweedieRegressor must be a str among {{'auto', 'identity', "
                             f"'log'}}. Got {self.link!r} instead.")
        identity = self.link == "identity" or (self.link == "auto" and power <= 0)
        if identity and power != 0.0:
            raise ValueError(f"link='identity' (or link='auto' with power <= 0) is supported at power 0 only, got "
                             f"power={self.power!r}")
        if identity:
            return native.GLM_IDENTITY, 0.0, "HalfTweedieLossIdentity"
        return native.GLM_LOG, power, "HalfTweedieLoss"

    def _sk_params(self) -> dict:
        return dict(power=self.power, link=self.link, **super()._sk_params())

    def __repr__(self) -> str:
        return f"B200TweedieRegressor(power={self.power}, alpha={self.alpha}, link={self.link!r})"


# ---- LogisticRegression, binary: Newton fits on the GLM passes with the half-binomial loss (DESIGN.md section 11) -----
_CONTINUOUS_MESSAGE = ("Unknown label type: continuous. Maybe you are trying to fit a classifier, which expects discrete "
                       "classes on a regression target with continuous values.")


def _one_class_message(c) -> str:
    return ("This solver needs samples of at least 2 classes in the data, but the data contains only one class: "
            f"{c!r}")


def _fp32_exact(v) -> bool:
    try:
        f = float(v)
    except (TypeError, ValueError):
        return False
    return bool(np.isfinite(f)) and float(np.float32(f)) == f


class B200LogisticRegression(_B200GLM):
    """``sklearn.linear_model.LogisticRegression(solver="newton-cholesky")`` for two classes, fitted on the H100.  The
    Newton iteration is the GLM regressors' (``_B200GLM._newton``) on the half-binomial loss: one pass for the loss,
    gradient and fp64 Hessian and one pass for the 21 line-search steps, from zeros (or the last fit with warm_start),
    with the L2 strength 1 / (C n) over the n kept rows (0 at C = inf).

    Labels: host y of any dtype (``classes_`` is ``np.unique`` over the kept rows; y is mapped to {0, 1} before staging),
    or an f32 ``DeviceArray`` scanned on the device (``classes_`` are its two fp32 values, the passes read y as stored).
    Refused: more than two classes (multinomial fits are not supported), l1_ratio != 0, class_weight, sample_weight and
    any solver but 'newton-cholesky'.  verbose is accepted and has no effect."""
    _sk_name = "LogisticRegression"
    _sk_attrs = ("coef_", "intercept_", "classes_", "n_iter_", "n_features_in_")

    def __init__(self, *, C: float = 1.0, l1_ratio: float = 0.0, tol: float = 1e-4, fit_intercept: bool = True,
                 class_weight=None, solver: str = "newton-cholesky", max_iter: int = 100, verbose: int = 0,
                 warm_start: bool = False, ctx: Optional[native.Context] = None):
        self.C = C
        self.l1_ratio = l1_ratio
        self.tol = tol
        self.fit_intercept = fit_intercept
        self.class_weight = class_weight
        self.solver = solver
        self.max_iter = max_iter
        self.verbose = verbose
        self.warm_start = warm_start
        self._ctx = ctx

    def _check_params(self):
        if self.solver != "newton-cholesky":
            raise ValueError(f"solver={self.solver!r} is not supported: {type(self).__name__} runs scikit-learn's "
                             "'newton-cholesky' solver (L-BFGS-B runs only as its fallback)")
        C = self.C
        if isinstance(C, bool) or not isinstance(C, (int, float, np.integer, np.floating)) or not C > 0:
            raise ValueError(f"The 'C' parameter of LogisticRegression must be a float in the range (0.0, inf]. "
                             f"Got {C!r} instead.")
        if self.l1_ratio != 0:
            raise ValueError(f"l1_ratio={self.l1_ratio!r} is not supported: {type(self).__name__} fits the L2 penalty "
                             "only (l1_ratio=0)")
        if self.class_weight is not None:
            raise ValueError(f"class_weight is not supported by {type(self).__name__}: every kept row has weight 1")
        if isinstance(self.max_iter, bool) or not isinstance(self.max_iter, (int, np.integer)) or self.max_iter < 0:
            raise ValueError(f"The 'max_iter' parameter of LogisticRegression must be an int in the range [0, inf). "
                             f"Got {self.max_iter!r} instead.")
        if not (np.isfinite(self.tol) and self.tol >= 0):
            raise ValueError(f"The 'tol' parameter of LogisticRegression must be a float in the range [0.0, inf). "
                             f"Got {self.tol!r} instead.")

    @staticmethod
    def _host_labels(y, row_mask, mask_keep):
        """(classes_, y as float32 {0, 1}, kept rows) of host y, with scikit-learn's checks on the kept rows"""
        from sklearn.utils.multiclass import check_classification_targets
        y = np.asarray(y)
        if y.ndim == 2 and y.shape[1] == 1:
            y = y.ravel()
        if y.ndim != 1:
            raise ValueError(f"y should be a 1d array, got an array of shape {y.shape} instead.")
        if isinstance(row_mask, native.DeviceArray):
            row_mask = row_mask.to_host()
        kept = y if row_mask is None else y[np.asarray(row_mask).ravel() == mask_keep]
        if kept.size == 0:
            raise _too_few_rows((0,), by="B200LogisticRegression")
        if kept.dtype.kind in "fc":
            if np.isnan(kept).any():
                raise ValueError("Input y contains NaN.")
            if np.isinf(kept).any():
                raise ValueError(f"Input y contains infinity or a value too large for {kept.dtype!r}.")
        check_classification_targets(kept)
        classes = np.unique(kept)
        if classes.size < 2:
            raise ValueError(_one_class_message(classes[0]))
        if classes.size > 2:
            raise ValueError(f"B200LogisticRegression fits two classes only, y has {classes.size}: multinomial fits are "
                             "not supported")
        return classes, (y == classes[1]).astype(np.float32), int(kept.size)

    @staticmethod
    def _device_labels(ctx, y, row_mask, mask_keep):
        """(classes_ (fp32), kept rows) of an f32 DeviceArray y, from one label scan on the device"""
        st = ctx.label_scan(y, row_mask, mask_keep)
        if st["kept"] == 0:
            raise _too_few_rows((0,), by="B200LogisticRegression")
        if st["nonfinite"] > 0:
            raise ValueError("Input y contains NaN or infinity.")
        if st["nonintegral"] > 0:
            raise ValueError(_CONTINUOUS_MESSAGE)
        if st["min"] == st["max"]:
            raise ValueError(_one_class_message(np.float32(st["min"])))
        if st["n_min"] + st["n_max"] != st["kept"]:
            raise ValueError("B200LogisticRegression fits two classes only, y has more than two: multinomial fits are "
                             "not supported")
        return np.array([st["min"], st["max"]], dtype=np.float32), int(st["kept"])

    # -- the hooks of _B200GLM.fit; labels: (classes_, kept rows, the negative and the positive label y holds) ----------
    @contextlib.contextmanager
    def _stage_targets(self, X, y, row_mask, mask_keep, fitting: bool = True):
        """(X, y, row_mask, labels) for the logistic passes, for the body of the ``with``; ``fit`` and ``score`` share
        it.  Device y (device rows only) is read as stored, with the labels of a label scan (fitting) or of classes_.
        Host y becomes float32 {0, 1}: classes_ found in y (fitting), or NaN outside classes_; it goes up to the
        device beside device rows and is staged with host rows."""
        ctx = self.ctx
        if isinstance(y, native.DeviceArray):
            if not isinstance(X, native.DeviceArray):
                raise ValueError("device y needs device rows: X must be a DeviceArray too")
            if fitting:
                classes, n = self._device_labels(ctx, y, row_mask, mask_keep)
                yield X, y, row_mask, (classes, n, float(classes[0]), float(classes[1]))
            else:
                yield X, y, row_mask, (None, None) + self._fp32_classes()
            return
        if fitting:
            classes, y01, n = self._host_labels(y, row_mask, mask_keep)
        else:
            yh = np.asarray(y).ravel()
            y01 = np.where(yh == self.classes_[1], 1.0, np.where(yh == self.classes_[0], 0.0, np.nan))
            y01, classes, n = y01.astype(np.float32), None, None
        if isinstance(X, native.DeviceArray):
            with _on_device(ctx, y01) as y:
                yield X, y, row_mask, (classes, n, 0.0, 1.0)
        else:
            with _stage_rows(ctx, X, y01, row_mask) as (X, y, row_mask):
                yield X, y, row_mask, (classes, n, 0.0, 1.0)

    def _passes(self, X, y, row_mask, mask_keep, model, labels):
        ctx, fi, d = self.ctx, bool(self.fit_intercept), X.shape[1]
        neg, pos = labels[2:]

        def run(c, hessian):
            return ctx.logistic_pass(X, y, c[:d], float(c[d]) if fi else 0.0, neg, pos, row_mask=row_mask,
                                     mask_keep=mask_keep, fit_intercept=fi, hessian=hessian)

        def line_search(c, step):
            return ctx.logistic_line_search(X, y, c[:d], float(c[d]) if fi else 0.0, step[:d],
                                            float(step[d]) if fi else 0.0, neg, pos, n_steps=native.GLM_STEPS,
                                            row_mask=row_mask, mask_keep=mask_keep)
        return run, line_search

    def _start(self, d, run, model, labels):
        """the first pass is the Hessian pass at the start"""
        n = labels[1]
        coef, _ = self._start_coef(d)
        first = run(coef, True)
        if first["kept"] != n or first["y_out_of_range"] > 0:
            raise RuntimeError("the logistic pass saw other labels than the label check")
        _check_finite(first["loss"], first["grad"])
        return coef, first, n

    def _l2(self, labels) -> float:
        return 1.0 / (float(self.C) * labels[1])

    def _store(self, coef, n_iter, d, labels) -> None:
        self.coef_ = coef[:d].reshape(1, d).copy()
        self.intercept_ = np.array([coef[d]]) if self.fit_intercept else np.zeros(1)
        self.classes_ = labels[0]
        self.n_iter_ = np.array([n_iter], dtype=np.int32)
        self.n_features_in_ = int(d)

    def _fp32_classes(self):
        """(neg, pos): classes_ as the fp32 labels device y holds and device predictions return"""
        if self.classes_.dtype.kind not in "biuf" or not all(_fp32_exact(c) for c in self.classes_):
            raise ValueError(f"device labels are fp32 values, but classes_ is {self.classes_!r}")
        return float(self.classes_[0]), float(self.classes_[1])

    def _predict(self, X, **want):
        """one logistic_predict pass; host rows take the labels 0 and 1 (indices into classes_)"""
        X = self._checked_rows(X)
        neg, pos = self._fp32_classes() if isinstance(X, native.DeviceArray) else (0.0, 1.0)
        return self.ctx.logistic_predict(X, self.coef_[0], float(self.intercept_[0]), neg, pos, **want)

    def decision_function(self, X):
        """eta = X coef_ + intercept_ in fp64: float64 for host rows, an f64 ``DeviceArray`` for device rows."""
        return self._predict(X, decision=True)["decision"]

    def predict_proba(self, X):
        """[1 - p, p] per row, p = expit(eta), in fp64: (n, 2) float64 for host rows, an (n, 2) f64 ``DeviceArray``
        for device rows."""
        return self._predict(X, proba=True)["proba"]

    def predict_log_proba(self, X):
        """log(predict_proba(X)) for host rows."""
        if isinstance(X, native.DeviceArray):
            raise ValueError("predict_log_proba takes host rows (predict_proba returns device probabilities)")
        return np.log(self.predict_proba(X))

    def predict(self, X):
        """classes_[1] where eta > 0, else classes_[0]: an ndarray of classes_' dtype for host rows, an f32
        ``DeviceArray`` for device rows (classes_ must then be fp32 values)."""
        labels = self._predict(X, label=True)["label"]
        if isinstance(labels, native.DeviceArray):
            return labels
        return self.classes_[labels.astype(np.intp)]

    def score(self, X, y, row_mask=None, mask_keep: int = 1):
        """Accuracy over the kept rows (labels outside classes_ count as wrong): the correct count of one pass."""
        ctx = self.ctx
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=False) as (X, y, row_mask, labels):
            s = ctx.logistic_pass(self._checked_rows(X), y, self.coef_[0], float(self.intercept_[0]), *labels[2:],
                                  row_mask=row_mask, mask_keep=mask_keep, hessian=False)
        if s["kept"] == 0:
            raise _too_few_rows((0,))
        return float(s["correct"] / s["kept"])

    def _sk_params(self) -> dict:
        return dict(C=self.C, l1_ratio=self.l1_ratio, tol=self.tol, fit_intercept=self.fit_intercept,
                    solver="newton-cholesky", max_iter=self.max_iter, verbose=self.verbose, warm_start=self.warm_start)

    _sk_prepare = _B200Estimator._sk_prepare      # LogisticRegression has no _base_loss to set

    def __repr__(self) -> str:
        return f"B200LogisticRegression(C={self.C})"


# ---- RidgeClassifier: the Gram, one class-sum pass and one multi-target solve (DESIGN.md section 12) -----------------
_SK_RIDGE_SOLVERS = ("saga", "sag", "svd", "lbfgs", "lsqr", "auto", "cholesky", "sparse_cg")


def _class_index(classes: np.ndarray, y: np.ndarray) -> np.ndarray:
    """float32 index of each y in the sorted classes, -1 where y is none of them"""
    try:
        idx = np.clip(np.searchsorted(classes, y), 0, classes.size - 1)
        hit = classes[idx] == y
    except TypeError:                           # labels that do not compare with classes_
        return np.full(y.shape, -1.0, dtype=np.float32)
    return np.where(hit, idx, -1).astype(np.float32)


def _kept_class_labels(y, row_mask, mask_keep, who: str, shape_message: str):
    """(host y as 1-D, its kept rows) after scikit-learn's checks of classification targets on the kept rows;
    ``shape_message``: the refusal of y with more than one column, formatted with its shape"""
    from sklearn.utils.multiclass import check_classification_targets
    y = np.asarray(y)
    if y.ndim == 2 and y.shape[1] == 1:
        y = y.ravel()
    if y.ndim != 1:
        raise ValueError(shape_message.format(y.shape))
    if isinstance(row_mask, native.DeviceArray):
        row_mask = row_mask.to_host()
    kept = y if row_mask is None else y[np.asarray(row_mask).ravel() == mask_keep]
    if kept.size == 0:
        raise _too_few_rows((0,), by=who)
    if kept.dtype.kind in "fc":
        if np.isnan(kept).any():
            raise ValueError("Input y contains NaN.")
        if np.isinf(kept).any():
            raise ValueError(f"Input y contains infinity or a value too large for {kept.dtype!r}.")
    check_classification_targets(kept)
    return y, kept


class B200RidgeClassifier(_B200Estimator):
    """``sklearn.linear_model.RidgeClassifier`` fitted on the H100: the ridge regression of LabelBinarizer's +-1 targets
    (one target for two classes, one per class for more) from the fp64 Gram of [x 1] (the Gram dispatch every fit uses),
    one pass for the centred class sums and one single-SM LDL^T solve with every target as a right-hand side.  A system
    the factorisation refuses (alpha = 0 on a rank-deficient Gram) is solved through the eigendecomposition of the
    centred Gram instead, as scikit-learn falls back to its 'svd' solver (``solver_ = "svd"``).

    Labels: host y of any dtype (``classes_`` is ``np.unique`` over the kept rows; y is staged as float32 class indices),
    or an f32 ``DeviceArray`` beside device rows (``classes_`` are its distinct fp32 values, found on the device).
    Refused: one class, continuous or non-finite y, multilabel (2-D) y, more than ``native.MAX_CLASSES`` classes,
    class_weight, sample_weight, positive=True, solvers other than 'auto' / 'cholesky' and an array alpha.  copy_X,
    max_iter, tol and random_state are accepted and have no effect."""
    _sk_name, _label_who = "RidgeClassifier", "B200RidgeClassifier"   # _label_who: the name the label refusals give
    _sk_attrs = ("coef_", "intercept_", "classes_", "n_features_in_", "solver_", "n_iter_")

    def __init__(self, alpha: float = 1.0, *, fit_intercept: bool = True, copy_X: bool = True, max_iter=None,
                 tol: float = 1e-4, class_weight=None, solver: str = "auto", positive: bool = False, random_state=None,
                 ctx: Optional[native.Context] = None):
        self.alpha = alpha
        self.fit_intercept = fit_intercept
        self.copy_X = copy_X
        self.max_iter = max_iter
        self.tol = tol
        self.class_weight = class_weight
        self.solver = solver
        self.positive = positive
        self.random_state = random_state
        self._ctx = ctx

    def _check_params(self) -> float:
        a = self.alpha
        if np.ndim(a) != 0:
            raise ValueError("an array alpha (one per class) is not supported by B200RidgeClassifier: alpha must be one "
                             "float shared by every class")
        if isinstance(a, bool) or not isinstance(a, (int, float, np.integer, np.floating)) or not 0 <= a < np.inf:
            raise ValueError(f"The 'alpha' parameter of RidgeClassifier must be a float in the range [0.0, inf) or an "
                             f"array-like. Got {a!r} instead.")
        if self.solver not in _SK_RIDGE_SOLVERS:
            raise ValueError(f"The 'solver' parameter of RidgeClassifier must be a str among "
                             f"{{{', '.join(repr(s) for s in _SK_RIDGE_SOLVERS)}}}. Got {self.solver!r} instead.")
        if self.solver not in ("auto", "cholesky"):
            raise ValueError(f"solver={self.solver!r} is not supported: B200RidgeClassifier solves the normal equations "
                             "('auto' / 'cholesky')")
        if self.positive:
            raise ValueError("positive=True is not supported by B200RidgeClassifier: the coefficients are unconstrained")
        if self.class_weight is not None:
            raise ValueError("class_weight is not supported by B200RidgeClassifier: every kept row has weight 1")
        return float(a)

    @classmethod
    def _host_labels(cls, y, row_mask, mask_keep):
        """(classes_, y as float32 class indices (-1 for rows not kept whose label is no class), kept rows) of host y,
        with scikit-learn's checks on the kept rows"""
        y, kept = _kept_class_labels(y, row_mask, mask_keep, cls._label_who,
                                     f"multilabel y (shape {{}}) is not supported by {cls._label_who}: y must hold one "
                                     "label per row")
        classes = np.unique(kept)
        cls._check_class_count(classes, classes.size > native.MAX_CLASSES)
        return classes, _class_index(classes, y)

    @classmethod
    def _check_class_count(cls, classes, more: bool) -> None:
        if more:
            raise ValueError(f"{cls._label_who} fits at most {native.MAX_CLASSES} classes, y has more")
        if classes.size < 2:
            raise ValueError(f"{cls._label_who} needs samples of at least 2 classes, y holds only one: {classes[0]!r}")

    @classmethod
    def _device_labels(cls, ctx, y, row_mask, mask_keep):
        """classes_ (fp32) of an f32 DeviceArray y: one label scan and one label discovery on the device"""
        st = ctx.label_scan(y, row_mask, mask_keep)
        if st["kept"] == 0:
            raise _too_few_rows((0,), by=cls._label_who)
        if st["nonfinite"] > 0:
            raise ValueError("Input y contains NaN or infinity.")
        if st["nonintegral"] > 0:
            raise ValueError(_CONTINUOUS_MESSAGE)
        values, more = ctx.label_values(y, row_mask, mask_keep, native.MAX_CLASSES)
        cls._check_class_count(values, more)
        return values

    @contextlib.contextmanager
    def _stage_targets(self, X, y, row_mask, mask_keep, fitting: bool):
        """(X, y, row_mask, the fp32 classes the passes read y against, classes_) for the body of the ``with``; ``fit``
        (classes_ found in y) and ``score`` (the fitted classes_) share it.  Device y (device rows only) is read as stored
        against classes_; host y becomes float32 indices into classes_ (-1 outside them), uploaded beside device rows or
        staged with host rows."""
        ctx = self.ctx
        if isinstance(y, native.DeviceArray):
            if not isinstance(X, native.DeviceArray):
                raise ValueError("device y needs device rows: X must be a DeviceArray too")
            classes = self._device_labels(ctx, y, row_mask, mask_keep) if fitting else self.classes_
            yield X, y, row_mask, self._fp32_classes(classes), classes
            return
        if fitting:
            classes, yk = self._host_labels(y, row_mask, mask_keep)
        else:
            classes = self.classes_
            yk = _class_index(classes, np.asarray(y).ravel())
        labels = np.arange(classes.size, dtype=np.float32)
        if isinstance(X, native.DeviceArray):
            with _on_device(ctx, yk) as yd:
                yield X, yd, row_mask, labels, classes
        else:
            with _stage_rows(ctx, X, yk, row_mask) as (X, yd, row_mask):
                yield X, yd, row_mask, labels, classes

    @staticmethod
    def _fp32_classes(classes) -> np.ndarray:
        """classes as the fp32 labels device y holds and device predictions return"""
        if classes.dtype.kind not in "biuf" or not all(_fp32_exact(c) for c in classes):
            raise ValueError(f"device labels are fp32 values, but classes_ is {classes!r}")
        return classes.astype(np.float32)

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, sample_weight=None) -> "B200RidgeClassifier":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``.  Sets coef_, intercept_, classes_,
        n_features_in_, solver_ and n_iter_ (None)."""
        _refuse_sample_weight(sample_weight, "B200RidgeClassifier")
        alpha = self._check_params()
        ctx, fi = self.ctx, bool(self.fit_intercept)
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=True) as (X, y, row_mask, labels, classes):
            d = X.shape[1]
            ctx.gram_reset(d)
            ctx.gram_accumulate(X, y, row_mask, mask_keep)
            S = ctx.gram_export()
            n = S[d, d]
            if n == 0:
                raise _too_few_rows((0, d), by="B200RidgeClassifier")
            _check_finite(S)
            cs = ctx.class_sums(X, y, labels, S[:d, d] / n if fi else None, row_mask=row_mask, mask_keep=mask_keep)
        if cs["kept"] != n or cs["unmatched"] > 0 or cs["nonfinite"] > 0:
            raise RuntimeError("the class-sum pass saw other labels than the label check")
        try:
            coef, b0 = ctx.solve_classes(cs["sums"], alpha, fi)
            solver = "cholesky"
        except np.linalg.LinAlgError:
            coef, b0 = self._solve_spectral(ctx, S, cs["sums"], alpha, fi)
            solver = "svd"
        _check_finite(coef, b0)
        self.classes_, self.solver_ = classes, solver
        self.coef_ = coef[0].copy() if classes.size == 2 else coef
        self.intercept_ = b0 if fi else 0.0
        self.n_features_in_ = int(d)
        self.n_iter_ = None
        return self

    @staticmethod
    def _solve_spectral(ctx, S, sums, alpha, fi):
        """(W (T, d), b) of a system the LDL^T refuses, through the eigendecomposition of the centred Gram: the
        minimum-norm solution over the eigenvalues above 1e-12 of the largest, the right-hand sides from the class sums
        as solve_classes_kernel forms them"""
        d = S.shape[0] - 2
        n = S[d, d]
        lam, Q = ctx.solve_eigh(fit_intercept=fi)
        tot, nk = sums[:, :d].sum(axis=0), sums[:, d]
        ks = [1] if sums.shape[0] == 2 else list(range(sums.shape[0]))
        R = np.stack([2.0 * (sums[k, :d] - nk[k] / n * tot) if fi else 2.0 * sums[k, :d] - tot for k in ks], axis=1)
        ev = lam + alpha
        inv = np.where(ev > ev.max() * 1e-12, 1.0 / np.where(ev > 0, ev, 1.0), 0.0)
        W = (Q * inv) @ (Q.T @ R)
        if not fi:
            return W.T, np.zeros(len(ks))
        return W.T, (2.0 * nk[ks] / n - 1.0) - (S[:d, d] / n) @ W

    def _model(self):
        """(W (T, d), b (T,)) of the fit"""
        W = np.atleast_2d(np.asarray(self.coef_, dtype=np.float64))
        b = np.broadcast_to(np.asarray(self.intercept_, dtype=np.float64), (W.shape[0],))
        return W, b

    def _classify(self, X, **want):
        """one classify pass; host rows take the class indices as labels"""
        X = self._checked_rows(X)
        labels = self._fp32_classes(self.classes_) if isinstance(X, native.DeviceArray) else \
            np.arange(self.classes_.size, dtype=np.float32)
        return self.ctx.classify(X, *self._model(), labels, **want)

    def decision_function(self, X):
        """X coef_^T + intercept_ in fp64: (n,) for two classes, (n, K) for more; float64 for host rows, an f64
        ``DeviceArray`` for device rows."""
        out = self._classify(X, decision=True)["decision"]
        if self.classes_.size == 2:
            if isinstance(out, native.DeviceArray):
                out.shape = out.shape[:1]
            else:
                out = out.ravel()
        return out

    def predict(self, X):
        """classes_ of the largest decision (two classes: classes_[1] where it is > 0): an ndarray of classes_' dtype for
        host rows, an f32 ``DeviceArray`` for device rows (classes_ must then be fp32 values)."""
        labels = self._classify(X, label=True)["label"]
        if isinstance(labels, native.DeviceArray):
            return labels
        return self.classes_[labels.astype(np.intp)]

    def score(self, X, y, row_mask=None, mask_keep: int = 1):
        """Accuracy over the kept rows (labels outside classes_ count as wrong): the counts of one classify pass."""
        ctx = self.ctx
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=False) as (X, y, row_mask, labels, _):
            s = ctx.classify(self._checked_rows(X), *self._model(), labels, y, row_mask=row_mask, mask_keep=mask_keep)
        if s["kept"] == 0:
            raise _too_few_rows((0,))
        return float(s["correct"] / s["kept"])

    def _sk_params(self) -> dict:
        return dict(alpha=self.alpha, fit_intercept=self.fit_intercept, copy_X=self.copy_X, max_iter=self.max_iter,
                    tol=self.tol, class_weight=self.class_weight, solver=self.solver, positive=self.positive,
                    random_state=self.random_state)

    def _sk_prepare(self, reg) -> None:
        """the fitted LabelBinarizer scikit-learn's predict reads classes_ from"""
        from sklearn.preprocessing import LabelBinarizer
        reg._label_binarizer = LabelBinarizer(pos_label=1, neg_label=-1).fit(self.classes_)

    def __repr__(self) -> str:
        return f"B200RidgeClassifier(alpha={self.alpha})"


# ---- RidgeClassifierCV: the leave-one-out error of every class and alpha in one pass (DESIGN.md section 13) ------------
def _checked_statistic(ctx: native.Context, d: int, res: dict) -> np.ndarray:
    """S of one b2_ridge_classifier_loo call, after B200RidgeClassifier.fit's checks: finite, and the class-sum pass kept
    the Gram's rows, every one of them of some class"""
    S = ctx.gram_export()
    _check_finite(S)
    if res["kept"] != S[d, d] or res["unmatched"] > 0 or res["nonfinite"] > 0:
        raise RuntimeError("the class-sum pass saw other labels than the label check")
    return S


class B200RidgeClassifierCV(B200RidgeClassifier):
    """``sklearn.linear_model.RidgeClassifierCV(alphas, scoring=..., store_cv_results=...)`` with its default ``cv=None``,
    fitted on the H100 by ``b2_ridge_classifier_loo``: the Gram, the class sums, the eigendecomposition of the centred
    Gram and one fp64 pass over the rows for the exact leave-one-out error of every class target and alpha, per chunk of
    up to MAX_ALPHAS alphas; then ``B200RidgeClassifier``'s solve at the chosen alpha (and its eigendecomposition fallback
    when the factorisation refuses the system).

    ``scoring=None`` chooses the first alpha with the smallest mean of e^2 over every row and target; ``"accuracy"`` the
    first with the most kept rows whose largest leave-one-out prediction p = t - e is at their class.  With two classes
    there is one target, and scikit-learn's accuracy scorer then compares the argmax of one column with the argmax of one
    column: every alpha scores 1.0 and the first alpha is chosen.  This restates scikit-learn exactly.

    Labels, predict, decision_function, score and the export are ``B200RidgeClassifier``'s.  Refused: alphas <= 0 or not
    finite, cv other than None (the k-fold grid search), scorers other than None and "accuracy", class_weight,
    sample_weight, and what ``B200RidgeClassifier`` refuses of y."""
    _sk_name = "RidgeClassifierCV"

    def __init__(self, alphas=(0.1, 1.0, 10.0), *, fit_intercept: bool = True, scoring=None, cv=None,
                 class_weight=None, store_cv_results: bool = False, ctx: Optional[native.Context] = None):
        self.alphas = alphas
        self.fit_intercept = fit_intercept
        self.scoring = scoring
        self.cv = cv
        self.class_weight = class_weight
        self.store_cv_results = store_cv_results
        self._ctx = ctx

    def _check_params(self) -> np.ndarray:
        al = _check_alphas(self.alphas)
        if self.cv is not None:
            raise ValueError(f"cv={self.cv!r} is not supported by B200RidgeClassifierCV: it runs the leave-one-out "
                             "search of cv=None, not the k-fold grid search")
        if not (self.scoring is None or (isinstance(self.scoring, str) and self.scoring == "accuracy")):
            raise ValueError(f"scoring={self.scoring!r} is not supported by B200RidgeClassifierCV: None (mean squared "
                             "leave-one-out error) or 'accuracy'")
        if self.class_weight is not None:
            raise ValueError("class_weight is not supported by B200RidgeClassifierCV: every kept row has weight 1")
        return al

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, sample_weight=None) -> "B200RidgeClassifierCV":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``.  Sets alpha_, best_score_, coef_, intercept_,
        classes_, n_features_in_ and, with store_cv_results, cv_results_ of shape (rows kept, T, n_alphas)."""
        _refuse_sample_weight(sample_weight, "B200RidgeClassifierCV")
        al = self._check_params()
        ctx, fi = self.ctx, bool(self.fit_intercept)
        accuracy = self.scoring == "accuracy"
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=True) as (X, y, row_mask, labels, classes):
            d = X.shape[1]
            chunks, cvs, sols = [], [], []
            for off in range(0, al.size, native.MAX_ALPHAS):
                part = al[off: off + native.MAX_ALPHAS]
                try:
                    res = ctx.ridge_classifier_loo(X, y, labels, part, row_mask, mask_keep, fit_intercept=fi,
                                                   scoring=native.LOO_ACCURACY if accuracy else native.LOO_SQUARED,
                                                   store_cv=self.store_cv_results)
                    coef, b0 = res["coef"], res["intercept"]
                    _checked_statistic(ctx, d, res)
                except np.linalg.LinAlgError as exc:
                    # scikit-learn's fallback to its 'svd' solver, from the statistic the call left resident
                    res = exc.result
                    S = _checked_statistic(ctx, d, res)
                    cs = ctx.class_sums(X, y, labels, S[:d, d] / S[d, d] if fi else None, row_mask=row_mask,
                                        mask_keep=mask_keep)
                    coef, b0 = self._solve_spectral(ctx, S, cs["sums"], float(part[res["best"]]), fi)
                except ValueError as exc:
                    if "no row kept" in str(exc):
                        raise _too_few_rows((0, d), by="B200RidgeClassifierCV") from None
                    raise
                n = res["kept"]
                chunks.append((off, res["mse"], res["correct"]))
                sols.append((off + res["best"], coef, b0))
                cv = res["cv"]
                if cv is not None:
                    cvs.append(cv.to_host() if isinstance(cv, native.DeviceArray) else cv)
                    if isinstance(cv, native.DeviceArray):
                        cv.free()
        best = merge_alpha_chunks([(off, -c if accuracy else m) for off, m, c in chunks])
        mse_all = np.concatenate([m for _, m, _ in chunks])
        correct_all = np.concatenate([c for _, _, c in chunks])
        coef, b0 = next((c, b) for i, c, b in sols if i == best)
        _check_finite(coef, b0, mse_all[best])
        self.alpha_ = float(al[best])
        self.best_score_ = float(correct_all[best] / n) if accuracy else float(-mse_all[best])
        self.classes_ = classes
        self.coef_ = coef[0].copy() if classes.size == 2 else coef
        self.intercept_ = b0 if fi else 0.0
        self.n_features_in_ = int(d)
        if self.store_cv_results:
            cv = np.concatenate(cvs, axis=2)
            keep = ~np.isnan(cv[:, 0, 0]) if cv.shape[0] else np.zeros(0, bool)
            self.cv_results_ = cv[keep]
        return self

    @property
    def _sk_attrs(self) -> tuple:
        return ("alpha_", "best_score_", "coef_", "intercept_", "classes_", "n_features_in_") \
            + (("cv_results_",) if self.store_cv_results else ())

    def _sk_params(self) -> dict:
        return dict(alphas=np.asarray(self.alphas, dtype=np.float64), fit_intercept=self.fit_intercept,
                    scoring=self.scoring, cv=self.cv, class_weight=self.class_weight,
                    store_cv_results=self.store_cv_results)

    def __repr__(self) -> str:
        return f"B200RidgeClassifierCV(alphas={self.alphas!r})"


# ---- LogisticRegression, multinomial: Newton fits with the class-pair Hessian blocks on the GPU (DESIGN.md section 14) --
class B200MultinomialLogisticRegression(B200LogisticRegression):
    """``sklearn.linear_model.LogisticRegression(solver="newton-cholesky")`` for 2 to ``native.MAX_CLASSES`` classes,
    fitted on the H100.  Three or more classes fit the multinomial loss (HalfMultinomialLoss) with ``_B200GLM._newton``:
    each iteration is one pass for the loss, the K x (D + 1) gradient and the K (K + 1) / 2 class-pair blocks of the fp64
    Hessian (``multinomial_pass``) and one pass for the 21 line-search steps (``multinomial_line_search``), from zeros (or
    the last fit with warm_start), with the L2 strength 1 / (C n) on the weights only and NewtonCholeskySolver's gauge:
    at C = inf the last class is held at zero, with an intercept at C < inf its intercept; the result is centred over
    the classes.  Two classes run ``B200LogisticRegression``'s binary fit, as scikit-learn does.

    Labels: host y of any dtype (``classes_`` is ``np.unique`` over the kept rows; y is staged as float32 class indices),
    or an f32 ``DeviceArray`` beside device rows (``classes_`` are its distinct fp32 values, found on the device).
    Refused: one class, more than ``native.MAX_CLASSES`` classes, continuous or non-finite y, l1_ratio != 0,
    class_weight, sample_weight and any solver but 'newton-cholesky'.  verbose is accepted and has no effect."""

    @staticmethod
    def _host_labels(y, row_mask, mask_keep):
        """(classes_, y as float32 class indices (-1 for rows not kept whose label is no class), kept rows) of host y"""
        y, kept = _kept_class_labels(y, row_mask, mask_keep, "B200MultinomialLogisticRegression",
                                     "y should be a 1d array, got an array of shape {} instead.")
        classes = np.unique(kept)
        if classes.size < 2:
            raise ValueError(_one_class_message(classes[0]))
        if classes.size > native.MAX_CLASSES:
            raise ValueError(f"B200MultinomialLogisticRegression fits at most {native.MAX_CLASSES} classes, y has "
                             f"{classes.size}")
        return classes, _class_index(classes, y), int(kept.size)

    @staticmethod
    def _device_labels(ctx, y, row_mask, mask_keep):
        """(classes_ (fp32), kept rows) of an f32 DeviceArray y: one label scan and one label discovery on the device"""
        st = ctx.label_scan(y, row_mask, mask_keep)
        if st["kept"] == 0:
            raise _too_few_rows((0,), by="B200MultinomialLogisticRegression")
        if st["nonfinite"] > 0:
            raise ValueError("Input y contains NaN or infinity.")
        if st["nonintegral"] > 0:
            raise ValueError(_CONTINUOUS_MESSAGE)
        if st["min"] == st["max"]:
            raise ValueError(_one_class_message(np.float32(st["min"])))
        values, more = ctx.label_values(y, row_mask, mask_keep, native.MAX_CLASSES)
        if more:
            raise ValueError(f"B200MultinomialLogisticRegression fits at most {native.MAX_CLASSES} classes, y has more")
        return values, int(st["kept"])

    # -- the hooks of _B200GLM.fit; labels: (classes_, kept rows, the K fp32 labels y holds), as the binary fit's for K = 2
    @contextlib.contextmanager
    def _stage_targets(self, X, y, row_mask, mask_keep, fitting: bool = True):
        """(X, y, row_mask, labels) for the passes, for the body of the ``with``; ``fit`` and ``score`` share it.  Device
        y (device rows only) is read as stored against the fp32 classes; host y becomes float32 indices into classes_
        (-1 outside them), uploaded beside device rows or staged with host rows.  Scoring leaves classes_ and the kept
        rows None."""
        ctx = self.ctx
        if isinstance(y, native.DeviceArray):
            if not isinstance(X, native.DeviceArray):
                raise ValueError("device y needs device rows: X must be a DeviceArray too")
            classes, n = self._device_labels(ctx, y, row_mask, mask_keep) if fitting else (self.classes_, None)
            values = tuple(float(c) for c in B200RidgeClassifier._fp32_classes(classes))
            yield X, y, row_mask, (classes if fitting else None, n) + values
            return
        if fitting:
            classes, yk, n = self._host_labels(y, row_mask, mask_keep)
        else:                                     # class by class: labels of any type, outside classes_ too
            classes, n = self.classes_, None
            yh = np.asarray(y).ravel()
            yk = np.full(yh.shape, -1.0, dtype=np.float32)
            for k, c in enumerate(classes):
                yk[yh == c] = k
        labels = (classes if fitting else None, n) + tuple(float(k) for k in range(classes.size))
        if isinstance(X, native.DeviceArray):
            with _on_device(ctx, yk) as yd:
                yield X, yd, row_mask, labels
        else:
            with _stage_rows(ctx, X, yk, row_mask) as (X, yd, row_mask):
                yield X, yd, row_mask, labels

    def _passes(self, X, y, row_mask, mask_keep, model, labels):
        if len(labels) == 4:
            return super()._passes(X, y, row_mask, mask_keep, model, labels)
        ctx, fi, d = self.ctx, bool(self.fit_intercept), X.shape[1]
        k, n_dof = len(labels) - 2, d + int(fi)
        classes = np.array(labels[2:], dtype=np.float32)

        def rows(c):                              # the raveled coefficients as the pass's rows [w_k, b_k]
            full = np.zeros((k, d + 1))
            full[:, :n_dof] = np.reshape(c, (k, n_dof), order="F")
            return full

        def run(c, hessian):
            s = ctx.multinomial_pass(X, y, classes, rows(c), row_mask=row_mask, mask_keep=mask_keep,
                                     fit_intercept=fi, hessian=hessian)
            if hessian:                           # blocks [k][l][i][j] -> scikit-learn's order, (i, k) x (j, l)
                s["hessian"] = s["hessian"].transpose(2, 0, 3, 1).reshape(k * (d + 1), k * (d + 1))
            s["h_nonpos"] = 0.0                   # the multinomial pointwise Hessian is never negative
            return s

        def line_search(c, step):
            return ctx.multinomial_line_search(X, y, classes, rows(c), rows(step), n_steps=native.GLM_STEPS,
                                               row_mask=row_mask, mask_keep=mask_keep)
        return run, line_search

    def _start(self, d, run, model, labels):
        """the start (zeros, or the last fit with warm_start) in NewtonCholeskySolver's gauge, then its Hessian pass"""
        if len(labels) == 4:
            return super()._start(d, run, model, labels)
        fi, k, n = bool(self.fit_intercept), len(labels) - 2, labels[1]
        coef = np.zeros((k, d + int(fi)))
        if self.warm_start and getattr(self, "coef_", None) is not None:
            prev = np.asarray(self.coef_, dtype=np.float64)
            if prev.shape != (k, d):
                raise ValueError(f"the warm start coef_ has shape {prev.shape}, ({k}, {d}) expected")
            coef[:, :d] = prev
            if fi:
                coef[:, d] = np.asarray(self.intercept_, dtype=np.float64)
        if self._l2(labels) == 0:
            coef -= coef[-1, :]
        elif fi:
            coef[:, -1] -= coef[-1, -1]
        coef = coef.ravel(order="F")
        first = run(coef, True)
        if first["kept"] != n or first["unmatched"] > 0 or first["nonfinite"] > 0:
            raise RuntimeError("the multinomial pass saw other labels than the label check")
        _check_finite(first["loss"], first["grad"])
        return coef, first, n

    def _layout(self, d, labels) -> dict:
        k = len(labels) - 2
        if k == 2:
            return {}
        size = k * (d + int(bool(self.fit_intercept)))
        if self._l2(labels) == 0:                 # the last class held at zero
            free = np.flatnonzero(np.arange(size) % k != k - 1)
        elif self.fit_intercept:                  # the last intercept held at zero
            free = np.arange(size - 1)
        else:
            free = None
        return dict(n_classes=k, free=free)

    def _store(self, coef, n_iter, d, labels) -> None:
        if len(labels) == 4:
            return super()._store(coef, n_iter, d, labels)
        fi, k = bool(self.fit_intercept), len(labels) - 2
        w = np.reshape(coef, (k, d + int(fi)), order="F").copy()
        if self._l2(labels) == 0:                 # NewtonCholeskySolver.finalize: the symmetric parametrisation
            w -= np.mean(w, axis=0)
        elif fi:
            w[:, -1] -= np.mean(w[:, -1])
        self.coef_ = w[:, :d].copy()
        self.intercept_ = w[:, d].copy() if fi else np.zeros(k)
        self.classes_ = labels[0]
        self.n_iter_ = np.array([n_iter], dtype=np.int32)
        self.n_features_in_ = int(d)

    # -- predictions: two classes as the binary estimator, more through one classify pass ------------------------------
    def _classify(self, X, **want):
        X = self._checked_rows(X)
        labels = B200RidgeClassifier._fp32_classes(self.classes_) if isinstance(X, native.DeviceArray) else \
            np.arange(self.classes_.size, dtype=np.float32)
        return self.ctx.classify(X, self.coef_, self.intercept_, labels, **want)

    def decision_function(self, X):
        """X coef_^T + intercept_ in fp64: (n,) for two classes, (n, K) for more; float64 for host rows, an f64
        ``DeviceArray`` for device rows."""
        if self.classes_.size == 2:
            return super().decision_function(X)
        return self._classify(X, decision=True)["decision"]

    def predict_proba(self, X):
        """The class probabilities, (n, K) fp64: scikit-learn's softmax of the decision for host rows; for device rows
        an f64 ``DeviceArray``, the decision turned into probabilities in place on the device."""
        if self.classes_.size == 2:
            return super().predict_proba(X)
        from sklearn.utils.extmath import softmax
        dec = self.decision_function(X)
        if isinstance(dec, native.DeviceArray):
            self.ctx.softmax_rows(dec)
            return dec
        return softmax(dec, copy=False)

    def predict(self, X):
        """classes_ of the first largest decision: an ndarray of classes_' dtype for host rows, an f32 ``DeviceArray``
        for device rows (classes_ must then be fp32 values)."""
        if self.classes_.size == 2:
            return super().predict(X)
        labels = self._classify(X, label=True)["label"]
        if isinstance(labels, native.DeviceArray):
            return labels
        return self.classes_[labels.astype(np.intp)]

    def score(self, X, y, row_mask=None, mask_keep: int = 1):
        """Accuracy over the kept rows (labels outside classes_ count as wrong): the counts of one pass."""
        if self.classes_.size == 2:
            return super().score(X, y, row_mask, mask_keep)
        ctx = self.ctx
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=False) as (X, y, row_mask, labels):
            s = ctx.classify(self._checked_rows(X), self.coef_, self.intercept_, np.array(labels[2:], np.float32), y,
                             row_mask=row_mask, mask_keep=mask_keep)
        if s["kept"] == 0:
            raise _too_few_rows((0,))
        return float(s["correct"] / s["kept"])

    def __repr__(self) -> str:
        return f"B200MultinomialLogisticRegression(C={self.C})"


# ---- LinearSVC / LinearSVR: liblinear's primal trust-region Newton fits (DESIGN.md section 15) -----------------------
_LIBLINEAR_CONV = "Liblinear failed to converge, increase the number of iterations."


def _tron(prob, f, g, eps: float, max_iter: int):
    """``TRON::tron`` of liblinear (sklearn/svm/src/liblinear/tron.cpp) line by line, from w = 0 with f and g there:
    ``prob.trial(w_new)`` is fun(w_new), ``prob.accept()`` takes the trial point and is grad(w), ``prob.hv(v)`` is Hv.
    Returns (w, n_iter) with n_iter = --iter, as liblinear counts it."""
    eta0, eta1, eta2 = 1e-4, 0.25, 0.75
    sigma1, sigma2, sigma3 = 0.25, 0.5, 4.0
    w = np.zeros(g.size)
    delta = float(np.linalg.norm(g))
    gnorm1 = delta
    search = not delta <= eps * gnorm1
    it = 1
    while it <= max_iter and search:
        s, r = _trcg(prob.hv, delta, g)
        w_new = w + s
        gs = float(g @ s)
        prered = -0.5 * (gs - float(s @ r))
        fnew = prob.trial(w_new)
        actred = f - fnew
        snorm = float(np.linalg.norm(s))
        if it == 1:
            delta = min(delta, snorm)
        if fnew - f - gs <= 0:
            alpha = sigma3
        else:
            alpha = max(sigma1, -0.5 * (gs / (fnew - f - gs)))
        if actred < eta0 * prered:
            delta = min(max(alpha, sigma1) * snorm, sigma2 * delta)
        elif actred < eta1 * prered:
            delta = max(sigma1 * delta, min(alpha * snorm, sigma2 * delta))
        elif actred < eta2 * prered:
            delta = max(sigma1 * delta, min(alpha * snorm, sigma3 * delta))
        else:
            delta = max(delta, min(alpha * snorm, sigma3 * delta))
        if actred > eta0 * prered:
            it += 1
            w, f = w_new, fnew
            g = prob.accept()
            if np.linalg.norm(g) <= eps * gnorm1:
                break
        if f < -1.0e32:
            break
        if abs(actred) <= 0 and prered <= 0:
            break
        if abs(actred) <= 1.0e-12 * abs(f) and abs(prered) <= 1.0e-12 * abs(f):
            break
    return w, it - 1


def _trcg(hv, delta: float, g):
    """``TRON::trcg``: conjugate gradients on H s = -g inside the trust region of radius delta; returns (s, r)"""
    s = np.zeros(g.size)
    r = -g
    d = r.copy()
    cgtol = 0.1 * np.linalg.norm(g)
    rTr = float(r @ r)
    while np.linalg.norm(r) > cgtol:
        Hd = hv(d)
        alpha = rTr / float(d @ Hd)
        s += alpha * d
        if np.linalg.norm(s) > delta:            # back to the boundary of the trust region
            s -= alpha * d
            std, sts, dtd, dsq = float(s @ d), float(s @ s), float(d @ d), delta * delta
            rad = np.sqrt(std * std + dtd * (dsq - sts))
            alpha = (dsq - sts) / (std + rad) if std >= 0 else (rad - std) / dtd
            s += alpha * d
            r -= alpha * Hd
            break
        r -= alpha * Hd
        rnewTrnew = float(r @ r)
        d = d * (rnewTrnew / rTr) + r
        rTr = rnewTrnew
    return s, r


class _SvmProblem:
    """liblinear's l2r_l2_svc_fun / l2r_l2_svr_fun on GPU passes.  w = [coef, w_b] with w_b the weight of the bias
    feature of value ``scale`` (intercept_scaling; absent without an intercept); f(w) = w.w / 2 + C sum loss, g = w +
    2 C sum g z, H = I + 2 C sum z z^T over the active rows.  H's sum is carried from pass to pass: each pass at
    (accepted w, trial w) returns the change over the rows that crossed, kept when the step is accepted.
    ``run(w_from, w_to, hessian)`` is one ``svm_pass`` (w_from None: the empty active set)."""

    def __init__(self, run, C: float, d: int, fit_intercept: bool, scale: float):
        self.run, self.C, self.d, self.fi, self.scale = run, C, d, fit_intercept, scale
        self.n = d + int(fit_intercept)
        self.w = self.pending = self.H = None

    def _fg(self, w, res):
        G = res["grad"][: self.n].copy()
        if self.fi:
            G[self.d] *= self.scale
        return 0.5 * float(w @ w) + self.C * res["loss"], w + 2.0 * self.C * G

    def start(self, gram=None):
        """(f, g, the pass) at w = 0; the Hessian sum from this pass, or ``gram`` (the sum over every kept row, which
        is the active set at 0 of the squared hinge) with a pass that changes no row"""
        self.w = np.zeros(self.n)
        res = self.run(None if gram is None else self.w, self.w, gram is None)
        self.H = (res["dhessian"] if gram is None else gram).copy()
        _check_finite(res["loss"], res["grad"])
        f, g = self._fg(self.w, res)
        self.g = g
        return f, g, res

    def trial(self, w_new) -> float:
        self.pending = (w_new, self.run(self.w, w_new, True))
        f, self.g_pending = self._fg(w_new, self.pending[1])
        return f

    def accept(self):
        self.w, res = self.pending
        self.H += res["dhessian"]
        self.g = self.g_pending
        return self.g

    def hv(self, v):
        u = v.copy()
        if self.fi:
            u[self.d] *= self.scale
        Hu = self.H[: self.n, : self.n] @ u
        if self.fi:
            Hu[self.d] *= self.scale
        return v + 2.0 * self.C * Hu

    def coef(self, w):
        """(coef, intercept): intercept = intercept_scaling w_b"""
        return w[: self.d].copy(), (self.scale * w[self.d] if self.fi else 0.0)


def _svm_run(ctx, X, y, row_mask, mask_keep, loss: int, param: float, fit_intercept: bool, scale: float):
    """run(w_from, w_to, hessian) of _SvmProblem: one svm_pass, the bias feature's weight as its intercept"""
    d = X.shape[1]

    def split(w):
        return w[:d], (scale * float(w[d]) if fit_intercept else 0.0)

    def run(w_from, w_to, hessian):
        c, b = split(w_to)
        cf, bf = split(w_from) if w_from is not None else (None, 0.0)
        return ctx.svm_pass(X, y, c, b, loss=loss, param=param, coef_from=cf, intercept_from=bf, row_mask=row_mask,
                            mask_keep=mask_keep, fit_intercept=fit_intercept, hessian=hessian)
    return run


class _B200LinearSVM:
    """The parameter checks LinearSVC and LinearSVR share: anything that selects another liblinear solver is refused"""

    def _check_svm_params(self, sk: str, loss_ok: str, penalty: str = "l2"):
        C = self.C
        if isinstance(C, bool) or not isinstance(C, (int, float, np.integer, np.floating)) or not 0 < C < np.inf:
            raise ValueError(f"The 'C' parameter of {sk} must be a float in the range (0.0, inf). Got {C!r} instead.")
        if not (isinstance(self.tol, (int, float, np.integer, np.floating)) and np.isfinite(self.tol) and self.tol > 0):
            raise ValueError(f"The 'tol' parameter of {sk} must be a float in the range (0.0, inf). Got {self.tol!r} "
                             "instead.")
        if isinstance(self.max_iter, bool) or not isinstance(self.max_iter, (int, np.integer)) or self.max_iter < 0:
            raise ValueError(f"The 'max_iter' parameter of {sk} must be an int in the range [0, inf). "
                             f"Got {self.max_iter!r} instead.")
        if self.loss != loss_ok:
            raise ValueError(f"loss={self.loss!r} is not supported: B200{sk} runs liblinear's primal solver for "
                             f"loss={loss_ok!r}")
        if penalty != "l2":
            raise ValueError(f"penalty={penalty!r} is not supported: B200{sk} runs liblinear's primal solver for the L2 "
                             "penalty")
        if self.dual not in ("auto", False):
            raise ValueError(f"dual={self.dual!r} is not supported: B200{sk} runs liblinear's primal solver "
                             "(dual=False, or 'auto' with at least as many rows as features)")
        if self.fit_intercept and not self.intercept_scaling > 0:
            raise ValueError(f"Intercept scaling is {self.intercept_scaling!r} but needs to be greater than 0. To "
                             "disable fitting an intercept, set fit_intercept=False.")

    def _check_rows(self, sk: str, n: float, d: int) -> None:
        """the kept rows: some, and (dual='auto') at least as many as features, where scikit-learn picks the primal
        solver"""
        if n == 0:
            raise _too_few_rows((0, d), by=f"B200{sk}")
        if self.dual == "auto" and n < d:
            raise ValueError(f"dual='auto' selects liblinear's dual solver with fewer rows ({int(n)}) than features "
                             f"({d}): B200{sk} runs the primal solver only (set dual=False)")

    def _warn_iter(self, n_iter: int) -> None:
        if n_iter >= self.max_iter:
            from sklearn.exceptions import ConvergenceWarning
            warnings.warn(_LIBLINEAR_CONV, ConvergenceWarning)


class B200LinearSVC(_B200LinearSVM, B200RidgeClassifier):
    """``sklearn.svm.LinearSVC`` with liblinear's primal solver (penalty='l2', loss='squared_hinge', dual=False, or
    dual='auto' with at least as many rows as features), fitted on the H100.  liblinear's trust-region Newton method
    (``_tron``) runs on the host; each iteration is one pass (``svm_pass``) for the loss and gradient at the trial point
    and the change of the generalized Hessian over the rows that crossed the margin, on the fp64 tensor core.  The
    intercept is liblinear's regularised bias feature of value intercept_scaling.  Two classes: one problem with
    classes_[1] as +1; more: one-vs-rest, one fit per class in class order.  At w = 0 every kept row is active for every
    class, so the first class's start pass computes the Gram of [x 1] and the others start from it.

    Labels, ``decision_function``, ``predict`` and ``score`` are ``B200RidgeClassifier``'s.  Refused: loss='hinge',
    penalty='l1', dual=True, multi_class='crammer_singer', class_weight, sample_weight, one class, more than
    ``native.MAX_CLASSES`` classes, non-finite X or y.  verbose and random_state are accepted and have no effect."""
    _sk_module = "svm"
    _sk_name = "LinearSVC"
    _sk_attrs = ("coef_", "intercept_", "classes_", "n_iter_", "n_features_in_")
    _label_who = "B200LinearSVC"

    def __init__(self, penalty: str = "l2", loss: str = "squared_hinge", *, dual="auto", tol: float = 1e-4,
                 C: float = 1.0, multi_class: str = "ovr", fit_intercept: bool = True, intercept_scaling: float = 1,
                 class_weight=None, verbose: int = 0, random_state=None, max_iter: int = 1000,
                 ctx: Optional[native.Context] = None):
        self.penalty = penalty
        self.loss = loss
        self.dual = dual
        self.tol = tol
        self.C = C
        self.multi_class = multi_class
        self.fit_intercept = fit_intercept
        self.intercept_scaling = intercept_scaling
        self.class_weight = class_weight
        self.verbose = verbose
        self.random_state = random_state
        self.max_iter = max_iter
        self._ctx = ctx

    @classmethod
    def _check_class_count(cls, classes, more: bool) -> None:
        if more:
            raise ValueError(f"B200LinearSVC fits at most {native.MAX_CLASSES} classes, y has more")
        if classes.size < 2:
            raise ValueError(_one_class_message(classes[0]))

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, sample_weight=None) -> "B200LinearSVC":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``.  Sets coef_, intercept_, classes_, n_iter_
        and n_features_in_."""
        _refuse_sample_weight(sample_weight, "B200LinearSVC")
        if self.multi_class == "crammer_singer":
            raise ValueError("multi_class='crammer_singer' is not supported: B200LinearSVC runs liblinear's primal "
                             "one-vs-rest solver")
        if self.multi_class != "ovr":
            raise ValueError(f"`multi_class` must be one of `ovr`, `crammer_singer`, got {self.multi_class!r}")
        if self.class_weight is not None:
            raise ValueError("class_weight is not supported by B200LinearSVC: every kept row has weight 1")
        self._check_svm_params("LinearSVC", "squared_hinge", self.penalty)
        ctx, fi, scale = self.ctx, bool(self.fit_intercept), float(self.intercept_scaling)
        C = float(self.C)
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=True) as (X, y, row_mask, labels, classes):
            d = X.shape[1]
            targets = labels[1:] if classes.size == 2 else labels
            W, b, iters, gram = [], [], [], None
            for pos in targets:
                prob = _SvmProblem(_svm_run(ctx, X, y, row_mask, mask_keep, native.SVM_SQUARED_HINGE, float(pos), fi,
                                            scale), C, d, fi, scale)
                f, g, first = prob.start(gram)
                n = first["kept"]
                self._check_rows("LinearSVC", n, d)
                if gram is None:
                    gram = prob.H.copy()
                # train_one: eps max(min(pos, neg), 1) / l
                eps = float(self.tol) * max(min(first["positive"], n - first["positive"]), 1) / n
                w, n_iter = _tron(prob, f, g, eps, int(self.max_iter))
                _check_finite(w)
                c, b0 = prob.coef(w)
                W.append(c)
                b.append(b0)
                iters.append(n_iter)
        self.classes_ = classes
        self.coef_ = np.array(W)
        self.intercept_ = np.array(b) if fi else 0.0
        self.n_iter_ = int(max(iters))
        self.n_features_in_ = int(d)
        self._warn_iter(self.n_iter_)
        return self

    def _sk_params(self) -> dict:
        return dict(penalty=self.penalty, loss=self.loss, dual=self.dual, tol=self.tol, C=self.C,
                    multi_class=self.multi_class, fit_intercept=self.fit_intercept,
                    intercept_scaling=self.intercept_scaling, class_weight=self.class_weight, verbose=self.verbose,
                    random_state=self.random_state, max_iter=self.max_iter)

    _sk_prepare = _B200Estimator._sk_prepare      # LinearSVC's predict reads classes_, coef_ and intercept_ only

    def __repr__(self) -> str:
        return f"B200LinearSVC(C={self.C})"


class B200LinearSVR(_B200LinearSVM, _B200Estimator):
    """``sklearn.svm.LinearSVR(loss="squared_epsilon_insensitive")`` with liblinear's primal solver (dual=False, or
    dual='auto' with at least as many rows as features), fitted on the H100: ``B200LinearSVC``'s trust-region Newton
    method on the squared epsilon-insensitive loss, with liblinear's tolerance tol.  ``predict`` is one fp64 pass and
    ``score`` is R^2 from two passes over the kept rows.  Refused: loss='epsilon_insensitive' (scikit-learn's default,
    a dual solver), dual=True, sample_weight, non-finite X or y.  verbose and random_state are accepted and have no
    effect."""
    _sk_module = "svm"
    _sk_name = "LinearSVR"
    _sk_attrs = ("coef_", "intercept_", "n_iter_", "n_features_in_")

    def __init__(self, *, epsilon: float = 0.0, tol: float = 1e-4, C: float = 1.0, loss: str = "epsilon_insensitive",
                 fit_intercept: bool = True, intercept_scaling: float = 1.0, dual="auto", verbose: int = 0,
                 random_state=None, max_iter: int = 1000, ctx: Optional[native.Context] = None):
        self.epsilon = epsilon
        self.tol = tol
        self.C = C
        self.loss = loss
        self.fit_intercept = fit_intercept
        self.intercept_scaling = intercept_scaling
        self.dual = dual
        self.verbose = verbose
        self.random_state = random_state
        self.max_iter = max_iter
        self._ctx = ctx

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, sample_weight=None) -> "B200LinearSVR":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16), y float (an f32
        ``DeviceArray`` beside device rows); ``row_mask`` (uint8 per row) restricts the fit to rows equal to
        ``mask_keep``.  Sets coef_, intercept_, n_iter_ and n_features_in_."""
        _refuse_sample_weight(sample_weight, "B200LinearSVR")
        self._check_svm_params("LinearSVR", "squared_epsilon_insensitive")
        eps = self.epsilon
        if isinstance(eps, bool) or not isinstance(eps, (int, float, np.integer, np.floating)) or not 0 <= eps < np.inf:
            raise ValueError(f"The 'epsilon' parameter of LinearSVR must be a float in the range [0.0, inf). Got "
                             f"{eps!r} instead.")
        ctx, fi, scale = self.ctx, bool(self.fit_intercept), float(self.intercept_scaling)
        with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
            d = X.shape[1]
            prob = _SvmProblem(_svm_run(ctx, X, y, row_mask, mask_keep, native.SVM_SQUARED_EPSILON, float(eps), fi,
                                        scale), float(self.C), d, fi, scale)
            f, g, first = prob.start()
            self._check_rows("LinearSVR", first["kept"], d)
            if first["y_nonfinite"] > 0:
                raise ValueError(_NAN_MESSAGE)
            w, n_iter = _tron(prob, f, g, float(self.tol), int(self.max_iter))
            _check_finite(w)
        c, b0 = prob.coef(w)
        self.coef_ = c
        self.intercept_ = np.array([b0]) if fi else 0.0
        self.n_iter_ = int(n_iter)
        self.n_features_in_ = int(d)
        self._warn_iter(self.n_iter_)
        return self

    def predict(self, X):
        """X coef_ + intercept_ in fp64: float64 for host rows, an f64 ``DeviceArray`` for device rows."""
        return self.ctx.glm_predict(self._checked_rows(X), self.coef_, float(np.sum(self.intercept_)),
                                    link=native.GLM_IDENTITY)

    def score(self, X, y, row_mask=None, mask_keep: int = 1):
        """R^2 over the kept rows, as scikit-learn's ``RegressorMixin.score`` computes it: the squared residuals of
        the model and of the mean of y, one pass each."""
        ctx = self.ctx
        with _stage_rows(ctx, X, y, row_mask) as (X, y, row_mask):
            d = self._checked_rows(X).shape[1]
            kw = dict(link=native.GLM_IDENTITY, power=0.0, row_mask=row_mask, mask_keep=mask_keep, hessian=False)
            model = ctx.glm_pass(X, y, self.coef_, float(np.sum(self.intercept_)), **kw)
            n = model["kept"]
            if n == 0:
                raise _too_few_rows((0, d))
            if model["y_nonfinite"] > 0:
                raise ValueError(_NAN_MESSAGE)
            null = ctx.glm_pass(X, y, np.zeros(d), model["sum_y"] / n, **kw)
        num, den = model["loss"], null["loss"]
        if den == 0:                                # r2_score's force_finite
            return 1.0 if num == 0 else 0.0
        return float(1 - num / den)

    def _sk_params(self) -> dict:
        return dict(epsilon=self.epsilon, tol=self.tol, C=self.C, loss=self.loss, fit_intercept=self.fit_intercept,
                    intercept_scaling=self.intercept_scaling, dual=self.dual, verbose=self.verbose,
                    random_state=self.random_state, max_iter=self.max_iter)

    def __repr__(self) -> str:
        return f"B200LinearSVR(C={self.C}, epsilon={self.epsilon})"


# ---- LinearDiscriminantAnalysis: the class means and one fp64 within-class scatter pass (DESIGN.md section 16) --------
_LDA_SOLVERS = ("svd", "lsqr", "eigen")


def _shrunk(cov: np.ndarray, shrinkage) -> np.ndarray:
    """sklearn.covariance.shrunk_covariance of a covariance (None: the covariance as it is)"""
    if shrinkage is None:
        return cov
    s = float(shrinkage)
    out = (1.0 - s) * cov
    out += s * (np.trace(cov) / cov.shape[0]) * np.eye(cov.shape[0])
    return out


def _lda_svd(sw1: np.ndarray, means: np.ndarray, nk: np.ndarray, priors: np.ndarray, tol: float, max_components: int):
    """scikit-learn's ``_solve_svd`` from the statistics: the within-class singular values and right singular vectors
    of the scaled centred rows are the square roots and eigenvectors of their Gram, S_w(1) / (n - K) / (std std^T);
    from the K x rank product on, scikit-learn's code as it is.  Returns (coef, intercept, xbar, scalings,
    explained_variance_ratio) before the two-class collapse."""
    import scipy.linalg
    n, K = float(nk.sum()), nk.size
    std = np.sqrt(np.diag(sw1) / n)
    std[std == 0] = 1.0
    lam, V = np.linalg.eigh(sw1 / (n - K) / np.outer(std, std))
    lam, V = lam[::-1], V[:, ::-1]
    S = np.sqrt(np.maximum(lam, 0.0))
    rank = int(np.sum(S > tol))
    scalings = V[:, :rank] / std[:, None] / S[:rank]
    xbar = priors @ means
    fac = 1.0 if K == 1 else 1.0 / (K - 1)
    Xb = ((np.sqrt((n * priors) * fac)) * (means - xbar).T).T @ scalings
    _, S, Vt = scipy.linalg.svd(Xb, full_matrices=False)
    evr = np.empty((0,)) if max_components == 0 else (S ** 2 / np.sum(S ** 2))[:max_components]
    rank = int(np.sum(S > tol * S[0]))
    scalings = scalings @ Vt.T[:, :rank]
    coef = (means - xbar) @ scalings
    intercept = -0.5 * np.sum(coef ** 2, axis=1) + np.log(priors)
    coef = coef @ scalings.T
    intercept -= xbar @ coef.T
    return coef, intercept, xbar, scalings, evr


def _lda_lstsq(cov: np.ndarray, means: np.ndarray, priors: np.ndarray):
    """scikit-learn's ``_solve_lstsq`` on the (shrunk) covariance"""
    import scipy.linalg
    coef = scipy.linalg.lstsq(cov, means.T)[0].T
    return coef, -0.5 * np.diag(np.dot(means, coef.T)) + np.log(priors)


def _lda_eigen(cov: np.ndarray, total: np.ndarray, means: np.ndarray, priors: np.ndarray, max_components: int):
    """scikit-learn's ``_solve_eigen`` on the (shrunk) within-class covariance and total covariance"""
    import scipy.linalg
    evals, evecs = scipy.linalg.eigh(total - cov, cov)
    evr = np.sort(evals / np.sum(evals))[::-1][:max_components]
    evecs = evecs[:, np.argsort(evals)[::-1]]
    coef = np.dot(means, evecs).dot(evecs.T)
    return coef, -0.5 * np.diag(np.dot(means, coef.T)) + np.log(priors), evecs, evr


class B200LinearDiscriminantAnalysis(B200RidgeClassifier):
    """``sklearn.discriminant_analysis.LinearDiscriminantAnalysis`` for 2 to ``native.MAX_CLASSES`` classes, fitted on
    the H100.  Every solver needs only the class counts and means (one class-sum pass) and the pooled within-class
    scatter S_w(w) = sum w_y (x - m_y)(x - m_y)^T, which one fp64 tensor-core pass (``class_scatter``) forms from rows
    centred on their class mean: w = 1 for 'svd', w_k = p_k / n_k (the priors' covariance) for 'lsqr' and 'eigen'.  A
    second pass with the other weights runs only where a fit needs both matrices and the priors are given: 'svd' with
    store_covariance, and 'eigen' (the total scatter is S_w(1) plus the between-class scatter of the means).  The
    solvers are scikit-learn's, restated on these statistics with numpy and scipy on the host; 'svd' takes the
    eigenvectors of the scaled scatter for the right singular vectors of the scaled rows.

    Labels, ``decision_function``, ``predict`` and ``score`` are ``B200RidgeClassifier``'s.  ``predict_proba`` is the
    logistic of the decision for two classes and scikit-learn's softmax of the decisions for more (on the device for
    device rows); ``transform`` is one fp64 decision pass with one output per component.  The columns of ``scalings_``
    and ``transform`` equal scikit-learn's up to the sign of each column; every other attribute and prediction does not
    depend on those signs.  ``transform`` computes x.s - xbar.s, so its error is relative to sum |x_j s_j|.

    Refused: shrinkage='auto' (Ledoit-Wolf needs each class's own covariance), a covariance_estimator, shrinkage with
    the 'svd' solver, other solvers, one class, more than ``native.MAX_CLASSES`` classes, continuous, multilabel or
    non-finite y, and non-finite X."""
    _sk_module = "discriminant_analysis"
    _sk_name = "LinearDiscriminantAnalysis"
    _sk_attrs = ("coef_", "intercept_", "classes_", "means_", "priors_", "n_features_in_", "_max_components",
                 "_n_features_out")
    _label_who = "B200LinearDiscriminantAnalysis"

    def __init__(self, solver: str = "svd", shrinkage=None, priors=None, n_components=None,
                 store_covariance: bool = False, tol: float = 1e-4, covariance_estimator=None,
                 ctx: Optional[native.Context] = None):
        self.solver = solver
        self.shrinkage = shrinkage
        self.priors = priors
        self.n_components = n_components
        self.store_covariance = store_covariance
        self.tol = tol
        self.covariance_estimator = covariance_estimator
        self._ctx = ctx

    def _check_params(self):
        who = "B200LinearDiscriminantAnalysis"
        if self.solver not in _LDA_SOLVERS:
            raise ValueError(f"The 'solver' parameter of {who} must be a str among {{'eigen', 'lsqr', 'svd'}}. Got "
                             f"{self.solver!r} instead.")
        s = self.shrinkage
        if isinstance(s, str) and s == "auto":
            raise ValueError(f"shrinkage='auto' is not supported by {who}: the Ledoit-Wolf estimate needs each class's "
                             "own covariance, and its weight falls like 1/n, so at the row counts this estimator serves "
                             "shrinkage=None or a float gives the same model")
        if s is not None and (isinstance(s, (bool, str)) or not isinstance(s, (int, float, np.integer, np.floating))
                              or not 0 <= s <= 1):
            raise ValueError(f"The 'shrinkage' parameter of {who} must be a str among {{'auto'}}, a float in the range "
                             f"[0, 1] or None. Got {s!r} instead.")
        if self.covariance_estimator is not None:
            raise ValueError(f"covariance_estimator is not supported by {who}: the covariance is the empirical one "
                             "(with shrinkage=None or a float)")
        if self.solver == "svd" and s is not None:
            raise NotImplementedError(f"shrinkage not supported with 'svd' solver. ({who})")
        if isinstance(self.tol, bool) or not isinstance(self.tol, (int, float, np.integer, np.floating)) \
                or not 0 <= self.tol < np.inf:
            raise ValueError(f"The 'tol' parameter of {who} must be a float in the range [0.0, inf). Got {self.tol!r} "
                             "instead.")

    def _priors(self, nk: np.ndarray) -> np.ndarray:
        """priors_: the class frequencies, or the given priors (non-negative, renormalised with scikit-learn's warning)"""
        if self.priors is None:
            return nk / float(nk.sum())
        p = np.asarray(self.priors, dtype=np.float64).ravel()
        if p.size != nk.size:
            raise ValueError(f"priors has {p.size} entries, but y holds {nk.size} classes")
        if np.any(p < 0):
            raise ValueError("priors must be non-negative")
        if np.abs(np.sum(p) - 1.0) > 1e-5:
            warnings.warn("The priors do not sum to 1. Renormalizing", UserWarning)
            p = p / p.sum()
        return p

    @staticmethod
    def _scatter(ctx, X, y, labels, means, weights, row_mask, mask_keep, n: float) -> np.ndarray:
        """one scatter pass, checked against the class-sum pass's rows"""
        res = ctx.class_scatter(X, y, labels, means, weights, row_mask=row_mask, mask_keep=mask_keep)
        if res["kept"] != n or res["unmatched"] > 0 or res["nonfinite"] > 0:
            raise RuntimeError("the scatter pass saw other labels than the label check")
        _check_finite(res["scatter"])
        return res["scatter"]

    def fit(self, X, y, row_mask=None, mask_keep: int = 1) -> "B200LinearDiscriminantAnalysis":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``.  Sets coef_, intercept_, classes_, means_,
        priors_, covariance_ (lsqr, eigen, or store_covariance), xbar_ (svd), scalings_ and explained_variance_ratio_
        (svd, eigen) and n_features_in_."""
        self._check_params()
        ctx, solver, shrink = self.ctx, self.solver, self.shrinkage
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=True) as (X, y, row_mask, labels, classes):
            d, K = X.shape[1], classes.size
            cs = ctx.class_sums(X, y, labels, None, row_mask=row_mask, mask_keep=mask_keep)
            nk, n = cs["sums"][:, d], cs["kept"]
            if cs["unmatched"] > 0 or cs["nonfinite"] > 0 or nk.sum() != n or np.any(nk == 0):
                raise RuntimeError("the class-sum pass saw other labels than the label check")
            _check_finite(cs["sums"])
            means = cs["sums"][:, :d] / nk[:, None]
            if n <= K:
                raise ValueError("The number of samples must be more than the number of classes.")
            priors = self._priors(nk)
            max_components = min(K - 1, d)
            if self.n_components is not None and self.n_components > max_components:
                raise ValueError("n_components cannot be larger than min(n_features, n_classes - 1).")
            freq = self.priors is None

            def scatter(weights):
                return self._scatter(ctx, X, y, labels, means, weights, row_mask, mask_keep, n)
            if solver == "svd":
                sw1 = scatter(None)
                cov = None if not self.store_covariance else (sw1 / n if freq else scatter(priors / nk))
            else:
                cov = scatter(priors / nk)
                sw1 = None if solver != "eigen" else (cov * n if freq else scatter(None))
        self._max_components = max_components if self.n_components is None else int(self.n_components)
        for name in ("covariance_", "xbar_", "scalings_", "explained_variance_ratio_"):
            self.__dict__.pop(name, None)
        if solver == "svd":
            coef, intercept, self.xbar_, self.scalings_, self.explained_variance_ratio_ = _lda_svd(
                sw1, means, nk, priors, float(self.tol), self._max_components)
            if cov is not None:
                self.covariance_ = cov
        elif solver == "lsqr":
            self.covariance_ = _shrunk(cov, shrink)
            coef, intercept = _lda_lstsq(self.covariance_, means, priors)
        else:
            self.covariance_ = _shrunk(cov, shrink)
            xbar = nk @ means / n
            total = (sw1 + (nk[:, None] * (means - xbar)).T @ (means - xbar)) / n
            coef, intercept, self.scalings_, self.explained_variance_ratio_ = _lda_eigen(
                self.covariance_, _shrunk(total, shrink), means, priors, self._max_components)
        if K == 2:                                      # scikit-learn's binary collapse
            coef = (coef[1, :] - coef[0, :]).reshape(1, -1)
            intercept = np.reshape(intercept[1] - intercept[0], (1,))
        _check_finite(coef)
        self.coef_, self.intercept_ = coef, intercept
        self.classes_, self.means_, self.priors_ = classes, means, priors
        self.n_features_in_ = int(d)
        self._n_features_out = self._max_components
        return self

    def predict_proba(self, X):
        """The class probabilities, (n, K) fp64: [1 - p, p] with p = expit(decision) for two classes (one pass), else
        scikit-learn's softmax of the decisions -- on the host for host rows, in place on the device for device rows
        (an f64 ``DeviceArray``)."""
        if self.classes_.size == 2:
            Xc = self._checked_rows(X)
            return self.ctx.logistic_predict(Xc, self.coef_[0], float(self.intercept_[0]), proba=True)["proba"]
        from sklearn.utils.extmath import softmax
        dec = self.decision_function(X)
        if isinstance(dec, native.DeviceArray):
            self.ctx.softmax_rows(dec)
            return dec
        return softmax(dec, copy=False)

    def predict_log_proba(self, X):
        """log(predict_proba(X)) for host rows, zeros raised to the smallest normal first, as scikit-learn does."""
        if isinstance(X, native.DeviceArray):
            raise ValueError("predict_log_proba takes host rows (predict_proba returns device probabilities)")
        p = self.predict_proba(X)
        p[p == 0.0] += np.finfo(p.dtype).smallest_normal
        return np.log(p)

    def transform(self, X):
        """The projection on the discriminant directions, (n, c) fp64 in one pass: (x - xbar_) scalings_ for 'svd'
        (c = min(rank, n_components)), x scalings_ for 'eigen' (c = n_components); float64 for host rows, an f64
        ``DeviceArray`` for device rows."""
        if self.solver == "lsqr":
            raise NotImplementedError("transform not implemented for 'lsqr' solver (use 'svd' or 'eigen').")
        S = self.scalings_[:, : self._max_components]
        Xc = self._checked_rows(X)
        if S.shape[1] == 0:
            return np.empty((Xc.shape[0], 0))
        b = -(self.xbar_ @ S) if self.solver == "svd" else np.zeros(S.shape[1])
        return self.ctx.classify(Xc, S.T, b, np.arange(max(S.shape[1], 2), dtype=np.float32),
                                 decision=True)["decision"]

    def fit_transform(self, X, y, row_mask=None, mask_keep: int = 1):
        """fit, then transform every row of X."""
        return self.fit(X, y, row_mask, mask_keep).transform(X)

    def _sk_params(self) -> dict:
        return dict(solver=self.solver, shrinkage=self.shrinkage, priors=self.priors, n_components=self.n_components,
                    store_covariance=self.store_covariance, tol=self.tol)

    def _sk_prepare(self, reg) -> None:
        """the attributes only some solvers set"""
        for name in ("covariance_", "xbar_", "scalings_", "explained_variance_ratio_"):
            if name in self.__dict__:
                setattr(reg, name, getattr(self, name).copy())

    def __repr__(self) -> str:
        return f"B200LinearDiscriminantAnalysis(solver={self.solver!r})"


# ---- QuadraticDiscriminantAnalysis: every class's scatter in one fp64 pass, K quadratic forms per row (DESIGN.md
# section 17) -------------------------------------------------------------------------------------------------------
_QDA_SOLVERS = ("svd", "eigen")


def _qda_class(scatter: np.ndarray, nk: int, solver: str, shrinkage, reg_param: float):
    """(scalings, rotations, covariance) of one class from its scatter S_k, as scikit-learn's ``_solve_svd`` and
    ``_solve_eigen`` compute them from its rows: 'svd' takes the eigenvalues and eigenvectors of S_k / (n_k - 1) for the
    squared singular values and right singular vectors of the centred rows (descending), 'eigen' those of the (shrunk)
    biased covariance S_k / n_k."""
    import scipy.linalg
    if solver == "svd":
        lam, V = np.linalg.eigh(scatter / (nk - 1))
        scaling = np.maximum(lam[::-1], 0.0)
        scaling = (1 - reg_param) * scaling + reg_param
        rotation = V[:, ::-1]
        return scaling, rotation, scaling * rotation @ rotation.T
    cov = _shrunk(scatter / nk, shrinkage)
    scaling, rotation = scipy.linalg.eigh(cov)
    order = np.argsort(scaling)[::-1]
    return scaling[order], rotation[:, order], cov


class B200QuadraticDiscriminantAnalysis(B200RidgeClassifier):
    """``sklearn.discriminant_analysis.QuadraticDiscriminantAnalysis`` for 2 to ``native.MAX_CLASSES`` classes, fitted
    on the H100.  A fit is the class counts and means (one class-sum pass) and every class's own scatter
    S_k = sum over its rows of (x - m_k)(x - m_k)^T from one fp64 tensor-core pass that reads the rows once, in class
    order (``class_scatters``).  The solvers are scikit-learn's, restated on these K D x D matrices on the host: 'svd'
    takes the eigendecomposition of S_k / (n_k - 1) for the SVD of the class's centred rows, 'eigen' that of the (shrunk)
    biased covariance S_k / n_k.  The columns of ``rotations_`` equal scikit-learn's up to their sign; nothing else
    depends on those signs.

    ``decision_function``, ``predict`` and ``score`` are one fp64 pass each (``qda_decision``: the K quadratic forms
    -1/2 |(x - m_k) W_k|^2 + c_k per row on the tensor core, W_k = rotations_[k] scalings_[k]^-1/2).  ``predict_proba``
    is scikit-learn's normalisation of the decisions, on the device for device rows.  Labels and their refusals are
    ``B200RidgeClassifier``'s.

    Refused: shrinkage='auto' (Ledoit-Wolf needs each class's fourth moments), a covariance_estimator, shrinkage with the
    'svd' solver, sample_weight, priors whose length is not the class count, more than ``native.MAX_CLASSES`` classes,
    continuous, multilabel or non-finite y, and non-finite X.  One class, a class of one row and a class covariance that
    is not full rank raise scikit-learn's errors."""
    _sk_module = "discriminant_analysis"
    _sk_name = "QuadraticDiscriminantAnalysis"
    _sk_attrs = ("classes_", "means_", "priors_", "n_features_in_")
    _label_who = "B200QuadraticDiscriminantAnalysis"

    def __init__(self, *, solver: str = "svd", shrinkage=None, priors=None, reg_param: float = 0.0,
                 store_covariance: bool = False, tol: float = 1e-4, covariance_estimator=None,
                 ctx: Optional[native.Context] = None):
        self.solver = solver
        self.shrinkage = shrinkage
        self.priors = priors
        self.reg_param = reg_param
        self.store_covariance = store_covariance
        self.tol = tol
        self.covariance_estimator = covariance_estimator
        self._ctx = ctx

    @staticmethod
    def _real(v) -> bool:
        return not isinstance(v, (bool, str)) and isinstance(v, (int, float, np.integer, np.floating))

    def _check_params(self):
        who = "B200QuadraticDiscriminantAnalysis"
        if self.solver not in _QDA_SOLVERS:
            raise ValueError(f"The 'solver' parameter of {who} must be a str among {{'eigen', 'svd'}}. Got "
                             f"{self.solver!r} instead.")
        s = self.shrinkage
        if isinstance(s, str) and s == "auto":
            raise ValueError(f"shrinkage='auto' is not supported by {who}: the Ledoit-Wolf estimate needs each class's "
                             "sum of |z|^4 over its standardised rows, a second gathered pass; use shrinkage=None or a "
                             "float")
        if s is not None and (not self._real(s) or not 0 <= s <= 1):
            raise ValueError(f"The 'shrinkage' parameter of {who} must be a str among {{'auto'}}, a float in the range "
                             f"[0, 1] or None. Got {s!r} instead.")
        if not self._real(self.reg_param) or not 0 <= self.reg_param <= 1:
            raise ValueError(f"The 'reg_param' parameter of {who} must be a float in the range [0, 1]. Got "
                             f"{self.reg_param!r} instead.")
        if not self._real(self.tol) or not 0 <= self.tol < np.inf:
            raise ValueError(f"The 'tol' parameter of {who} must be a float in the range [0.0, inf). Got {self.tol!r} "
                             "instead.")
        if self.covariance_estimator is not None:
            raise ValueError(f"covariance_estimator is not supported by {who}: each class's covariance is the "
                             "empirical one (with shrinkage=None or a float)")
        if self.solver == "svd" and s is not None:
            raise NotImplementedError(f"shrinkage not supported with 'svd' solver. ({who})")

    @classmethod
    def _check_class_count(cls, classes, more: bool) -> None:
        if more:
            raise ValueError(f"{cls._label_who} fits at most {native.MAX_CLASSES} classes, y has more")
        if classes.size < 2:
            raise ValueError(f"The number of classes has to be greater than one. Got {classes.size} class.")

    def fit(self, X, y, row_mask=None, mask_keep: int = 1,
            sample_weight=None) -> "B200QuadraticDiscriminantAnalysis":
        """X: (n, D) host array (any float dtype; staged as fp32) or a ``DeviceArray`` (f32 / bf16); ``row_mask``
        (uint8 per row) restricts the fit to rows equal to ``mask_keep``.  Sets classes_, means_, priors_, scalings_ and
        rotations_ (lists of K), covariance_ (with store_covariance) and n_features_in_."""
        _refuse_sample_weight(sample_weight, "B200QuadraticDiscriminantAnalysis")
        self._check_params()
        ctx = self.ctx
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=True) as (X, y, row_mask, labels, classes):
            d, K = X.shape[1], classes.size
            if self.priors is not None and np.size(self.priors) != K:
                raise ValueError(f"priors has {np.size(self.priors)} entries, but y holds {K} classes "
                                 "(B200QuadraticDiscriminantAnalysis)")
            cs = ctx.class_sums(X, y, labels, None, row_mask=row_mask, mask_keep=mask_keep)
            nk, n = cs["sums"][:, d], cs["kept"]
            if cs["unmatched"] > 0 or cs["nonfinite"] > 0 or nk.sum() != n or np.any(nk == 0):
                raise RuntimeError("the class-sum pass saw other labels than the label check")
            _check_finite(cs["sums"])
            means = cs["sums"][:, :d] / nk[:, None]
            sc = ctx.class_scatters(X, y, labels, means, row_mask=row_mask, mask_keep=mask_keep)
            if sc["kept"] != n or sc["unmatched"] > 0 or sc["nonfinite"] > 0 or np.any(sc["class_counts"] != nk):
                raise RuntimeError("the scatter pass saw other labels than the class-sum pass")
            _check_finite(sc["scatters"])
        priors = nk / float(n) if self.priors is None else np.array(self.priors)
        cov, scalings, rotations = [], [], []
        for k, label in enumerate(classes):
            if nk[k] == 1:
                raise ValueError(f"y has only 1 sample in class {label!s}, covariance is ill defined.")
            n_k = int(nk[k])
            # scikit-learn's svd of fewer rows than features has only n_k singular values, so its rank check fails
            # whatever reg_param is; the eigendecomposition has d values and cannot decide that
            small = self.solver == "svd" and n_k < d
            scaling, rotation, cov_k = (None, None, None) if small else _qda_class(
                sc["scatters"][k], n_k, self.solver, self.shrinkage, float(self.reg_param))
            if small or np.sum(scaling > self.tol) < d:
                if self.solver == "svd" and n_k <= d:
                    raise np.linalg.LinAlgError(
                        f"The covariance matrix of class {label} is not full rank. When using `solver='svd'` the "
                        f"number of samples in each class should be more than the number of features, but class "
                        f"{label} has {n_k} samples and {d} features. Try using `solver='eigen'` and setting the "
                        f"parameter `shrinkage` for regularization.")
                param = "shrinkage" if self.solver == "eigen" else "reg_param"
                raise np.linalg.LinAlgError(f"The covariance matrix of class {label} is not full rank. Increase the "
                                            f"value of `{param}` to reduce the collinearity.")
            cov.append(cov_k)
            scalings.append(scaling)
            rotations.append(rotation)
        self.__dict__.pop("covariance_", None)
        if self.store_covariance:
            self.covariance_ = cov
        self.classes_, self.means_, self.priors_ = classes, means, priors
        self.scalings_, self.rotations_ = scalings, rotations
        self.n_features_in_ = int(d)
        return self

    def _operands(self):
        """(means, W (K, d, d), c (K,)) of the decisions d_k = -1/2 |(x - m_k) W_k|^2 + c_k"""
        W = np.stack([R * (S ** (-0.5)) for R, S in zip(self.rotations_, self.scalings_)])
        c = -0.5 * np.array([np.sum(np.log(S)) for S in self.scalings_]) + np.log(self.priors_)
        return self.means_, W, c

    def _decide(self, X, y=None, **kw):
        """one qda_decision pass; host rows take the class indices as labels"""
        labels = self._fp32_classes(self.classes_) if isinstance(X, native.DeviceArray) else \
            np.arange(self.classes_.size, dtype=np.float32)
        return self.ctx.qda_decision(X, *self._operands(), labels, y, **kw)

    def decision_function(self, X):
        """d_1 - d_0 ((n,)) for two classes, the (n, K) decisions for more, in fp64: float64 for host rows, an f64
        ``DeviceArray`` for device rows."""
        X = self._checked_rows(X)
        if self.classes_.size == 2:
            return self._decide(X, diff=True)["diff"]
        return self._decide(X, decision=True)["decision"]

    def predict(self, X):
        """classes_ of the largest decision (the first of equal ones): an ndarray of classes_' dtype for host rows, an
        f32 ``DeviceArray`` for device rows (classes_ must then be fp32 values)."""
        labels = self._decide(self._checked_rows(X), label=True)["label"]
        if isinstance(labels, native.DeviceArray):
            return labels
        return self.classes_[labels.astype(np.intp)]

    def score(self, X, y, row_mask=None, mask_keep: int = 1):
        """Accuracy over the kept rows (labels outside classes_ count as wrong): the counts of one decision pass."""
        with self._stage_targets(X, y, row_mask, mask_keep, fitting=False) as (X, y, row_mask, labels, _):
            s = self.ctx.qda_decision(self._checked_rows(X), *self._operands(), labels, y, row_mask=row_mask,
                                      mask_keep=mask_keep)
        if s["kept"] == 0:
            raise _too_few_rows((0,))
        return float(s["correct"] / s["kept"])

    def predict_proba(self, X):
        """The class probabilities, (n, K) fp64: scikit-learn's exp(d - max - log sum exp(d - max)) of the decisions for
        host rows, ``softmax_rows`` in place on the device for device rows (an f64 ``DeviceArray``)."""
        X = self._checked_rows(X)
        dec = self._decide(X, decision=True)["decision"]
        if isinstance(dec, native.DeviceArray):
            self.ctx.softmax_rows(dec)
            return dec
        return np.exp(self._log_proba(dec))

    @staticmethod
    def _log_proba(dec: np.ndarray) -> np.ndarray:
        ll = dec - dec.max(axis=1)[:, np.newaxis]
        return ll - np.log(np.exp(ll).sum(axis=1)[:, np.newaxis])

    def predict_log_proba(self, X):
        """The log class probabilities of host rows, scikit-learn's formula on the decisions."""
        if isinstance(X, native.DeviceArray):
            raise ValueError("predict_log_proba takes host rows (predict_proba returns device probabilities)")
        return self._log_proba(self._decide(self._checked_rows(X), decision=True)["decision"])

    def _sk_params(self) -> dict:
        return dict(solver=self.solver, shrinkage=self.shrinkage, priors=self.priors, reg_param=self.reg_param,
                    store_covariance=self.store_covariance, tol=self.tol)

    def _sk_prepare(self, reg) -> None:
        """the per-class lists"""
        reg.scalings_ = [s.copy() for s in self.scalings_]
        reg.rotations_ = [r.copy() for r in self.rotations_]
        if "covariance_" in self.__dict__:
            reg.covariance_ = [c.copy() for c in self.covariance_]

    def __repr__(self) -> str:
        return f"B200QuadraticDiscriminantAnalysis(solver={self.solver!r})"
