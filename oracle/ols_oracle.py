"""CPU ORACLE for the stage_1 retrain hot path.  TEST INFRASTRUCTURE ONLY.

This module is the *checker*, never the product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it.  Nothing under ``bodywork-mlops-demo_b200/`` imports it.

It restates, in plain numpy (float64), the arithmetic the reference performs in
``mlops_simulation/stage_1_train_model.py``:

====================  =====================================================================
oracle function       reference it follows
====================  =====================================================================
``split_indices``     ``train_test_split(X, y, test_size=0.2, random_state=42)``
                      stage_1_train_model.py:98-103 -> sklearn/model_selection/_split.py
                      (ShuffleSplit._iter_indices: ``perm = RandomState(seed).permutation(n)``,
                      ``test = perm[:n_test]``, ``train = perm[n_test:n_test+n_train]``,
                      ``n_test = ceil(test_size*n)``, ``n_train = floor((1-test_size)*n)``)
``fit_lstsq``         ``LinearRegression(fit_intercept=True).fit``  stage_1_train_model.py:105-106
                      -> sklearn/linear_model/_base.py: centre X and y, ``scipy.linalg.lstsq``
                      (LAPACK gelsd, ``cond=tol=1e-6``), ``intercept_ = y_mean - x_mean @ coef_``
``gram_stats``        (no reference counterpart: the sufficient statistic ``[X 1 y]^T [X 1 y]``
                      the CUDA path accumulates; defined here in float64, chunked)
``fit_from_stats``    same minimiser as ``fit_lstsq`` written on the normal equations of the
                      centred problem; ridge term as in sklearn/linear_model/_ridge.py
                      (``(Xc^T Xc + alpha I) w = Xc^T yc``).  Rank-deficient problems fall back
                      to the eigen pseudo-inverse == gelsd's minimum-norm solution.
``predict``           ``model.predict``  stage_1_train_model.py:107, stage_2_serve_model.py:78
                      -> ``X @ coef_ + intercept_``
``metrics``           ``model_metrics``  stage_1_train_model.py:79-90 -> sklearn/metrics/_regression.py
                      MAPE = mean(|yhat-y| / max(|y|, eps_f64)); R^2 = 1 - SSres/SStot;
                      max_error = max|y - yhat|
``train_model``       ``train_model``  stage_1_train_model.py:93-108 (generalised from the
                      reference's single ``X`` column to ``X0..X{D-1}``)
``generate_dataset``  ``generate_dataset`` stage_3_synthetic_data_generation.py:28-43, seeded and
                      generalised to D columns
``column_table``      (no reference counterpart: seeded columns of the shapes real tables have --
                      offset, scaled, integer / 0-1, constant, correlated -- for the kernels' precision)
``stat_error``        (no reference counterpart: a scale-free distance between two statistics)
====================  =====================================================================

Pinning.  The reference has no tests and no golden vectors for this path (SURVEY.md section 8c);
the arithmetic lives in scikit-learn (pinned 0.24.0 by the reference's bodywork.yaml:15;
1.9.0 in this image).  The oracle is therefore pinned two ways:

* ``tests/golden/*.npz`` were produced by importing the *unmodified* reference module
  ``/root/reference/mlops_simulation/stage_1_train_model.py`` (boto3 stubbed) and calling its
  ``train_model`` on seeded data -- see ``oracle/make_golden.py`` (committed).
* ``tests/test_oracle.py`` checks every function here against those vectors and against
  scikit-learn itself (installed in the image) on seeded inputs.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import numpy as np

F64_EPS = float(np.finfo(np.float64).eps)


# --------------------------------------------------------------------------------------
# split  (stage_1_train_model.py:98-103)
# --------------------------------------------------------------------------------------
def split_sizes(n: int, test_size: float = 0.2) -> Tuple[int, int]:
    """(n_train, n_test) as sklearn's _validate_shuffle_split computes them."""
    n_test = int(math.ceil(test_size * n))
    n_train = int(math.floor((1.0 - test_size) * n))
    return n_train, n_test


def split_indices(n: int, test_size: float = 0.2, seed: int = 42) -> Tuple[np.ndarray, np.ndarray]:
    """(train_idx, test_idx) exactly as train_test_split(..., random_state=seed) draws them."""
    n_train, n_test = split_sizes(n, test_size)
    perm = np.random.RandomState(seed).permutation(n)
    test = perm[:n_test]
    train = perm[n_test:n_test + n_train]
    return train, test


# --------------------------------------------------------------------------------------
# fit  (stage_1_train_model.py:105-106)
# --------------------------------------------------------------------------------------
def fit_lstsq(X: np.ndarray, y: np.ndarray, fit_intercept: bool = True, cond: float = 1e-6) -> Dict:
    """Centre, minimum-norm least squares (gelsd), intercept -- the reference's fit."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    if fit_intercept:
        x_mean = X.mean(axis=0)
        y_mean = y.mean()
    else:
        x_mean = np.zeros(X.shape[1])
        y_mean = 0.0
    Xc = X - x_mean
    yc = y - y_mean
    coef, _, rank, sing = np.linalg.lstsq(Xc, yc, rcond=cond)
    intercept = y_mean - x_mean @ coef
    return {"coef": coef, "intercept": float(intercept), "rank": int(rank), "singular": sing}


def gram_stats(X: np.ndarray, y: np.ndarray, chunk: int = 1 << 16) -> np.ndarray:
    """S = [X 1 y]^T [X 1 y] in float64, accumulated over row chunks.  Shape (D+2, D+2).

    Index order: features 0..D-1, then the ones column (D), then y (D+1).
    """
    n, d = X.shape
    S = np.zeros((d + 2, d + 2), dtype=np.float64)
    for r0 in range(0, n, chunk):
        Xb = np.asarray(X[r0:r0 + chunk], dtype=np.float64)
        yb = np.asarray(y[r0:r0 + chunk], dtype=np.float64)
        Z = np.empty((Xb.shape[0], d + 2), dtype=np.float64)
        Z[:, :d] = Xb
        Z[:, d] = 1.0
        Z[:, d + 1] = yb
        S += Z.T @ Z
    return S


def fit_from_stats(S: np.ndarray, alpha: float = 0.0, fit_intercept: bool = True,
                   cond: float = 1e-6) -> Dict:
    """Solve the (ridge) least-squares problem from the sufficient statistic S."""
    S = np.asarray(S, dtype=np.float64)
    d = S.shape[0] - 2
    n = S[d, d]
    sx = S[:d, d]
    sy = S[d, d + 1]
    if fit_intercept:
        x_mean = sx / n
        y_mean = sy / n
    else:
        x_mean = np.zeros(d)
        y_mean = 0.0
    A = S[:d, :d] - n * np.outer(x_mean, x_mean) if fit_intercept else S[:d, :d].copy()
    r = S[:d, d + 1] - n * x_mean * y_mean if fit_intercept else S[:d, d + 1].copy()
    A = 0.5 * (A + A.T)
    lam, V = np.linalg.eigh(A)
    lam = np.maximum(lam, 0.0)
    sing = np.sqrt(lam)[::-1]
    smax = sing[0] if sing.size else 0.0
    keep = np.sqrt(lam) > cond * smax
    rank = int(keep.sum())
    if alpha > 0.0:
        coef = np.linalg.solve(A + alpha * np.eye(d), r)
    elif rank == d:
        coef = np.linalg.solve(A, r)
    else:
        inv = np.zeros_like(lam)
        inv[keep] = 1.0 / lam[keep]
        coef = V @ (inv * (V.T @ r))
    intercept = y_mean - x_mean @ coef
    return {"coef": coef, "intercept": float(intercept), "rank": rank, "singular": sing}


# --------------------------------------------------------------------------------------
# predict / metrics  (stage_1_train_model.py:107, 79-90)
# --------------------------------------------------------------------------------------
def predict(X: np.ndarray, coef: np.ndarray, intercept: float) -> np.ndarray:
    return np.asarray(X, dtype=np.float64) @ np.asarray(coef, dtype=np.float64) + intercept


def metrics(y_actual: np.ndarray, y_predicted: np.ndarray) -> Dict[str, float]:
    y = np.asarray(y_actual, dtype=np.float64)
    p = np.asarray(y_predicted, dtype=np.float64)
    mape = float(np.mean(np.abs(p - y) / np.maximum(np.abs(y), F64_EPS)))
    ss_res = float(np.sum((y - p) ** 2))
    ss_tot = float(np.sum((y - y.mean()) ** 2))
    if ss_tot != 0.0:
        r2 = 1.0 - ss_res / ss_tot
    else:  # sklearn: perfect fit of a constant -> 1.0, otherwise 0.0 (force_finite)
        r2 = 1.0 if ss_res == 0.0 else 0.0
    max_res = float(np.max(np.abs(y - p)))
    return {"MAPE": mape, "r_squared": r2, "max_residual": max_res}


def score_stats(y: np.ndarray, p: np.ndarray) -> np.ndarray:
    """The ten reductions the CUDA scoring kernel produces (include/b2gram.h, b2_score):
    [sum_ape, sse, sum_y, sum_yy, max_abs_res, n, sum_p, sum_pp, sum_yp, max_ape]."""
    y = np.asarray(y, dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        max_ape = np.max(np.abs(p - y) / np.abs(y)) if y.size else 0.0
    return np.array([
        np.sum(np.abs(p - y) / np.maximum(np.abs(y), F64_EPS)),
        np.sum((y - p) ** 2), np.sum(y), np.sum(y * y), np.max(np.abs(y - p)) if y.size else 0.0,
        float(y.size), np.sum(p), np.sum(p * p), np.sum(y * p), max_ape])


def service_test_metrics(label: np.ndarray, score: np.ndarray) -> Dict[str, float]:
    """stage_4_test_model_scoring_service.py:86-90,101-105: APE = |score/label - 1|, MAPE = mean APE,
    'r_squared' = Pearson correlation(score, label), 'max_residual' = max APE."""
    label = np.asarray(label, dtype=np.float64)
    score = np.asarray(score, dtype=np.float64)
    ape = np.abs(score / label - 1.0)
    return {"MAPE": float(ape.mean()), "r_squared": float(np.corrcoef(score, label)[0, 1]),
            "max_residual": float(ape.max())}


# --------------------------------------------------------------------------------------
# train_model  (stage_1_train_model.py:93-108), generalised to D feature columns
# --------------------------------------------------------------------------------------
def train_model(X: np.ndarray, y: np.ndarray, test_size: float = 0.2, seed: int = 42) -> Dict:
    X = np.asarray(X)
    if X.ndim == 1:
        X = X.reshape(-1, 1)
    tr, te = split_indices(X.shape[0], test_size, seed)
    fit = fit_lstsq(X[tr], y[tr])
    m = metrics(y[te], predict(X[te], fit["coef"], fit["intercept"]))
    return {**fit, **m, "n_train": int(tr.size), "n_test": int(te.size)}


def train_model_sklearn(X: np.ndarray, y: np.ndarray) -> Dict:
    """The same sequence through scikit-learn itself -- the reference's own dependency calls
    (stage_1_train_model.py:98-107).  Used as the timed CPU arm and to pin this oracle."""
    from sklearn.linear_model import LinearRegression
    from sklearn.metrics import max_error, mean_absolute_percentage_error, r2_score
    from sklearn.model_selection import train_test_split
    if X.ndim == 1:
        X = X.reshape(-1, 1)
    X_train, X_test, y_train, y_test = train_test_split(X, y, test_size=0.2, random_state=42)
    reg = LinearRegression(fit_intercept=True)
    reg.fit(X_train, y_train)
    p = reg.predict(X_test)
    return {"coef": np.asarray(reg.coef_), "intercept": float(reg.intercept_), "rank": int(reg.rank_),
            "singular": np.asarray(reg.singular_),
            "MAPE": float(mean_absolute_percentage_error(y_test, p)),
            "r_squared": float(r2_score(y_test, p)), "max_residual": float(max_error(y_test, p)),
            "n_train": int(X_train.shape[0]), "n_test": int(X_test.shape[0])}


# --------------------------------------------------------------------------------------
# data  (stage_3_synthetic_data_generation.py:28-43), seeded, D columns
# --------------------------------------------------------------------------------------
def alpha_of_day(day_of_year: int, f: float = 6.0, kappa: float = 1.0, A: float = 0.5) -> float:
    """stage_3_synthetic_data_generation.py:31-33."""
    return kappa + A * math.sin(2.0 * math.pi * f * (day_of_year - 1) / 364.0)


def generate_dataset(n: int, d: int = 1, seed: int = 0, alpha: float = 1.0, beta: float = 0.5,
                     sigma: float = 10.0, drop_negative: bool = False,
                     dtype=np.float64) -> Tuple[np.ndarray, np.ndarray]:
    """X ~ U(0,100), eps ~ N(0,1), y = alpha + beta * sum_j X_j + sigma * eps."""
    rng = np.random.RandomState(seed)
    X = rng.uniform(0.0, 100.0, size=(n, d))
    eps = rng.normal(0.0, 1.0, size=n)
    y = alpha + beta * X.sum(axis=1) + sigma * eps
    if drop_negative:  # stage_3...:43  dataset.query('y >= 0')
        keep = y >= 0
        X, y = X[keep], y[keep]
    return np.ascontiguousarray(X.astype(dtype)), np.ascontiguousarray(y.astype(dtype))


# --------------------------------------------------------------------------------------
# structured columns: the shapes of real tabular features, for the kernels' precision
# --------------------------------------------------------------------------------------
COLUMN_FAMILIES = ("offset", "scaled", "integer", "constant", "correlated")

_OFFSET_COLUMNS = ((2021.0, 1.0), (1.0e4, 1.0), (-3.0e3, 10.0), (1.0e5, 10.0))   # (mean, sigma): a year, price levels
_SCALED_SIGMAS = (0.1, 0.3, 1.0, 3.0, 10.0)                                       # times the table's scale
_SCALED_MEANS = (0.0, 3.0, -3.0)                                                   # in units of the column's sigma
CONSTANT_VALUE = 2021.5                                                            # not representable in bf16


def bf16_spacing(x) -> np.ndarray:
    """Distance between adjacent bf16 values (8 significand bits) at |x|."""
    a = np.maximum(np.abs(np.asarray(x, dtype=np.float64)), np.finfo(np.float32).tiny)
    return np.exp2(np.floor(np.log2(a)) - 7.0)


def column_table(n: int, d: int, family: str, seed: int = 0, rho: float = 0.9, scale: float = 1.0,
                 bf16: bool = False) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Seeded float64 (X, y, sigma): n rows of d columns of one family, and each column's design spread.

    offset      means 2021, 1e4, -3e3, 1e5 with sigma 1 or 10 (cycled over the columns)
    scaled      sigma ``scale`` * (0.1 .. 10) with means 0, +3 sigma, -3 sigma; tables at scale 1e-3 and 1e3 cover
                sigma 1e-4 .. 1e4 (one table spans two decades only: sigma ratios of 1e6 within a table would make the
                centred Gram singular at the 1e-6 cutoff of sklearn's gelsd)
    integer     small integers 0..9, sparse 0/1 (p = 0.05), integers -3..3
    constant    column 0 holds CONSTANT_VALUE, the others are the offset family
    correlated  blocks of 8 columns with pairwise correlation ``rho``, mean 0, sigma 1

    Column j moves y by beta_j = b_j / sigma_j with |b_j| in [0.5, 2], so every column matters whatever its scale;
    y = 3 + X beta + N(0, 1).  ``bf16=True``: each offset column's sigma is raised to twice the bf16 spacing at its mean,
    so that rows stored as bf16 still vary (the caller rounds them).
    """
    if family not in COLUMN_FAMILIES:
        raise ValueError(f"unknown column family {family!r}")
    rng = np.random.RandomState(seed)
    j = np.arange(d)
    if family == "scaled":
        sigma = scale * np.array([_SCALED_SIGMAS[k % len(_SCALED_SIGMAS)] for k in j])
        mu = np.array([_SCALED_MEANS[k % len(_SCALED_MEANS)] for k in j]) * sigma
        X = mu + sigma * rng.standard_normal((n, d))
    elif family == "integer":
        kind = j % 3
        X = np.empty((n, d))
        X[:, kind == 0] = rng.randint(0, 10, size=(n, int((kind == 0).sum())))
        X[:, kind == 1] = (rng.rand(n, int((kind == 1).sum())) < 0.05)
        X[:, kind == 2] = rng.randint(-3, 4, size=(n, int((kind == 2).sum())))
        sigma = np.where(kind == 0, math.sqrt(99.0 / 12.0), np.where(kind == 1, math.sqrt(0.05 * 0.95), 2.0))
    elif family == "correlated":
        X = np.empty((n, d))
        for b0 in range(0, d, 8):
            w = min(8, d - b0)
            common = rng.standard_normal((n, 1))
            X[:, b0:b0 + w] = math.sqrt(rho) * common + math.sqrt(1.0 - rho) * rng.standard_normal((n, w))
        sigma = np.ones(d)
    else:                                           # offset, constant
        mu = np.array([_OFFSET_COLUMNS[k % len(_OFFSET_COLUMNS)][0] for k in j])
        sigma = np.array([_OFFSET_COLUMNS[k % len(_OFFSET_COLUMNS)][1] for k in j])
        if bf16:
            sigma = np.maximum(sigma, 2.0 * bf16_spacing(mu))
        X = mu + sigma * rng.standard_normal((n, d))
        if family == "constant":
            X[:, 0] = CONSTANT_VALUE
            sigma[0] = 0.0
    b = rng.uniform(0.5, 2.0, size=d) * rng.choice([-1.0, 1.0], size=d)
    beta = np.where(sigma > 0, b / np.where(sigma > 0, sigma, 1.0), 0.0)
    y = 3.0 + X @ beta + rng.standard_normal(n)
    return np.ascontiguousarray(X), y, sigma


def centred_moments(S: np.ndarray) -> Tuple[float, np.ndarray, np.ndarray]:
    """(n, means, C) of the statistic S: C = the centred second moments of [X y] (features 0..d-1, then y)."""
    S = np.asarray(S, dtype=np.float64)
    d = S.shape[0] - 2
    idx = list(range(d)) + [d + 1]
    n = float(S[d, d])
    m = S[idx, d] / n
    return n, m, S[np.ix_(idx, idx)] - n * np.outer(m, m)


def stat_error(S: np.ndarray, So: np.ndarray, floor: float = 1e-10) -> Tuple[float, float]:
    """Scale-free distance of a statistic S from the oracle's So, both [X 1 y]^T [X 1 y].

    Returns (max_ab |C_ab - Co_ab| / sqrt(Co_aa Co_bb),  max_j |xbar_j - xbaro_j| / sigma_j) over the features and y,
    with C the centred second moments (``centred_moments``) and sigma_j^2 = Co_jj / n.  Both are invariant to a column's
    offset and scale, so an error in a column's centred variance counts the same whether the column has mean 0 or
    1e5, and whether the largest entry of S is 1e3 or 1e13.  A column whose centred variance is zero (a constant) is
    measured against ``floor`` times its raw second moment: the level at which fp64 centring of S cancels anyway.
    """
    _, m, C = centred_moments(S)
    no, mo, Co = centred_moments(So)
    d = np.asarray(So).shape[0] - 2
    raw = np.abs(np.diag(np.asarray(So, dtype=np.float64)))[list(range(d)) + [d + 1]]
    var = np.maximum(np.diag(Co), floor * raw)
    stat = float(np.max(np.abs(C - Co) / np.sqrt(np.outer(var, var))))
    mean = float(np.max(np.abs(m - mo) / np.sqrt(var / no)))
    return stat, mean


def centred_condition(S: np.ndarray) -> float:
    """Condition number (largest / smallest eigenvalue) of the centred feature Gram of S."""
    C = centred_moments(S)[2][:-1, :-1]
    lam = np.linalg.eigvalsh(0.5 * (C + C.T))
    return float(lam[-1] / lam[0]) if lam[0] > 0 else float("inf")


def coef_error(coef: np.ndarray, coef_o: np.ndarray, So: np.ndarray) -> float:
    """max_j |coef_j - coefo_j| * sigma_j (sigma_j: the oracle's spread of feature j): the largest change of a
    prediction, in units of y, when feature j moves by one standard deviation.  For sigma = 1 columns it is the plain
    coefficient error."""
    no, _, Co = centred_moments(So)
    sd = np.sqrt(np.maximum(np.diag(Co)[:-1], 0.0) / no)
    return float(np.max(np.abs(np.asarray(coef) - np.asarray(coef_o)) * sd))
