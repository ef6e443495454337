"""Designed statistics and high-precision references for the fp64 solve kernels (csrc/solve.cu: the blocked LDL^T,
the Householder + Sturm eigenvalue kernel and the Jacobi minimum-norm kernel).  Test infrastructure only.

A designed statistic S = [X 1 y]^T [X 1 y] is assembled from a chosen centred Gram A = Q diag(eigs) Q^T, column means m,
a mean of y and a right-hand side r, with no rows behind it: the spectrum, the conditioning and the rank of what the
kernels are asked to solve are known in advance.  With zero means the kernels' centring leaves S_xx untouched, so the
factorisation is tested alone.  References are computed in ``np.longdouble`` (64-bit significand on x86-64), which
resolves residuals a thousand times below fp64 rounding.
"""
from typing import Optional, Sequence, Tuple

import numpy as np

LD = np.longdouble
EPS = float(np.finfo(np.float64).eps)


def random_orthogonal(d: int, seed: int) -> np.ndarray:
    """Q of the QR of a seeded Gaussian, signs fixed so that diag(R) > 0."""
    G = np.random.RandomState(seed).standard_normal((d, d))
    Q, R = np.linalg.qr(G)
    return Q * np.where(np.diag(R) < 0, -1.0, 1.0)


def designed_statistic(d: int, eigs: Sequence[float], *, n: int = 1024, means: Optional[np.ndarray] = None,
                       ybar: float = 0.0, beta: Optional[np.ndarray] = None, r_perp: Optional[dict] = None,
                       seed: int = 0, Q: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(S, Q, eigs): the statistic of a centred Gram A = Q diag(eigs) Q^T (formed in longdouble, rounded to fp64).

    r = A beta (beta seeded if None) plus r_perp[k] * q_k for each {k: coefficient} in ``r_perp`` -- components along
    chosen eigen-directions, e.g. dropped ones.  S is assembled as [X 1 y]^T [X 1 y] would be:
    S_xx = A + n m m^T, S_x1 = n m, S_11 = n, S_1y = n ybar, S_xy = r + n m ybar, S_yy = beta.A.beta + n (1 + ybar^2)
    (a residual variance of 1 per row).  ``Q``: use this basis instead of a seeded random one."""
    eigs = np.asarray(eigs, dtype=np.float64)
    if Q is None:
        Q = random_orthogonal(d, seed)
    QL = Q.astype(LD)
    AL = (QL * eigs.astype(LD)) @ QL.T
    AL = (AL + AL.T) / 2
    rng = np.random.RandomState(seed + 7919)
    if beta is None:
        beta = rng.uniform(-1.0, 1.0, size=d)
    betaL = np.asarray(beta, dtype=np.float64).astype(LD)
    rL = AL @ betaL
    for k, c in (r_perp or {}).items():
        rL = rL + LD(c) * QL[:, k]
    m = np.zeros(d) if means is None else np.asarray(means, dtype=np.float64)
    mL, nL, yL = m.astype(LD), LD(n), LD(ybar)
    S = np.zeros((d + 2, d + 2))
    S[:d, :d] = (AL + nL * np.outer(mL, mL)).astype(np.float64)
    S[:d, d] = S[d, :d] = (nL * mL).astype(np.float64)
    S[d, d] = float(n)
    S[d, d + 1] = S[d + 1, d] = float(nL * yL)
    S[:d, d + 1] = S[d + 1, :d] = (rL + nL * mL * yL).astype(np.float64)
    S[d + 1, d + 1] = float(betaL @ (AL @ betaL) + nL * (1 + yL * yL))
    return S, Q, eigs


def exact_centred(S: np.ndarray, fit_intercept: bool = True):
    """(A, r, m, ybar) in longdouble: the centred (or, without an intercept, raw) normal equations of S -- the system
    the kernels are asked to solve, before their own fp64 rounding of the centring."""
    S = np.asarray(S, dtype=np.float64).astype(LD)
    d = S.shape[0] - 2
    n = S[d, d]
    if not fit_intercept:
        return S[:d, :d].copy(), S[:d, d + 1].copy(), np.zeros(d, dtype=LD), LD(0)
    m = S[:d, d] / n
    ybar = S[d, d + 1] / n
    return S[:d, :d] - n * np.outer(m, m), S[:d, d + 1] - n * m * ybar, m, ybar


def refined_solve(A, r, passes: int = 6) -> np.ndarray:
    """Reference beta* of A beta = r (A: longdouble, symmetric positive definite, kappa <= 1e13): an fp64 solve, then
    residual corrections with the residual in longdouble.  Each pass divides the error by about 1 / (kappa eps)."""
    A = np.asarray(A, dtype=LD)
    r = np.asarray(r, dtype=LD)
    A64 = A.astype(np.float64)
    beta = np.linalg.solve(A64, r.astype(np.float64)).astype(LD)
    for _ in range(passes):
        res = r - A @ beta
        beta = beta + np.linalg.solve(A64, res.astype(np.float64)).astype(LD)
    return beta


def truncated_solution(Q: np.ndarray, eigs: Sequence[float], r, cond: float = 1e-6) -> Tuple[np.ndarray, int]:
    """(beta, rank): the minimum-norm solution over the kept eigen-pairs of Q diag(eigs) Q^T, in longdouble.  An
    eigen-pair is kept when sqrt(max(lambda, 0)) > cond * sqrt(lambda_max): sklearn's rule for the singular values of
    the centred rows (lstsq(cond=tol)), with lambda <= 0 treated as 0."""
    lam = np.maximum(np.asarray(eigs, dtype=np.float64), 0.0)
    keep = np.sqrt(lam) > cond * np.sqrt(lam.max()) if lam.size else np.zeros(0, bool)
    QL = np.asarray(Q, dtype=np.float64).astype(LD)
    w = QL.T @ np.asarray(r, dtype=LD)
    inv = np.zeros(lam.size, dtype=LD)
    inv[keep] = 1 / lam[keep].astype(LD)
    return QL @ (inv * w), int(keep.sum())


def backward_error(A, r, beta) -> float:
    """||r - A beta||_inf / (||A||_inf ||beta||_inf + ||r||_inf), the residual in longdouble."""
    A = np.asarray(A, dtype=LD)
    r = np.asarray(r, dtype=LD)
    b = np.asarray(beta).astype(LD)
    res = np.max(np.abs(r - A @ b))
    den = np.max(np.sum(np.abs(A), axis=1)) * np.max(np.abs(b)) + np.max(np.abs(r))
    return float(res / den) if den > 0 else float(res)


def ldlt_pivots(A) -> np.ndarray:
    """Pivots D_k of the unpivoted LDL^T of A (longdouble).  The LDL^T kernel refuses a statistic when a pivot is not
    above 1e-12 times the largest diagonal entry."""
    A = np.array(A, dtype=LD)
    d = A.shape[0]
    piv = np.empty(d, dtype=LD)
    for k in range(d):
        piv[k] = A[k, k]
        if k + 1 < d:
            col = A[k + 1:, k].copy()
            A[k + 1:, k + 1:] -= np.outer(col, col) / piv[k]
    return piv.astype(np.float64)


def integer_window_rows(n: int = 50_000, top: int = 10_000, seed: int = 1) -> Tuple[np.ndarray, np.ndarray]:
    """Integer-valued fp32 rows whose statistic is exact in fp64 and whose centred Gram is accepted by the LDL^T test
    yet has rank 1 under sklearn's rule: x1 uniform on 0 .. top, x2 = x1 except one entry raised by 1,
    y = 0.5 x1 + integer noise."""
    rng = np.random.RandomState(seed)
    x1 = rng.randint(0, top + 1, n).astype(np.float32)
    x2 = x1.copy()
    x2[n // 2] += 1
    y = (0.5 * x1 + rng.randint(-50, 50, n)).astype(np.float32)
    return np.stack([x1, x2], 1), y
