"""numpy restatement of the refined fit (b2_fit_refined, DESIGN.md section 2), beside the fp64 oracle in
oracle/ols_oracle.py, which it uses for the unrefined solve.  Test infrastructure only: the CPU tests pin it to
scikit-learn, the GPU tests hold the CUDA path to the same algebra."""
from typing import Dict

import numpy as np

from oracle.ols_oracle import fit_from_stats


def refine_fit(X: np.ndarray, y: np.ndarray, S_approx: np.ndarray, alpha: float = 0.0, fit_intercept: bool = True,
               max_passes: int = 2, tol: float = 1e-10) -> Dict:
    """The refined fit of ``b2_fit_refined``: solve from an approximate statistic, then correct the solution with the
    exact float64 gradient of the rows, through the same approximate matrix.

    Model y = b0' + (x - m).beta with m = S_approx's column means (0 without an intercept) and b0' = its mean of y.  A pass
    forms e = y - b0' - (X - m) beta, g = (X - m)^T e, g_1 = sum e, and corrects dbeta = (A + alpha I)^-1 (g - alpha beta)
    (A: the centred / uncentred Gram of S_approx), db0' = g_1 / n.  step = max_j |dbeta_j| sigma_j / sigma_y (S_approx's
    centred diagonal).  It stops when step <= tol, or when a step exceeds the one before: the last kept correction then
    left a larger error than it found, and the state returns to before it.
    Returns coef, intercept, passes (corrections kept), step (the last one computed, 0 without passes), steps."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    S = np.asarray(S_approx, dtype=np.float64)
    d = S.shape[0] - 2
    n = S[d, d]
    base = fit_from_stats(S, alpha=alpha, fit_intercept=fit_intercept)
    beta = np.asarray(base["coef"], dtype=np.float64).copy()
    if fit_intercept:
        m, b0 = S[:d, d] / n, S[d, d + 1] / n
    else:
        m, b0 = np.zeros(d), 0.0
    out = {"coef": beta, "intercept": base["intercept"], "passes": 0, "step": 0.0, "steps": []}
    if max_passes == 0:
        return out
    A = S[:d, :d] - n * np.outer(m, m) if fit_intercept else S[:d, :d].copy()
    A = 0.5 * (A + A.T) + alpha * np.eye(d)
    sx = S[:d, d]
    sig = np.sqrt(np.maximum(np.diag(S)[:d] - sx * sx / n, 0.0))
    sy = np.sqrt(max(S[d + 1, d + 1] - S[d, d + 1] ** 2 / n, 0.0))
    Xm = X - m
    prev = (beta.copy(), b0)
    last, kept = np.inf, 0
    for _ in range(max_passes):
        e = y - b0 - Xm @ beta
        g, g1 = Xm.T @ e, float(e.sum())
        dbeta = np.linalg.solve(A, g - alpha * beta)
        step = float(np.max(np.abs(dbeta) * sig))
        step = step / sy if sy > 0 else step
        out["steps"].append(step)
        out["step"] = step
        if not step <= last:
            beta, b0 = prev[0].copy(), prev[1]
            kept = max(kept - 1, 0)
            break
        prev = (beta.copy(), b0)
        beta = beta + dbeta
        b0 = b0 + (g1 / n if fit_intercept else 0.0)
        last, kept = step, kept + 1
        if step <= tol:
            break
    out.update(coef=beta, intercept=float(b0 - m @ beta), passes=kept)
    return out

