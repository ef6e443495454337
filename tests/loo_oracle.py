"""numpy fp64 statement of the leave-one-out error b2_ridge_loo computes (DESIGN.md section 6).  Test infrastructure.

Rows kept by the mask, n of them.  With an intercept m is their column mean and ybar their y mean, without both are 0.
V = X - m, A = V^T V = Q diag(lambda) Q^T (negative rounding eigenvalues as 0), c = Q^T V^T (y - ybar), Z = V Q.  For alpha:
w = 1 / (lambda + alpha), yhat = Z (c w), h = h0 + Z^2 w with h0 = 1 / n (0 without an intercept), e = ((y - ybar) - yhat) /
(1 - h); cv = e^2 per row and alpha, mse = mean over the kept rows.  This is scikit-learn's _RidgeGCV for n > D.
"""
from typing import Optional, Sequence, Tuple

import numpy as np


def ridge_loo(X, y, alphas: Sequence[float], mask: Optional[np.ndarray] = None, keep: int = 1,
              fit_intercept: bool = True) -> Tuple[np.ndarray, np.ndarray, int]:
    """(mse per alpha, cv of the kept rows (n_kept, n_alphas), index of the first smallest mse)."""
    X = np.asarray(X, dtype=np.float64)
    if X.ndim == 1:
        X = X.reshape(-1, 1)
    y = np.asarray(y, dtype=np.float64).ravel()
    if mask is not None:
        sel = np.asarray(mask) == keep
        X, y = X[sel], y[sel]
    n = X.shape[0]
    m = X.mean(axis=0) if fit_intercept else np.zeros(X.shape[1])
    ybar = y.mean() if fit_intercept else 0.0
    V = X - m
    yc = y - ybar
    lam, Q = np.linalg.eigh(V.T @ V)
    lam = np.maximum(lam, 0.0)
    c = Q.T @ (V.T @ yc)
    Z = V @ Q
    h0 = 1.0 / n if fit_intercept else 0.0
    al = np.asarray(alphas, dtype=np.float64).ravel()
    cv = np.empty((n, al.size))
    for a, alpha in enumerate(al):
        w = 1.0 / (lam + alpha)
        e = (yc - Z @ (c * w)) / (1.0 - (h0 + (Z * Z) @ w))
        cv[:, a] = e * e
    mse = cv.mean(axis=0)
    return mse, cv, int(np.argmin(mse))

