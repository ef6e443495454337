"""numpy fp64 statement of the multi-target leave-one-out error b2_ridge_classifier_loo computes (DESIGN.md section 13).
Test infrastructure, in the notation of tests/loo_oracle.py.

Rows kept by the mask, n of them, with class indices k(row) into K classes; T = 1 for two classes (the target of class
1), else K.  Targets t_k = +1 where the row's class is k, -1 otherwise; with an intercept m is the rows' column mean and
ybar_k = 2 n_k / n - 1, without both are 0.  V = X - m, A = V^T V = Q diag(lambda) Q^T (negative rounding eigenvalues as
0), R = V^T (t - ybar), C = Q^T R, Z = V Q.  For alpha: w = 1 / (lambda + alpha), h = h0 + Z^2 w (h0 = 1 / n with an
intercept), yhat = Z (C o w), e = ((t - ybar) - yhat) / (1 - h).  scoring None: cv = e^2, mse = mean over n T entries;
"accuracy": cv = p = t - e, correct = rows whose first argmax of p is the first argmax of t.  The first strictly best
alpha wins.  This is scikit-learn's _RidgeGCV with is_clf=True for n > D.
"""
from typing import Optional, Sequence

import numpy as np


def targets(k: np.ndarray, n_classes: int) -> np.ndarray:
    """(n, T) +-1 targets of class indices k (LabelBinarizer(pos_label=1, neg_label=-1))."""
    t = np.where(np.asarray(k)[:, None] == np.arange(n_classes)[None, :], 1.0, -1.0)
    return t[:, 1:2] if n_classes == 2 else t


def ridge_classifier_loo(X, k, n_classes: int, alphas: Sequence[float], mask: Optional[np.ndarray] = None,
                         keep: int = 1, fit_intercept: bool = True, scoring: Optional[str] = None) -> dict:
    """mse and correct per alpha, cv of the kept rows (n_kept, T, n_alphas), best, and coef (T, d) / intercept (T,) of
    the ridge classifier at alphas[best]."""
    X = np.asarray(X, dtype=np.float64)
    if X.ndim == 1:
        X = X.reshape(-1, 1)
    k = np.asarray(k).ravel()
    if mask is not None:
        sel = np.asarray(mask) == keep
        X, k = X[sel], k[sel]
    n, d = X.shape
    Y = targets(k, n_classes)
    m = X.mean(axis=0) if fit_intercept else np.zeros(d)
    ybar = Y.mean(axis=0) if fit_intercept else np.zeros(Y.shape[1])
    V = X - m
    Yc = Y - ybar
    lam, Q = np.linalg.eigh(V.T @ V)
    lam = np.maximum(lam, 0.0)
    C = Q.T @ (V.T @ Yc)
    Z = V @ Q
    h0 = 1.0 / n if fit_intercept else 0.0
    al = np.asarray(alphas, dtype=np.float64).ravel()
    cv = np.empty((n, Y.shape[1], al.size))
    mse, correct = np.empty(al.size), np.empty(al.size)
    for a, alpha in enumerate(al):
        w = 1.0 / (lam + alpha)
        h = h0 + (Z * Z) @ w
        e = (Yc - Z @ (C * w[:, None])) / (1.0 - h)[:, None]
        p = Y - e
        cv[:, :, a] = p if scoring == "accuracy" else e * e
        mse[a] = np.mean(e * e)
        correct[a] = np.sum(np.argmax(p, axis=1) == np.argmax(Y, axis=1))
    score = correct if scoring == "accuracy" else -mse
    best = 0
    for a in range(al.size):
        if score[a] > score[best]:
            best = a
    W = Q @ (C / (lam + al[best])[:, None])
    b = ybar - m @ W if fit_intercept else np.zeros(Y.shape[1])
    return {"mse": mse, "correct": correct, "cv": cv, "best": best, "coef": W.T, "intercept": b}
