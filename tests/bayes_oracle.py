"""numpy statement of b2_solve_bayes_ridge / b2_solve_ard / b2_score_std (DESIGN.md section 9).

Both iterations run from the statistic S = [X 1 y]^T [X 1 y] and, optionally, the anchor [w0, g0, s0, sse0] of one fp64
pass over the rows at w0 (g0 = sum (x - m) e, s0 = sum e, sse0 = sum e^2).  With the anchor the residual sum of squares is
exact for any w: sse(w) = sse0 - s0^2 / n - 2 D.g0 + D^T A D, D = w - w0; without it, sse = ||yc||^2 - 2 w.r + w^T A w.
"""
from __future__ import annotations

import numpy as np

EPS = np.finfo(np.float64).eps


def normal_equations(S: np.ndarray, fit_intercept: bool):
    """(A, r, m, ybar, n, ||yc||^2, y.var()) of S."""
    d = S.shape[0] - 2
    n = S[d, d]
    sy, syy = S[d, d + 1], S[d + 1, d + 1]
    m = S[:d, d] / n if fit_intercept else np.zeros(d)
    ybar = sy / n if fit_intercept else 0.0
    A = S[:d, :d] - n * np.outer(m, m)
    r = S[:d, d + 1] - n * m * ybar
    yy = syy - n * ybar * ybar
    y_var = max(syy / n - (sy / n) ** 2, 0.0)
    return A, r, m, ybar, n, yy, y_var


def anchor_of(X: np.ndarray, y: np.ndarray, w0: np.ndarray, fit_intercept: bool) -> np.ndarray:
    """[w0, g0, s0, sse0] of float64 rows at w0 (intercept ybar - m.w0), what b2_residual_moments returns after w0."""
    m = X.mean(axis=0) if fit_intercept else np.zeros(X.shape[1])
    b0 = (y.mean() - m @ w0) if fit_intercept else 0.0
    e = y - b0 - X @ w0
    return np.concatenate([w0, (X - m).T @ e, [e.sum(), e @ e]])


def _sse(A, r, yy, n, w, anchor, fit_intercept):
    d = w.size
    if anchor is None:
        return yy - 2.0 * w @ r + w @ A @ w
    w0, g0, s0, sse0 = anchor[:d], anchor[d:2 * d], anchor[2 * d], anchor[2 * d + 1]
    D = w - w0
    return sse0 - (s0 * s0 / n if fit_intercept else 0.0) - 2.0 * D @ g0 + D @ A @ D


def bayes_ridge(S, *, fit_intercept=True, alpha_1=1e-6, alpha_2=1e-6, lambda_1=1e-6, lambda_2=1e-6, alpha_init=None,
                lambda_init=None, max_iter=300, tol=1e-3, anchor=None, compute_score=False) -> dict:
    """BayesianRidge.fit (scikit-learn 1.9) in the eigenbasis of the centred Gram."""
    A, r, m, ybar, n, yy, y_var = normal_equations(S, fit_intercept)
    d = A.shape[0]
    lam, Q = np.linalg.eigh(A)
    lam = np.maximum(lam, 0.0)
    c = Q.T @ r
    alpha = 1.0 / (y_var + EPS) if alpha_init is None else float(alpha_init)
    lmb = 1.0 if lambda_init is None else float(lambda_init)

    def update():
        coef = Q @ (c / (lam + lmb / alpha))
        return coef, _sse(A, r, yy, n, coef, anchor, fit_intercept)

    def score(coef, sse):
        logdet = -np.sum(np.log(lmb + alpha * lam))
        s = lambda_1 * np.log(lmb) - lambda_2 * lmb + alpha_1 * np.log(alpha) - alpha_2 * alpha
        return s + 0.5 * (d * np.log(lmb) + n * np.log(alpha) - alpha * sse - lmb * np.sum(coef ** 2) + logdet
                          - n * np.log(2 * np.pi))

    scores, coef_old = [], None
    for it in range(max_iter):
        coef, sse = update()
        if compute_score:
            scores.append(score(coef, sse))
        gamma = np.sum(alpha * lam / (lmb + alpha * lam))
        lmb = (gamma + 2 * lambda_1) / (np.sum(coef ** 2) + 2 * lambda_2)
        alpha = (n - gamma + 2 * alpha_1) / (sse + 2 * alpha_2)
        if it != 0 and np.sum(np.abs(coef_old - coef)) < tol:
            break
        coef_old = coef.copy()
    coef, sse = update()
    if compute_score:
        scores.append(score(coef, sse))
    sigma = (Q / (alpha * lam + lmb)) @ Q.T
    return {"coef": coef, "intercept": ybar - m @ coef if fit_intercept else 0.0, "alpha": alpha, "lambda": lmb,
            "n_iter": it + 1, "scores": np.array(scores) if compute_score else None, "sigma": sigma}


def ard(S, *, fit_intercept=True, alpha_1=1e-6, alpha_2=1e-6, lambda_1=1e-6, lambda_2=1e-6, threshold_lambda=1e4,
        max_iter=300, tol=1e-3, anchor=None, compute_score=False) -> dict:
    """ARDRegression.fit (scikit-learn 1.9): sigma the exact inverse on the kept set; sigma returned d x d with zeros
    outside the kept rows and columns."""
    A, r, m, ybar, n, yy, y_var = normal_equations(S, fit_intercept)
    d = A.shape[0]
    alpha = 1.0 / (y_var + EPS)
    lmb = np.ones(d)
    keep = np.ones(d, dtype=bool)
    coef = np.zeros(d)
    scores, coef_old = [], None

    def solve():
        K = np.ix_(keep, keep)
        sig = np.linalg.inv(np.diag(lmb[keep]) + alpha * A[K])
        coef[keep] = alpha * sig @ r[keep]
        return sig

    for it in range(max_iter):
        sig = solve()
        sse = _sse(A, r, yy, n, coef, anchor, fit_intercept)
        gamma = 1.0 - lmb[keep] * np.diag(sig)
        lmb[keep] = (gamma + 2.0 * lambda_1) / (coef[keep] ** 2 + 2.0 * lambda_2)
        alpha = (n - gamma.sum() + 2.0 * alpha_1) / (sse + 2.0 * alpha_2)
        keep = lmb < threshold_lambda
        coef[~keep] = 0
        if compute_score:
            s = (lambda_1 * np.log(lmb) - lambda_2 * lmb).sum() + alpha_1 * np.log(alpha) - alpha_2 * alpha
            s += 0.5 * (np.linalg.slogdet(sig)[1] + n * np.log(alpha) + np.sum(np.log(lmb)))
            s -= 0.5 * (alpha * sse + (lmb * coef ** 2).sum())
            scores.append(s)
        if it > 0 and np.sum(np.abs(coef_old - coef)) < tol:
            break
        coef_old = coef.copy()
        if not keep.any():
            break
    sigma = np.zeros((d, d))
    if keep.any():
        sigma[np.ix_(keep, keep)] = solve()
    return {"coef": coef, "intercept": ybar - m @ coef if fit_intercept else 0.0, "alpha": alpha, "lambda": lmb,
            "n_iter": it + 1, "scores": np.array(scores) if compute_score else None, "sigma": sigma}


def score_std(X, mean, sigma, noise_var, coef, intercept):
    """(yhat, ystd) of predict(X, return_std=True)."""
    V = np.asarray(X, dtype=np.float64) - mean
    q = np.einsum("ij,ij->i", V @ sigma, V)
    return np.asarray(X, dtype=np.float64) @ coef + intercept, np.sqrt(np.maximum(q, 0.0) + noise_var)
