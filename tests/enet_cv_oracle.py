"""numpy statement of b2_gram_folds + b2_solve_enet_cv (csrc/folds.cu, csrc/solve.cu: solve_enet_kernel in its
cross-validation mode), built on enet_oracle.enet_path_from_stats.  Test infrastructure only.

  * S_k: the statistic [X 1 y]^T [X 1 y] of the rows of fold k; S = sum_k S_k and T_k = sum_{j != k} S_j, both added in
    fold order from 0 (the kernels' order, so the sums here are bit-identical to theirs);
  * per l1_ratio, one grid from S (sklearn's _alpha_grid on the summed statistic), or the given alphas for all;
  * per (l1_ratio, fold), the Gram path of T_k over that grid;
  * the held-out error of a solution (w, b) from S_k alone: with n_k rows, means mu (x) and vbar (y) and C the centred
    second moments of [x y],  mse = (vbar - b - mu.w)^2 + max(w~^T C w~, 0) / n_k,  w~ = [w; -1];
  * the choice: the mean over folds, the first minimum per l1_ratio, a later l1_ratio only when strictly better.
"""
import numpy as np

from enet_oracle import alpha_grid, enet_path_from_stats, gram_inputs


def stat(X, y):
    A = np.column_stack([np.asarray(X, np.float64), np.ones(X.shape[0]), np.asarray(y, np.float64)])
    return A.T @ A


def fold_stats(X, y, ids, n_folds):
    """(n_folds, d + 2, d + 2): the statistic of the rows whose id is k (ids >= n_folds: dropped)."""
    return np.stack([stat(X[ids == k], y[ids == k]) for k in range(n_folds)])


def fold_sum(fold_S, skip=-1):
    """sum of the fold statistics other than `skip`, in fold order from 0."""
    t = np.zeros_like(fold_S[0])
    for j in range(fold_S.shape[0]):
        if j != skip:
            t = t + fold_S[j]
    return t


def heldout_mse(Sk, w, b):
    """The mean squared error of y ~ X w + b over the rows of the statistic Sk."""
    d = Sk.shape[0] - 2
    sel = list(range(d)) + [d + 1]
    nk = Sk[d, d]
    mu = Sk[sel, d] / nk
    C = Sk[np.ix_(sel, sel)] - nk * np.outer(mu, mu)
    wt = np.append(np.asarray(w, np.float64), -1.0)
    res = mu[d] - b - float(mu[:d] @ wt[:d])
    return res * res + max(float(wt @ C @ wt), 0.0) / nk


def enet_cv_from_stats(fold_S, l1_ratios=(1.0,), alphas=None, n_alphas=100, eps=1e-3, max_iter=1000, tol=1e-4,
                       positive=False, fit_intercept=True):
    """What b2_solve_enet_cv returns: alphas (L, A), mse (L, A, K), n_iter and gaps (L, K, A), coefs (L, K, A, d)."""
    fold_S = np.asarray(fold_S, np.float64)
    K, d = fold_S.shape[0], fold_S.shape[1] - 2
    l1 = np.atleast_1d(np.asarray(l1_ratios, np.float64))
    S = fold_sum(fold_S)
    _, q, _, _, _, n, _ = gram_inputs(S, fit_intercept)
    grids = [alpha_grid(q, n, r, eps, n_alphas, positive) if alphas is None else np.asarray(alphas, np.float64)
             for r in l1]
    A = grids[0].size
    out = {"alphas": np.stack(grids), "mse": np.empty((l1.size, A, K)), "n_iter": np.empty((l1.size, K, A), np.int64),
           "gaps": np.empty((l1.size, K, A)), "coefs": np.empty((l1.size, K, A, d))}
    for li, r in enumerate(l1):
        for k in range(K):
            p = enet_path_from_stats(fold_sum(fold_S, k), r, alphas=grids[li], max_iter=max_iter, tol=tol,
                                     positive=positive, fit_intercept=fit_intercept)
            out["n_iter"][li, k], out["gaps"][li, k], out["coefs"][li, k] = p["n_iter"], p["gaps"], p["coefs"]
            b = p["intercepts"] if fit_intercept else np.zeros(A)
            out["mse"][li, :, k] = [heldout_mse(fold_S[k], p["coefs"][i], b[i]) for i in range(A)]
    return out


def choose(mse, alphas, l1_ratios):
    """(alpha_, l1_ratio_, l index, alpha index) by sklearn's rule on mse (L, A, K)."""
    mean = np.mean(np.moveaxis(np.asarray(mse), 2, 1), axis=1)
    best, best_mse = (0, 0), np.inf
    for li in range(mean.shape[0]):
        i = int(np.argmin(mean[li]))
        if mean[li, i] < best_mse:
            best, best_mse = (li, i), mean[li, i]
    return float(alphas[best[0]][best[1]]), float(np.atleast_1d(l1_ratios)[best[0]]), best[0], best[1]
