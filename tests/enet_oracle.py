"""numpy statement of b2_solve_enet_path (csrc/solve.cu: solve_enet_kernel): scikit-learn's Gram coordinate descent
(sklearn/linear_model/_cd_fast.pyx: enet_coordinate_descent_gram, gap_enet_gram) with enet_path's scaling and
_alpha_grid, run on Q, q and ||yc||^2 formed from the statistic S = [X 1 y]^T [X 1 y].  Test infrastructure only.

The constant-column rule is the kernel's: a column whose centred diagonal is not above 1e-12 of its raw diagonal has its
row and column of Q and its entry of q set to 0, which is what exactly centred rows give sklearn (Q_jj == 0).
"""
import numpy as np

CONST_COL = 1e-12
RESOLUTION = float(np.finfo(np.float64).resolution)


def gram_inputs(S, fit_intercept=True):
    """(Q, q, y_norm2, m, ybar, n, live) from S, formed as build_normal_equations forms them (fp64)."""
    S = np.asarray(S, dtype=np.float64)
    d = S.shape[0] - 2
    n = S[d, d]
    inv_n = 1.0 / n if n > 0 else 0.0
    m = S[:d, d] * inv_n if fit_intercept else np.zeros(d)
    ybar = S[d, d + 1] * inv_n if fit_intercept else 0.0
    Q = S[:d, :d] - n * m[:, None] * m[None, :]
    q = S[:d, d + 1] - n * m * ybar
    y_norm2 = S[d + 1, d + 1] - n * ybar * ybar
    live = np.diag(Q) > CONST_COL * np.diag(S)[:d]
    Q = Q.copy()
    Q[~live, :] = 0.0
    Q[:, ~live] = 0.0
    q = np.where(live, q, 0.0)
    return Q, q, y_norm2, m, ybar, n, live


def alpha_grid(q, n, l1_ratio, eps=1e-3, n_alphas=100, positive=False):
    """sklearn's _alpha_grid from Xy = q."""
    amax = (max(0.0, float(np.max(q))) if positive else float(np.max(np.abs(q)))) / (n * l1_ratio)
    if amax <= RESOLUTION:
        return np.full(n_alphas, RESOLUTION)
    return np.geomspace(amax, amax * eps, num=n_alphas)


def _gap(w, Qw, q, y_norm2, l1, l2, positive):
    ww = float(w @ w) if l2 > 0 else 0.0
    qdw = float(w @ q)
    wqw = float(w @ Qw)
    r_norm2 = y_norm2 + wqw - 2.0 * qdw
    ry = y_norm2 - qdw
    if l1 == 0:
        xta = q - Qw
        dn = float(xta @ xta)
        if l2 == 0:
            return dn, xta, dn
        return r_norm2 + 0.5 * l2 * ww - ry + 1.0 / (2.0 * l2) * dn, xta, dn
    xta = q - Qw - l2 * w
    dn = float(np.max(xta)) if positive else float(np.max(np.abs(xta)))
    primal = 0.5 * (r_norm2 + l2 * ww) + l1 * float(np.sum(np.abs(w)))
    scale = l1 / dn if dn > l1 else 1.0
    dual = -0.5 * scale ** 2 * (r_norm2 + l2 * ww) + scale * ry
    return primal - dual, xta, dn


def cd_gram(w, l1, l2, Q, q, y_norm2, max_iter, tol, positive=False):
    """One alpha of enet_coordinate_descent_gram (cyclic, screening on when l1 > 0): (w, gap, tol * y_norm2, n_iter)."""
    w = np.array(w, dtype=np.float64)
    d = w.size
    Qw = Q @ w
    dw_tol = tol
    tol = tol * y_norm2
    gap, xta, dn = _gap(w, Qw, q, y_norm2, l1, l2, positive)
    if 0 <= gap <= tol:
        return w, gap, tol, 0
    screening = l1 > 0
    excluded = np.zeros(d, bool)
    active = np.arange(d)

    def screen(cands):
        radius = np.sqrt(2 * abs(gap)) / l1
        act = []
        for j in cands:
            if Q[j, j] == 0:
                w[j] = 0.0
                excluded[j] = True
                continue
            dj = (1 - abs(xta[j] / max(l1, dn))) / np.sqrt(Q[j, j] + l2)
            if dj <= radius:
                act.append(j)
                excluded[j] = False
            else:
                if w[j] != 0:
                    Qw[:] -= w[j] * Q[j]
                    w[j] = 0.0
                excluded[j] = True
        return np.asarray(act, dtype=np.int64)

    if screening:
        active = screen(range(d))
    for it in range(max_iter):
        w_max = dw_max = 0.0
        for j in active:
            if Q[j, j] == 0.0:
                continue
            wj = w[j]
            t = q[j] - Qw[j] + wj * Q[j, j]
            if positive and t < 0:
                w[j] = 0.0
            else:
                w[j] = np.sign(t) * max(abs(t) - l1, 0.0) / (Q[j, j] + l2)
            if w[j] != wj:
                Qw += (w[j] - wj) * Q[j]
            dw_max = max(dw_max, abs(w[j] - wj))
            w_max = max(w_max, abs(w[j]))
        if w_max == 0.0 or dw_max / w_max <= dw_tol or it == max_iter - 1:
            gap, xta, dn = _gap(w, Qw, q, y_norm2, l1, l2, positive)
            if gap <= tol:
                return w, gap, tol, it + 1
            if screening:
                active = screen([j for j in active if not excluded[j]])
    return w, gap, tol, max_iter


def enet_path_from_stats(S, l1_ratio=1.0, alphas=None, n_alphas=100, eps=1e-3, max_iter=1000, tol=1e-4,
                         positive=False, coef_init=None, fit_intercept=True):
    """The whole path as b2_solve_enet_path returns it: alphas, coefs (n_alphas, d), intercepts, gaps (/ n), n_iter and
    tol (tol y_norm2 / n).  Alphas are solved in the order given."""
    Q, q, y_norm2, m, ybar, n, live = gram_inputs(S, fit_intercept)
    d = q.size
    al = alpha_grid(q, n, l1_ratio, eps, n_alphas, positive) if alphas is None else np.asarray(alphas, np.float64)
    w = np.zeros(d) if coef_init is None else np.where(live, np.asarray(coef_init, np.float64), 0.0)
    coefs, gaps, iters = np.empty((al.size, d)), np.empty(al.size), np.empty(al.size, dtype=np.int64)
    for i, alpha in enumerate(al):
        l1, l2 = alpha * l1_ratio * n, alpha * (1.0 - l1_ratio) * n
        w, gap, tol_abs, it = cd_gram(w, l1, l2, Q, q, y_norm2, max_iter, tol, positive)
        coefs[i], gaps[i], iters[i] = w, gap / n, it
    return {"alphas": al, "coefs": coefs, "intercepts": ybar - coefs @ m, "gaps": gaps, "n_iter": iters,
            "tol": tol * y_norm2 / n, "Q": Q, "q": q, "y_norm2": y_norm2, "live": live}


def kkt_violation(S, w, alpha, l1_ratio, positive=False, fit_intercept=True):
    """max_j of the violation of the elastic-net optimality conditions at w, in longdouble from S, relative to the scale
    max|q|:  g = q - Q w - l2 w;  w_j != 0: g_j = l1 sign(w_j);  w_j == 0: |g_j| <= l1 (g_j <= l1 with positive)."""
    LD = np.longdouble
    S = np.asarray(S, dtype=np.float64).astype(LD)
    d = S.shape[0] - 2
    n = S[d, d]
    m = S[:d, d] / n if fit_intercept else np.zeros(d, dtype=LD)
    ybar = S[d, d + 1] / n if fit_intercept else LD(0)
    Q = S[:d, :d] - n * np.outer(m, m)
    q = S[:d, d + 1] - n * m * ybar
    _, _, _, _, _, _, live = gram_inputs(np.asarray(S, dtype=np.float64), fit_intercept)
    wl = np.asarray(w, dtype=np.float64).astype(LD)
    l1, l2 = LD(alpha) * LD(l1_ratio) * n, LD(alpha) * (1 - LD(l1_ratio)) * n
    g = q - Q @ wl - l2 * wl
    viol = np.where(wl != 0, np.abs(g - l1 * np.sign(wl)),
                    np.maximum(g - l1, 0) if positive else np.maximum(np.abs(g) - l1, 0))
    viol = np.where(live, viol, 0)
    scale = max(float(np.max(np.abs(q[live]))) if live.any() else 1.0, 1e-300)
    return float(np.max(viol)) / scale if d else 0.0
