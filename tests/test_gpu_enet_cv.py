"""LassoCV / ElasticNetCV on the H100: b2_gram_folds and b2_solve_enet_cv against the numpy oracle
(tests/enet_cv_oracle.py) and scikit-learn's LassoCV / ElasticNetCV(precompute=True), and the estimators.

Tolerances (asserted; the worst case measured on one H100 80GB HBM3 is printed by each test with -s):
  * designed fold statistics at every D in 1..128 (3 folds, 5 alphas, tol 1e-8, one or two l1_ratios): coefficients of
    every fold path within the tol-derived bound of test_gpu_enet.py, 2 sqrt(2 tol_abs / (lambda_min + l2_reg)) with
    lambda_min of T_k's centred Gram; n_iter equal to the oracle's in at least 99 % of the alphas, off by at most 1;
    mse within 1e-12 relative of the oracle; the grid bit-identical to b2_solve_enet_path on the summed statistic.
    Measured: |dw| at most 2.5e-9 of its bound, mse 1.3e-13, n_iter differs in 0 of 2 565 alphas.
  * b2_gram_folds on every Gram path (5 contiguous folds of 4 001 / 4 000 rows, and shuffled folds): each fold's S against
    fp64 numpy by oracle.stat_error within test_gpu_columns.TOL of its kernel; the summed S bit-equal to the fold sum
    in fold order; at D = 128 one tensor-core launch per fold.
  * the estimators against sklearn on the offset and correlated tables of every path (20 alphas, 5 folds): mse_path_
    within MSE_TOL (relative, 5x the worst measured over both tables: tensor core 3.1e-5 .. 6.4e-4, narrow
    3.2e-8 .. 1.2e-6, SIMT 5.1e-7), alpha_ equal (it was on every path) or sklearn's own mean mse at our alpha within
    MSE_TOL of its minimum, coef_ within test_gpu_enet.PATH_TOL of sklearn's fit at our alpha_ (worst 8.3e-6).
  * masked NaN / Inf rows, device and host: mse_path_ 1e-6 (4.6e-8); bf16 rows on the tensor core: 7e-4 (1.3e-4); host
    rows against device rows on the SIMT kernel: bit-identical.
  * b2_gram_folds: stat error 3.2e-6 (tensor core, bound 2e-5), 4.3e-7 (narrow, SIMT); 5 timed launches at D = 128.
Measured on one H100 80GB HBM3 at a 700 W power limit.
"""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import ElasticNet, ElasticNetCV, LassoCV
from sklearn.model_selection import KFold

import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc
from enet_cv_oracle import enet_cv_from_stats, fold_stats, fold_sum
from enet_oracle import gram_inputs
from solve_oracle import designed_statistic
from test_gpu_columns import PATHS, TOL, _table
from test_gpu_enet import PATH_TOL

pytestmark = pytest.mark.gpu

SIMT = b2.KERNEL_SIMT
TC = b2.KERNEL_TCGEN05

# path -> bound on max |mse_path_ - sklearn| / sklearn, 5x the worst of the offset and correlated tables.  The held-out
# error comes from the fold's statistic, so it carries the statistic's error times (sum_j |w_j| sigma_j)^2 / mse: large
# on the tensor-core paths, whose S is ~3e-6 (scale-free), and on tables that y fits closely.
MSE_TOL = {"f32-d128": 3.2e-3, "f32-d72": 1.8e-3, "f32-d100": 2.4e-3, "packed-d24": 6.5e-4, "packed-d32": 1.1e-3,
           "packed-d48": 1.3e-3, "rawb-d128": 1.9e-4, "bf16-d96": 2.7e-3, "tc-d8": 1.9e-4, "narrow-d1": 6.1e-7,
           "narrow-d4": 6e-7, "narrow-d16": 3.2e-6, "narrow-bf16-d1": 3.1e-7, "narrow-bf16-d4": 8e-7,
           "narrow-bf16-d16": 6e-6, "simt-d8": 2.6e-6}


def _sk(cls, X, y, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return cls(precompute=True, **kw).fit(np.asarray(X, np.float64), np.asarray(y, np.float64))


def _designed_folds(d, K, seed):
    eigs = np.geomspace(2.0, 0.05, d)
    return np.stack([designed_statistic(d, eigs, n=1024 + 256 * k, means=np.linspace(-1, 3, d), ybar=0.5,
                                        seed=seed + 101 * k)[0] for k in range(K)])


@pytest.mark.parametrize("dims", [(1, 65), (65, 129)])
def test_kernel_against_oracle_at_every_d(ctx, dims):
    worst_w = worst_mse = 0.0
    mism, total = [], 0
    K = 3
    for d in range(*dims):
        fs = _designed_folds(d, K, d)
        l1 = [(1.0,), (0.5, 1.0), (0.2,)][d % 3]
        kw = dict(n_alphas=5, eps=1e-2, tol=1e-8, positive=(d % 4 == 1))
        g = ctx.solve_enet_cv(K, l1, fold_S=fs, want_coefs=True, **kw)
        o = enet_cv_from_stats(fs, l1, **kw)
        # the grid: bit-identical to b2_solve_enet_path on the summed statistic (which the call left resident)
        assert np.array_equal(ctx.gram_export(), fold_sum(fs))
        for li, r in enumerate(l1):
            p = ctx.solve_enet_path(l1_ratio=r, n_alphas=5, eps=1e-2, tol=1e-8, positive=kw["positive"])
            assert np.array_equal(g["alphas"][li], p["alphas"]), (d, r)
        rel = np.abs(g["mse"] - o["mse"]) / np.abs(o["mse"])
        worst_mse = max(worst_mse, float(np.max(rel)))
        assert float(np.max(rel)) <= 1e-12, (d, float(np.max(rel)))
        for k in range(K):
            Q, _, y_norm2, _, _, n, _ = gram_inputs(fold_sum(fs, k))
            lam0 = float(np.linalg.eigvalsh(Q)[0])
            tol_abs = 1e-8 * y_norm2
            for li, r in enumerate(l1):
                for i, a in enumerate(o["alphas"][li]):
                    total += 1
                    bw = 2 * np.sqrt(2 * tol_abs / (lam0 + a * (1 - r) * n))
                    ew = float(np.linalg.norm(g["coefs"][li, k, i] - o["coefs"][li, k, i]))
                    assert ew <= bw, f"D = {d}, fold {k}, l1 {r}, alpha {i}: |dw| {ew:.3e} > {bw:.3e}"
                    worst_w = max(worst_w, ew / bw)
                    if g["n_iter"][li, k, i] != o["n_iter"][li, k, i]:
                        mism.append((d, k, i, int(g["n_iter"][li, k, i]), int(o["n_iter"][li, k, i])))
    print(f"\nD in {dims}: |dw| worst {worst_w:.3g} of its bound, mse worst {worst_mse:.3g}, n_iter differs in "
          f"{len(mism)} / {total}: {mism[:10]}")
    assert all(abs(a - b) <= 1 for *_, a, b in mism) and len(mism) <= 0.01 * total


def _stat_err(S, So):
    return orc.stat_error(S, So)


@pytest.mark.parametrize("path", list(PATHS))
def test_gram_folds_every_path(ctx, path):
    d, kind, kernel = PATHS[path]
    n, K = 20_003, 5
    Xr, up, y = _table(n, d, "offset", kind, seed=d + 3)
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    ctx.set_kernel(kernel)
    try:
        for cv in (K, KFold(K, shuffle=True, random_state=d)):
            ids, _ = b2.fold_ids(n, cv=cv)
            idd = ctx.to_device(ids)
            ctx.last_kernel_ms()
            fs = ctx.gram_folds(Xd, yd, idd, K)
            _, launches = ctx.last_kernel_ms()
            idd.free()
            So = fold_stats(Xr, y, ids, K)
            worst = (0.0, 0.0)
            for k in range(K):
                stat, mean = _stat_err(fs[k], So[k])
                worst = (max(worst[0], stat), max(worst[1], mean))
                assert stat < TOL[kernel][0] and mean < TOL[kernel][1], (path, k, stat, mean)
                assert fs[k][d, d] == So[k][d, d]
            assert np.array_equal(ctx.gram_export(), fold_sum(fs))
            print(f"\n{path} {'contiguous' if cv == K else 'shuffled'}: stat {worst[0]:.2e}, mean {worst[1]:.2e}, "
                  f"{launches} timed launches")
            if d == 128 and cv == K:
                assert launches == K, launches
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        Xd.free(); yd.free()


@pytest.mark.parametrize("family", ["offset", "correlated"])
@pytest.mark.parametrize("path", list(PATHS))
def test_estimators_on_every_gram_path(ctx, path, family):
    d, kind, kernel = PATHS[path]
    Xr, up, y = _table(20_000, d, family, kind, seed=d + 17)
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    ctx.set_kernel(kernel)
    try:
        est = b2.B200LassoCV(alphas=20, cv=5, ctx=ctx).fit(Xd, yd)
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        Xd.free(); yd.free()
    sk = _sk(LassoCV, Xr, y, alphas=20, cv=5)
    e_mse = float(np.max(np.abs(est.mse_path_ - sk.mse_path_) / sk.mse_path_))
    np.testing.assert_allclose(est.alphas_, sk.alphas_, rtol=1e-5)
    i_ours = int(np.argmin(np.abs(est.alphas_ - est.alpha_)))
    mean_sk = sk.mse_path_.mean(axis=1)
    assert est.alpha_ == pytest.approx(sk.alpha_, rel=1e-5) or \
        mean_sk[i_ours] <= np.min(mean_sk) * (1 + MSE_TOL[path])
    ref = _sk(ElasticNet, Xr, y, alpha=est.alpha_, l1_ratio=1.0)
    e_coef = float(np.max(np.abs(est.coef_ - ref.coef_))) / max(float(np.max(np.abs(ref.coef_))), 1e-300)
    print(f"\n{path} {family}: mse_path_ {e_mse:.3e}, coef {e_coef:.3e}, alpha_ {est.alpha_:.6g} vs {sk.alpha_:.6g}")
    assert e_mse <= MSE_TOL[path], e_mse
    assert e_coef <= PATH_TOL[path], e_coef


def test_rows_masks_layouts_and_repeats(ctx):
    n, d = 9000, 12
    Xr, up, y = _table(n, d, "correlated", "f32", seed=3)
    mask = (np.random.RandomState(2).uniform(size=n) < 0.7).astype(np.uint8)
    bad, yb = up.copy(), y.copy()
    bad[mask == 0, 0] = np.nan; bad[mask == 0, 1] = np.inf; yb[mask == 0] = np.nan
    keep = mask == 1
    cv = KFold(4, shuffle=True, random_state=5)
    sk = _sk(ElasticNetCV, Xr[keep], y[keep], l1_ratio=[0.3, 0.9], alphas=12, cv=cv)
    Xd, yd, md = ctx.to_device(bad), ctx.to_device(yb), ctx.to_device(mask)
    try:
        for Xin, yin, min_ in ((Xd, yd, md), (bad, yb, mask)):
            est = b2.B200ElasticNetCV(l1_ratio=[0.3, 0.9], alphas=12, cv=cv, ctx=ctx).fit(Xin, yin, row_mask=min_)
            e = float(np.max(np.abs(est.mse_path_ - sk.mse_path_) / sk.mse_path_))
            print(f"\nmasked NaN / Inf rows ({'device' if Xin is Xd else 'host'}): mse_path_ {e:.3e}")
            assert e <= 1e-6 and est.l1_ratio_ == sk.l1_ratio_ and est.alpha_ == pytest.approx(sk.alpha_, rel=1e-6)
    finally:
        Xd.free(); yd.free(); md.free()
    # host rows against device rows on the exact kernel: identical statistics, identical everything
    ctx.set_kernel(SIMT)
    try:
        h = b2.B200LassoCV(alphas=15, cv=5, ctx=ctx).fit(up, y)
        Xd, yd = ctx.to_device(up), ctx.to_device(y)
        dv = b2.B200LassoCV(alphas=15, cv=5, ctx=ctx).fit(Xd, yd)
        Xd.free(); yd.free()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
    for k in ("mse_path_", "alphas_", "coef_", "intercept_", "dual_gap_", "n_iter_", "alpha_"):
        assert np.array_equal(getattr(h, k), getattr(dv, k)), k
    # bf16 rows: against sklearn on the bf16-rounded rows
    Xb, ub, yb16 = _table(20_000, 16, "correlated", "bf16", seed=5)
    ubd, ybd = ctx.to_device(ub, "bf16"), ctx.to_device(yb16)
    try:
        est = b2.B200LassoCV(alphas=12, cv=5, ctx=ctx).fit(ubd, ybd)
    finally:
        ubd.free(); ybd.free()
    sk = _sk(LassoCV, Xb, yb16, alphas=12, cv=5)
    e = float(np.max(np.abs(est.mse_path_ - sk.mse_path_) / sk.mse_path_))
    print(f"\nbf16 rows: mse_path_ {e:.3e}")
    assert e <= 7e-4                       # 4 000-row folds: below the narrow kernel's 4 096, on the tensor core
    # bit-identical repeats, and one launch for the paths whatever the number of l1_ratios
    Xr, up, y = _table(50_000, 32, "correlated", "f32", seed=31)
    ids, K = b2.fold_ids(50_000, cv=5)
    ctx.gram_folds(up, y, ids, K)
    runs = []
    for l1 in ((1.0,), (0.1, 0.5, 0.7, 0.9, 0.95, 0.99, 1.0), (1.0,)):
        n0 = ctx.launch_count()
        runs.append(ctx.solve_enet_cv(K, l1, n_alphas=30, want_coefs=True))
        assert ctx.launch_count() - n0 == 1
    for k in ("alphas", "mse", "n_iter", "gaps", "coefs"):
        assert np.array_equal(runs[0][k], runs[2][k]), k
        assert np.array_equal(runs[0][k][0], runs[1][k][-1]), k      # l1_ratio 1 is the same path in both calls


def test_errors(ctx):
    X = np.random.RandomState(1).standard_normal((300, 4)).astype(np.float32)
    y = X @ np.ones(4, np.float32)
    ids, K = b2.fold_ids(300, cv=3)
    for n_folds in (1, 255):
        with pytest.raises(ValueError, match="n_folds"):
            ctx.gram_folds(X, y, ids, n_folds)
    empty = ids.copy(); empty[empty == 1] = 255
    with pytest.raises(ValueError, match="fold 1 has no rows"):
        ctx.gram_folds(X, y, empty, 3)
    ctx.gram_reset(4)
    with pytest.raises(RuntimeError, match="b2_gram_folds first"):
        ctx.solve_enet_cv(3)
    ctx.gram_folds(X, y, ids, K)
    for kw in (dict(l1_ratios=[1.5]), dict(l1_ratios=[0.5, -0.1]), dict(l1_ratios=[0.0]), dict(l1_ratios=[]),
               dict(alphas=[1.0, -1.0]), dict(alphas=[np.nan]), dict(max_iter=0), dict(tol=-1.0), dict(n_alphas=0),
               dict(eps=0.0)):
        with pytest.raises(ValueError):
            ctx.solve_enet_cv(K, **kw)
    with pytest.raises(ValueError, match="n_folds"):
        ctx.solve_enet_cv(1)
    fs = ctx.gram_folds(X, y, ids, K)
    fs[2] = 0.0
    with pytest.raises(ValueError, match="fold 2 has no rows"):
        ctx.solve_enet_cv(K, fold_S=fs)
    ctx.solve_enet_cv(K, l1_ratios=[0.0], alphas=[1.0])       # a given grid is fine at l1_ratio 0
    with pytest.raises(ValueError, match="selection"):
        b2.B200LassoCV(selection="random", ctx=ctx).fit(X, y)
    with pytest.raises(ValueError, match="l1_ratio=0"):
        b2.B200ElasticNetCV(l1_ratio=[0.0, 0.5], ctx=ctx).fit(X, y)
    with pytest.raises(ValueError, match="Cannot have number of splits"):
        b2.B200LassoCV(ctx=ctx).fit(X, y, row_mask=np.zeros(300, np.uint8))


def test_joblib_round_trip_predict_and_warnings(ctx, tmp_path):
    import joblib
    Xr, up, y = _table(6000, 10, "correlated", "f32", seed=41)
    for cls, sk_cls, kw in ((b2.B200LassoCV, LassoCV, {}), (b2.B200ElasticNetCV, ElasticNetCV, {"l1_ratio": [0.3, 1.0]})):
        est = cls(cv=4, ctx=ctx, **kw).fit(up, y)
        sk = _sk(sk_cls, Xr, y, cv=4, **kw)
        assert est.mse_path_.shape == sk.mse_path_.shape and est.alphas_.shape == sk.alphas_.shape
        assert hasattr(est, "l1_ratio_") == hasattr(sk, "l1_ratio_") and est.n_features_in_ == 10
        path = tmp_path / "cv.joblib"
        joblib.dump(est.to_sklearn(), path)
        reg = joblib.load(path)
        assert type(reg) is sk_cls and reg.alpha_ == est.alpha_ and reg.n_iter_ == est.n_iter_
        np.testing.assert_allclose(reg.predict(Xr[:200]), est.predict(up[:200]), rtol=1e-5, atol=1e-3)
    with pytest.warns(ConvergenceWarning, match="Objective did not converge"):
        b2.B200LassoCV(alphas=[1e-4], max_iter=2, tol=1e-12, cv=3, ctx=ctx).fit(up, y)
