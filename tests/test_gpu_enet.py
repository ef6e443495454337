"""ElasticNet / Lasso on the H100: b2_solve_enet_path (solve_enet_kernel) against the numpy oracle (tests/enet_oracle.py)
and scikit-learn's Gram coordinate descent, the estimators and the path functions.

Tolerances (asserted; the worst case measured on one H100 80GB HBM3 is printed by each test with -s):
  * designed statistics at every D in 1..128 (5 alphas, tol 1e-8, l1_ratio 1 / 0.5 / 0.2, some positive): both
    solutions lie within sqrt(2 gap / (lambda_min + l2_reg)) of the optimum, so |w_gpu - w_oracle|_2 <=
    2 sqrt(2 tol_abs / (lambda_min + l2_reg)) (worst 1.4e-9 of it: the trajectories agree to rounding); the KKT
    conditions, in longdouble from S, within 2 sqrt(2 tol_abs (lambda_max + l2_reg)) (worst 6.4e-7 of it); every
    gap <= tol_out; n_iter equal to the oracle's, allowing a one-sweep difference in at most 1 % of the alphas where a
    check sits on the threshold (measured: 0 of 640 differ).
  * every Gram path against sklearn on the same rounded rows, l1_ratio 0.5, 8 alphas, tol 1e-4: max |coef - sk| over
    max |sk| within PATH_TOL, 5x the worst of the offset and correlated tables (tensor core 6.9e-7 .. 1.2e-5, narrow
    3.4e-9 .. 1.0e-7, SIMT 2.5e-7): the tensor-core S error (~1e-6 kappa) moves the optimum.  tol = 1e-10 runs on
    the exact SIMT path only (1e-10, measured 3.8e-14): the gap tolerance is tol ||yc||^2, and ||yc||^2 from a
    tensor-core S is itself only ~1e-6 relative, so a 1e-10 gap is not resolvable there.
  * masked rows holding NaN / Inf (narrow path), device and host: 1e-7 (1.6e-8); bf16 rows: 5e-7 (7.1e-8); the
    estimators against ElasticNet / Lasso(precompute=True): 1e-6 (2.1e-8); host rows against device rows (SIMT, one
    staging block): bit-identical.
Measured on one H100 80GB HBM3 at a 400 W power limit.
"""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import ElasticNet, Lasso, enet_path

import bodywork_mlops_demo_b200 as b2
from enet_oracle import enet_path_from_stats, gram_inputs, kkt_violation
from solve_oracle import designed_statistic
from test_gpu_columns import PATHS, _table

pytestmark = pytest.mark.gpu

SIMT = b2.KERNEL_SIMT


def _stat(X, y):
    A = np.column_stack([np.asarray(X, np.float64), np.ones(X.shape[0]), np.asarray(y, np.float64)])
    return A.T @ A


def _path_on_device(ctx, up, y, kind, kernel=b2.KERNEL_AUTO, mask=None, **kw):
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    md = ctx.to_device(mask) if mask is not None else None
    ctx.set_kernel(kernel)
    try:
        ctx.gram_reset(up.shape[1])
        ctx.gram_accumulate(Xd, yd, md, 1)
        return ctx.solve_enet_path(**kw)
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        for a in (Xd, yd, md):
            if a is not None:
                a.free()


def _sk_path(X, y, l1_ratio, alphas, tol=1e-4, fit_intercept=True, max_iter=1000):
    """sklearn's Gram path on the exactly centred rows (float64)."""
    X = np.asarray(X, np.float64)
    y = np.asarray(y, np.float64)
    if fit_intercept:
        X, y = X - X.mean(0), y - y.mean()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return enet_path(np.asfortranarray(X), y, l1_ratio=l1_ratio, alphas=alphas, precompute=X.T @ X, Xy=X.T @ y,
                         tol=tol, max_iter=max_iter, return_n_iter=True)


@pytest.mark.parametrize("dims", [(1, 65), (65, 129)])
def test_kernel_against_oracle_at_every_d(ctx, dims):
    worst_w = worst_kkt = 0.0
    mism, total = [], 0
    for d in range(*dims):
        eigs = np.geomspace(2.0, 0.05, d)
        S = designed_statistic(d, eigs, n=1024, means=np.linspace(-1, 3, d), ybar=0.5, seed=d)[0]
        l1_ratio = (1.0, 0.5, 0.2)[d % 3]
        kw = dict(l1_ratio=l1_ratio, n_alphas=5, eps=1e-2, tol=1e-8, positive=(d % 4 == 1))
        ctx.gram_import(S)
        g = ctx.solve_enet_path(**kw)
        o = enet_path_from_stats(S, **kw)
        np.testing.assert_allclose(g["alphas"], o["alphas"], rtol=1e-14)
        assert g["tol"] == pytest.approx(o["tol"], rel=1e-14)
        lam = np.linalg.eigvalsh(o["Q"])
        tol_abs = o["tol"] * 1024
        for i, a in enumerate(o["alphas"]):
            total += 1
            l2 = a * (1 - l1_ratio) * 1024
            bw = 2 * np.sqrt(2 * tol_abs / (lam[0] + l2))
            ew = float(np.linalg.norm(g["coefs"][i] - o["coefs"][i]))
            bk = 2 * np.sqrt(2 * tol_abs * (lam[-1] + l2))
            ek = kkt_violation(S, g["coefs"][i], a, l1_ratio, positive=kw["positive"]) * float(np.max(np.abs(o["q"])))
            assert ew <= bw, f"D = {d}, alpha {i}: |dw| {ew:.3e} > {bw:.3e}"
            assert ek <= bk, f"D = {d}, alpha {i}: KKT {ek:.3e} > {bk:.3e}"
            assert g["gaps"][i] <= g["tol"], f"D = {d}, alpha {i}: gap {g['gaps'][i]:.3e} > {g['tol']:.3e}"
            worst_w, worst_kkt = max(worst_w, ew / bw), max(worst_kkt, ek / bk)
            if g["n_iter"][i] != o["n_iter"][i]:
                mism.append((d, i, int(g["n_iter"][i]), int(o["n_iter"][i])))
        np.testing.assert_allclose(g["intercepts"], o["intercepts"], rtol=1e-9, atol=1e-9)
    print(f"\nD in {dims}: |dw| worst {worst_w:.3g} of its bound, KKT worst {worst_kkt:.3g}, n_iter differs in "
          f"{len(mism)} / {total}: {mism[:10]}")
    assert all(abs(a - b) <= 1 for _, _, a, b in mism) and len(mism) <= 0.01 * total


# path -> bound on max |coef - coef_sklearn| / max |coef_sklearn|, 5x the worst of the offset and correlated tables
PATH_TOL = {"f32-d128": 3.2e-5, "f32-d72": 3e-5, "f32-d100": 3.2e-5, "packed-d24": 3.2e-5, "packed-d32": 2.4e-5,
            "packed-d48": 3e-5, "rawb-d128": 3.5e-6, "bf16-d96": 6.2e-5, "tc-d8": 3.6e-5, "narrow-d1": 4e-8,
            "narrow-d4": 1.8e-7, "narrow-d16": 2e-7, "narrow-bf16-d1": 1.7e-8, "narrow-bf16-d4": 1e-7,
            "narrow-bf16-d16": 5.2e-7, "simt-d8": 1.2e-6}


@pytest.mark.parametrize("family", ["offset", "correlated"])
@pytest.mark.parametrize("path", list(PATHS))
def test_every_gram_path(ctx, path, family):
    d, kind, kernel = PATHS[path]
    Xr, up, y = _table(20_000, d, family, kind, seed=d + 7)
    g = _path_on_device(ctx, up, y, kind, kernel, l1_ratio=0.5, n_alphas=8, eps=1e-2)
    alphas, coefs, gaps, iters = _sk_path(Xr, y, 0.5, g["alphas"])
    np.testing.assert_allclose(g["alphas"], alphas, rtol=1e-5)
    e = float(np.max(np.abs(g["coefs"].T - coefs))) / max(float(np.max(np.abs(coefs))), 1e-300)
    print(f"\n{path} {family}: coef {e:.3e}, n_iter {list(g['n_iter'])} vs {list(iters)}")
    assert e <= PATH_TOL[path], f"{path} {family}: {e:.3e}"
    assert np.all(g["gaps"] <= g["tol"])


def test_tight_tolerance_on_the_exact_path(ctx):
    for d in (1, 8, 40, 128):
        Xr, up, y = _table(30_000, d, "correlated", "f32", seed=d)
        for l1_ratio in (1.0, 0.5):
            g = _path_on_device(ctx, up, y, "f32", SIMT, l1_ratio=l1_ratio, n_alphas=6, eps=1e-2, tol=1e-10)
            alphas, coefs, gaps, iters = _sk_path(Xr, y, l1_ratio, g["alphas"], tol=1e-10)
            e = float(np.max(np.abs(g["coefs"].T - coefs))) / float(np.max(np.abs(coefs)))
            print(f"\nSIMT D = {d}, l1_ratio {l1_ratio}, tol 1e-10: coef {e:.3e}, n_iter {list(g['n_iter'])} vs "
                  f"{list(iters)}")
            assert e <= 1e-10


def test_rows_masks_and_layouts(ctx):
    n, d = 9000, 12
    Xr, up, y = _table(n, d, "correlated", "f32", seed=3)
    mask = (np.random.RandomState(2).uniform(size=n) < 0.7).astype(np.uint8)
    bad = up.copy(); yb = y.copy()
    bad[mask == 0, 0] = np.nan; bad[mask == 0, 1] = np.inf; yb[mask == 0] = np.nan
    kw = dict(l1_ratio=0.7, n_alphas=6, eps=1e-2)
    dev = _path_on_device(ctx, bad, yb, "f32", mask=mask, **kw)
    ctx.gram_reset(d); ctx.gram_accumulate(bad, yb, mask, 1)
    host = ctx.solve_enet_path(**kw)
    keep = mask == 1
    alphas, coefs, _, _ = _sk_path(Xr[keep], y[keep], 0.7, dev["alphas"])
    for res in (dev, host):
        assert np.all(np.isfinite(res["coefs"]))
        e = float(np.max(np.abs(res["coefs"].T - coefs))) / float(np.max(np.abs(coefs)))
        print(f"\nmasked NaN / Inf rows: coef {e:.3e}")
        assert e <= 1e-7
    # host rows against device rows on the exact path: one staging block, identical statistic and path
    ctx.set_kernel(SIMT)
    try:
        ctx.gram_reset(d); ctx.gram_accumulate(up, y)
        h = ctx.solve_enet_path(**kw)
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
    dv = _path_on_device(ctx, up, y, "f32", SIMT, **kw)
    for k in ("alphas", "coefs", "intercepts", "gaps", "n_iter"):
        assert np.array_equal(h[k], dv[k]), k
    # bf16 rows: against sklearn on the bf16-rounded rows
    Xb, ub, yb16 = _table(20_000, 16, "correlated", "bf16", seed=5)
    g = _path_on_device(ctx, ub, yb16, "bf16", **kw)
    alphas, coefs, _, _ = _sk_path(Xb, yb16, 0.7, g["alphas"])
    e = float(np.max(np.abs(g["coefs"].T - coefs))) / float(np.max(np.abs(coefs)))
    print(f"\nbf16 rows: coef {e:.3e}")
    assert e <= 5e-7


@pytest.mark.parametrize("path", list(PATHS))
def test_constant_column_gets_zero_on_every_path(ctx, path):
    d, kind, kernel = PATHS[path]
    Xr, up, y = _table(20_000, d, "offset", kind, seed=d + 11)
    j = d // 2
    up = up.copy()
    up[:, j] = up[0, j]
    g = _path_on_device(ctx, up, y, kind, kernel, l1_ratio=0.5, n_alphas=5, eps=1e-2)
    assert np.all(g["coefs"][:, j] == 0.0), path
    assert np.all(np.isfinite(g["coefs"])) and np.all(g["gaps"] <= g["tol"])


def test_errors(ctx):
    X = np.random.RandomState(1).standard_normal((300, 4)).astype(np.float32)
    y = X @ np.ones(4, np.float32)
    with pytest.raises(ValueError, match="0 sample"):
        b2.B200ElasticNet(ctx=ctx).fit(X, y, row_mask=np.zeros(300, np.uint8))
    with pytest.raises(ValueError, match="0 sample"):
        b2.lasso_path(X, y, row_mask=np.zeros(300, np.uint8), ctx=ctx)
    ctx.gram_reset(4); ctx.gram_accumulate(X, y)
    for kw in (dict(l1_ratio=1.5), dict(l1_ratio=-0.1), dict(l1_ratio=0.0), dict(alphas=[1.0, -1.0]),
               dict(alphas=[np.nan]), dict(alphas=[np.inf]), dict(max_iter=0), dict(tol=-1.0), dict(n_alphas=0),
               dict(eps=0.0)):
        with pytest.raises(ValueError):
            ctx.solve_enet_path(**kw)
    ctx.solve_enet_path(l1_ratio=0.0, alphas=[1.0])          # a given grid is fine at l1_ratio 0 (ridge)
    with pytest.raises(ValueError, match="selection"):
        b2.B200Lasso(selection="random", ctx=ctx).fit(X, y)


def test_repeatable_and_one_launch(ctx):
    Xr, up, y = _table(200_000, 64, "correlated", "f32", seed=31)
    Xd, yd = ctx.to_device(up), ctx.to_device(y)
    try:
        ctx.gram_reset(64); ctx.gram_accumulate(Xd, yd)
        n0 = ctx.launch_count()
        r1 = ctx.solve_enet_path(l1_ratio=0.5)
        assert ctx.launch_count() - n0 == 1
        r2 = ctx.solve_enet_path(l1_ratio=0.5)
        for k in ("alphas", "coefs", "intercepts", "gaps", "n_iter"):
            assert np.array_equal(r1[k], r2[k]), k
        assert r1["tol"] == r2["tol"] and int(np.sum(r1["n_iter"])) > 100
    finally:
        Xd.free(); yd.free()


def test_estimators_against_sklearn(ctx, tmp_path):
    import joblib
    Xr, up, y = _table(6000, 10, "correlated", "f32", seed=41)
    for cls, sk_cls, kw in ((b2.B200Lasso, Lasso, {}), (b2.B200ElasticNet, ElasticNet, {"l1_ratio": 0.3})):
        for rows in ("f32", "f64", "device"):
            Xin, yin = (up.astype(np.float64) if rows == "f64" else up), y
            if rows == "device":
                Xin, yin = ctx.to_device(up), ctx.to_device(y)
            est = cls(alpha=0.05, ctx=ctx, **kw).fit(Xin, yin)
            sk = sk_cls(alpha=0.05, precompute=True, **kw).fit(Xr, y.astype(np.float64))
            e = float(np.max(np.abs(est.coef_ - sk.coef_))) / float(np.max(np.abs(sk.coef_)))
            print(f"\n{cls.__name__} {rows}: coef {e:.3e}, n_iter {est.n_iter_} vs {sk.n_iter_}")
            assert e <= 1e-6 and est.n_features_in_ == 10
            assert est.intercept_ == pytest.approx(sk.intercept_, rel=1e-4, abs=1e-4)
            assert est.dual_gap_ <= est.tol * np.var(y.astype(np.float64)) * 1.01
            if rows == "device":
                np.testing.assert_allclose(est.predict(Xin).to_host(), sk.predict(Xr), rtol=1e-4, atol=1e-3)
                Xin.free(); yin.free()
        path = tmp_path / "enet.joblib"
        joblib.dump(est.to_sklearn(), path)
        reg = joblib.load(path)
        assert type(reg) is sk_cls and reg.n_iter_ == est.n_iter_
        np.testing.assert_allclose(reg.predict(Xr[:200]), est.predict(up[:200]), rtol=1e-5, atol=1e-3)
    # ConvergenceWarning with sklearn's wording
    with pytest.warns(ConvergenceWarning, match="Objective did not converge"):
        est = b2.B200ElasticNet(alpha=1e-4, max_iter=2, tol=1e-12, ctx=ctx).fit(up, y)
    assert est.n_iter_ == 2
    # warm start: the second fit starts from coef_, as sklearn's
    est = b2.B200ElasticNet(alpha=0.1, warm_start=True, ctx=ctx).fit(up, y)
    sk = ElasticNet(alpha=0.1, warm_start=True, precompute=True).fit(Xr, y.astype(np.float64))
    est.alpha = sk.alpha = 0.02
    est.fit(up, y)
    sk.fit(Xr, y.astype(np.float64))
    e = float(np.max(np.abs(est.coef_ - sk.coef_))) / float(np.max(np.abs(sk.coef_)))
    cold = b2.B200ElasticNet(alpha=0.02, ctx=ctx).fit(up, y)
    print(f"\nwarm start: coef {e:.3e}, n_iter {est.n_iter_} vs {sk.n_iter_} (cold {cold.n_iter_})")
    assert e <= 1e-6 and est.n_iter_ <= cold.n_iter_


def test_path_functions(ctx):
    Xr, up, y = _table(8000, 20, "correlated", "f32", seed=51)
    ctx.set_kernel(SIMT)
    try:
        al, coefs, gaps, iters = b2.lasso_path(up, y, alphas=30, return_n_iter=True, ctx=ctx)
        ska, skc, skg, ski = enet_path(Xr, y.astype(np.float64), l1_ratio=1.0, alphas=30, precompute=Xr.T @ Xr,
                                       Xy=Xr.T @ y.astype(np.float64), return_n_iter=True)
        assert coefs.shape == (20, 30) and len(iters) == 30
        np.testing.assert_allclose(al, ska, rtol=1e-12)
        e = float(np.max(np.abs(coefs - skc))) / float(np.max(np.abs(skc)))
        print(f"\nlasso_path, no intercept: coef {e:.3e}")
        assert e <= 1e-6
        user = [0.001, 0.1, 0.01]
        al2, c2, g2, b0 = b2.enet_path(up, y, l1_ratio=0.5, alphas=user, fit_intercept=True, ctx=ctx)
        assert list(al2) == sorted(user, reverse=True) and c2.shape == (20, 3) and b0.shape == (3,)
        sk = ElasticNet(alpha=0.01, l1_ratio=0.5, precompute=True, tol=1e-4).fit(Xr, y.astype(np.float64))
        assert float(np.max(np.abs(c2[:, 1] - sk.coef_))) <= 1e-3 * float(np.max(np.abs(sk.coef_)))
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
