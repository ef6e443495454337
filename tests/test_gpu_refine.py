"""The refined fit (b2_fit_refined, DESIGN.md section 2): b2_fit, then residual passes over the same rows that take any
Gram path to the fp64 least-squares solution of the stored rows.

Every comparison is against scikit-learn (or lstsq / Ridge) fitted on the float64 values of the rows as stored (fp32, or
bf16-rounded), scaled as in test_gpu_columns.py: coef error = max_j |coef_j - coef_sk_j| * sigma_j.

Tolerances (largest value measured on one H100 80GB HBM3 at a 400 W power limit -> asserted):
  correlated columns, rho up to 0.999 (kappa 8.5e3), 4 passes:  4.4e-13 -> 1e-10; unrefined tensor core 7.2e-3
  offset columns, every path, 3 passes:                          1.2e-13 -> 1e-6 (the SIMT tolerance of test_gpu_columns)
  single bf16 operand, 2 M rows, 4 passes:                       2.9e-14 -> 1e-6 (unrefined 7.4e-5)
  estimator, refine=2, rho = 0.999 at D = 64:                    3.5e-8 -> 1e-6 (unrefined 5.6e-3)
"""
import ctypes as C
import warnings

import numpy as np
import pytest
from sklearn.linear_model import LinearRegression, Ridge

import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc
from test_gpu_columns import PATHS, _table

pytestmark = pytest.mark.gpu

TC, NARROW, SIMT = b2.KERNEL_TCGEN05, b2.KERNEL_NARROW, b2.KERNEL_SIMT
E_ARG, E_SINGULAR, E_UNSUPPORTED = -1, -4, -6
REFINED_TOL = 1e-10             # refined fit on correlated columns
SIMT_TOL = 1e-6                 # the exact kernel's coefficient tolerance (test_gpu_columns.TOL[SIMT])


def _sk(Xr, y, mask=None, keep=1, **kw):
    sel = slice(None) if mask is None else (mask == keep)
    return LinearRegression(**kw).fit(Xr[sel], np.asarray(y, dtype=np.float64)[sel])


def _err(coef, ref_coef, Xr, mask=None, keep=1):
    sel = slice(None) if mask is None else (mask == keep)
    So = orc.gram_stats(Xr[sel], np.zeros(Xr[sel].shape[0]))
    return orc.coef_error(coef, ref_coef, So)


def _refined(ctx, up, y, kind, kernel, mask=None, keep=1, **kw):
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    md = ctx.to_device(mask) if mask is not None else None
    ctx.set_kernel(kernel)
    try:
        return ctx.fit_refined(Xd, yd, md, keep, **kw)
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        for a in (Xd, yd, md):
            if a is not None:
                a.free()


def _raw_refined(ctx, X_ptr, x_dtype, y_ptr, n, d, ldx, mask_ptr=None, keep=1, alpha=0.0, fit_intercept=1,
                 max_passes=3, tol=1e-10, mem_kind=b2.native.MEM_DEVICE):
    coef = np.empty(d, dtype=np.float64)
    b0, step, passes = C.c_double(0.0), C.c_double(0.0), C.c_int(0)
    rc = b2.native.load().b2_fit_refined(ctx._h, X_ptr, x_dtype, y_ptr, n, d, ldx, mem_kind, mask_ptr, keep, alpha,
                                         fit_intercept, max_passes, tol, coef.ctypes.data, C.byref(b0), C.byref(passes),
                                         C.byref(step))
    return rc, coef, b0.value, passes.value, step.value


@pytest.mark.parametrize("path", list(PATHS))
def test_no_passes_is_bit_identical_to_b2_fit(ctx, path):
    d, kind, kernel = PATHS[path]
    _, up, y = _table(30_011, d, "offset", kind, seed=500 + d)
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    ctx.set_kernel(kernel)
    try:
        c0, b0 = ctx.fit(Xd, yd)
        S0 = ctx.gram_export()
        c1, b1, passes, step = ctx.fit_refined(Xd, yd, max_passes=0)
        S1 = ctx.gram_export()
        c2, b2_, _, _ = ctx.fit_refined(Xd, yd, max_passes=2)
        S2 = ctx.gram_export()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        Xd.free(); yd.free()
    assert np.array_equal(c0, c1) and b0 == b1 and passes == 0 and step == 0.0
    assert np.array_equal(S0, S1) and np.array_equal(S0, S2)          # the passes leave b2_fit's S in place


CORR_PATHS = ["f32-d128", "rawb-d128", "packed-d32", "tc-d8", "narrow-d16"]


@pytest.mark.parametrize("path", CORR_PATHS)
def test_correlated_columns_reach_the_fp64_solution(ctx, path):
    d, kind, kernel = PATHS[path]
    for rho in (0.9, 0.99, 0.999):
        X, y, _ = orc.column_table(200_000, d, "correlated", seed=400, rho=rho)
        y = y.astype(np.float32)
        if kind == "bf16":
            up = b2.native.to_bf16_bits(X.astype(np.float32))
            Xr = b2.native.from_bf16_bits(up).astype(np.float64)
        else:
            up = X.astype(np.float32)
            Xr = up.astype(np.float64)
        sk = _sk(Xr, y)
        kappa = orc.centred_condition(orc.gram_stats(Xr, y))
        c0, _, _, _ = _refined(ctx, up, y, kind, kernel, max_passes=0)
        c, b, passes, step = _refined(ctx, up, y, kind, kernel, max_passes=4)
        e0, e = _err(c0, sk.coef_, Xr), _err(c, sk.coef_, Xr)
        print(f"[refine] {path} rho={rho} kappa={kappa:.3g} unrefined={e0:.3g} refined={e:.3g} passes={passes} "
              f"step={step:.3g}")
        if rho == 0.999 and kernel == TC:
            assert e0 > 1e-4, (kappa, e0)                             # the plain tensor-core fit breaks the contract
        assert e < REFINED_TOL, (rho, kappa, e0, e, passes, step)
        assert abs(b - sk.intercept_) < 1e-6 * max(1.0, abs(sk.intercept_)), (b, sk.intercept_)


@pytest.mark.parametrize("path", list(PATHS))
def test_offset_columns_refined_on_every_path(ctx, path):
    d, kind, kernel = PATHS[path]
    Xr, up, y = _table(100_003, d, "offset", kind, seed=d)
    sk = _sk(Xr, y)
    c, b, passes, step = _refined(ctx, up, y, kind, kernel, max_passes=3)
    e = _err(c, sk.coef_, Xr)
    print(f"[refine] offset {path} err={e:.3g} passes={passes} step={step:.3g}")
    assert e < SIMT_TOL, (e, passes, step)


@pytest.mark.parametrize("keep", [0, 1])
@pytest.mark.parametrize("path", ["f32-d128", "rawb-d128", "packed-d48", "narrow-d4", "narrow-bf16-d16", "simt-d8"])
def test_masked_rows_may_hold_nan(ctx, path, keep):
    d, kind, kernel = PATHS[path]
    n = 60_001
    Xr, up, y = _table(n, d, "correlated", kind, seed=600 + d)
    mask = (np.random.RandomState(d + keep).rand(n) < 0.6).astype(np.uint8)
    drop = np.flatnonzero(mask != keep)
    up = up.copy(); y = y.copy()
    nan_bits, inf_bits = (0x7FC0, 0x7F80) if kind == "bf16" else (np.nan, np.inf)
    up[drop[::3]] = nan_bits
    up[drop[1::3]] = inf_bits
    y[drop[::5]] = np.nan
    sk = _sk(Xr, y, mask, keep)
    c, b, passes, step = _refined(ctx, up, y, kind, kernel, mask=mask, keep=keep, max_passes=3)
    assert np.all(np.isfinite(c)) and np.isfinite(b)
    assert _err(c, sk.coef_, Xr, mask, keep) < SIMT_TOL
    assert abs(b - sk.intercept_) < 1e-6 * max(1.0, abs(sk.intercept_))


@pytest.mark.parametrize("kind", ["f32", "bf16"])
def test_strided_and_unaligned_rows_take_the_register_fed_kernel(ctx, kind):
    """ldx > d, and rows that start 4 bytes into the buffer: no TMA and no vector loads, the same solution."""
    n, d, ldx = 50_000, 24, 29
    Xr, up, y = _table(n, d, "correlated", kind, seed=77)
    sk = _sk(Xr, y)
    wide = np.zeros((n, ldx), dtype=up.dtype)
    wide[:, :d] = up
    es = up.dtype.itemsize
    xdt = b2.F32 if kind == "f32" else b2.BF16
    Xw, yd = ctx.to_device(wide, kind), ctx.to_device(y)
    try:
        rc, c, b, passes, step = _raw_refined(ctx, Xw.ptr, xdt, yd.ptr, n, d, ldx)
        assert rc == 0, b2.native.last_error()
        assert _err(c, sk.coef_, Xr) < SIMT_TOL and passes >= 1
    finally:
        Xw.free()
    flat = np.zeros(n * d + 8 // es, dtype=up.dtype)
    flat[4 // es: 4 // es + n * d] = up.ravel()
    Xu = ctx.to_device(flat, kind)
    try:
        rc, cu, bu, _, _ = _raw_refined(ctx, Xu.ptr + 4, xdt, yd.ptr, n, d, d)
        assert rc == 0, b2.native.last_error()
        assert _err(cu, sk.coef_, Xr) < SIMT_TOL
    finally:
        Xu.free(); yd.free()


def test_host_rows_equal_device_rows(ctx):
    """One staging block of contiguous rows runs the same kernels on the same rows wherever they live: pinned, pageable
    and device-resident rows give bit-identical results.  Over several blocks pinned and pageable rows still agree."""
    n, d = 200_003, 64
    Xr, up, y = _table(n, d, "correlated", "f32", seed=88)
    mask = (np.arange(n) % 7 != 0).astype(np.uint8)
    Xp, yp, mp = ctx.pinned((n, d), np.float32), ctx.pinned((n,), np.float32), ctx.pinned((n,), np.uint8)
    Xp.array[:] = up; yp.array[:] = y; mp.array[:] = mask
    try:
        r_pin = ctx.fit_refined(Xp.array, yp.array, mp.array, 1, max_passes=3)
        r_pag = ctx.fit_refined(up, y, mask, 1, max_passes=3)
        r_dev = _refined(ctx, up, y, "f32", b2.KERNEL_AUTO, mask=mask, keep=1, max_passes=3)
    finally:
        for a in (Xp, yp, mp):
            a.free()
    for r in (r_pag, r_dev):
        assert np.array_equal(r[0], r_pin[0]) and r[1:] == r_pin[1:]
    big = 2 * (1 << 18) + 999
    Xb, ub, yb = _table(big, 16, "correlated", "f32", seed=89)
    Xq, yq = ctx.pinned((big, 16), np.float32), ctx.pinned((big,), np.float32)
    Xq.array[:] = ub; yq.array[:] = yb
    try:
        a = ctx.fit_refined(Xq.array, yq.array, max_passes=2)
        b_ = ctx.fit_refined(ub, yb, max_passes=2)
    finally:
        Xq.free(); yq.free()
    assert np.array_equal(a[0], b_[0]) and a[1:] == b_[1:]
    assert _err(a[0], _sk(Xb, yb).coef_, Xb) < SIMT_TOL


def test_ridge_and_no_intercept(ctx):
    n, d = 120_000, 32
    Xr, up, y = _table(n, d, "correlated", "f32", seed=90)
    c, b, _, _ = _refined(ctx, up, y, "f32", TC, alpha=50.0, max_passes=4)
    rd = Ridge(alpha=50.0).fit(Xr, y.astype(np.float64))
    assert _err(c, rd.coef_, Xr) < REFINED_TOL and abs(b - rd.intercept_) < 1e-6
    c0, b0, _, _ = _refined(ctx, up, y, "f32", TC, fit_intercept=False, max_passes=4)
    ls = np.linalg.lstsq(Xr, y.astype(np.float64), rcond=None)[0]
    assert _err(c0, ls, Xr) < REFINED_TOL and b0 == 0.0


def test_single_operand_mode_refines_to_the_contract_and_beyond(ctx):
    n, d = 2_000_000, 128
    Xr, up, y = _table(n, d, "offset", "f32", seed=47)
    sk = _sk(Xr, y)
    ctx.set_precision(b2.PRECISION_BF16)
    try:
        c0, _, _, _ = _refined(ctx, up, y, "f32", TC, max_passes=0)
        c, b, passes, step = _refined(ctx, up, y, "f32", TC, max_passes=4)
    finally:
        ctx.set_precision(b2.PRECISION_SPLIT)
    e0, e = _err(c0, sk.coef_, Xr), _err(c, sk.coef_, Xr)
    print(f"[refine] single operand 2M: unrefined={e0:.3g} refined={e:.3g} passes={passes} step={step:.3g}")
    assert e < 1e-6, (e0, e, passes, step)


# One pass streams the rows through the kernels of b2_score's row plan: each segment of rows is one kernel plus its ordered
# reduce.  (d, kind, n, ldx, segments); a tail is the rows after the ring's whole tiles, left to the register-fed kernel.
LAUNCH_LAYOUTS = {
    "narrow-d1-tail": (1, "f32", 100_001, 1, 2),
    "narrow-d12-tail": (12, "f32", 100_001, 12, 2),
    "wide-d128": (128, "f32", 600_000, 128, 1),        # a whole number of 60-row TMA tiles: no register-fed tail
    "wide-d48-tail": (48, "f32", 100_001, 48, 2),
    "wide-d24-tail": (24, "f32", 100_001, 24, 2),
    "bf16-d100": (100, "bf16", 100_001, 100, 1),       # 200-byte rows: register-fed only
    "strided-d24": (24, "f32", 50_000, 29, 1),
}


def test_repeatable_and_launches_per_pass(ctx):
    for layout, (d, kind, n, ldx, segments) in LAUNCH_LAYOUTS.items():
        _, up, y = _table(n, d, "correlated", kind, seed=91)
        rows = np.zeros((n, ldx), dtype=up.dtype)
        rows[:, :d] = up
        xdt = b2.F32 if kind == "f32" else b2.BF16
        Xd, yd = ctx.to_device(rows, kind), ctx.to_device(y)
        try:
            r1 = _raw_refined(ctx, Xd.ptr, xdt, yd.ptr, n, d, ldx, max_passes=2, tol=0.0)
            r2 = _raw_refined(ctx, Xd.ptr, xdt, yd.ptr, n, d, ldx, max_passes=2, tol=0.0)
            assert r1[0] == 0, (layout, b2.native.last_error())
            assert np.array_equal(r1[1], r2[1]) and r1[2:] == r2[2:], layout
            l0 = ctx.launch_count()
            _raw_refined(ctx, Xd.ptr, xdt, yd.ptr, n, d, ldx, max_passes=0)
            l1 = ctx.launch_count()
            rc, coef, b0, passes, _ = _raw_refined(ctx, Xd.ptr, xdt, yd.ptr, n, d, ldx, max_passes=2, tol=0.0)
            l2 = ctx.launch_count()
            stats = np.zeros(10, dtype=np.float64)
            rc_s = b2.native.load().b2_score(ctx._h, Xd.ptr, xdt, n, d, ldx, b2.native.MEM_DEVICE, coef.ctypes.data, b0,
                                             yd.ptr, None, 1, None, stats.ctypes.data)
            l3 = ctx.launch_count()
        finally:
            Xd.free(); yd.free()
        assert rc == 0 and rc_s == 0 and passes == 2, (layout, rc, rc_s, passes)
        # a pass: the refinement solve + b2_score's launches on the same rows
        assert (l2 - l1) - (l1 - l0) == 2 * (1 + (l3 - l2)), (layout, l0, l1, l2, l3)
        assert l3 - l2 == 2 * segments, (layout, l3 - l2)


def test_errors(ctx):
    n, d = 20_000, 8
    X, y, _ = orc.column_table(n, d, "constant", seed=3)
    up, yf = X.astype(np.float32), y.astype(np.float32)
    Xd, yd = ctx.to_device(up), ctx.to_device(yf)
    try:
        with pytest.raises(np.linalg.LinAlgError):
            ctx.fit_refined(Xd, yd, max_passes=2)
        est = b2.B200LinearRegression(ctx=ctx, refine=2).fit(Xd, yd)          # min-norm fallback, unrefined
        assert est.rank_ == d - 1 and abs(est.coef_[0]) < 1e-6
        for passes, tol in ((-1, 0.0), (17, 0.0), (2, -1.0), (2, float("nan"))):
            rc = _raw_refined(ctx, Xd.ptr, b2.F32, yd.ptr, n, d, d, max_passes=passes, tol=tol)[0]
            assert rc == E_ARG, (passes, tol, rc)
    finally:
        Xd.free(); yd.free()
    other = b2.Context(0)
    try:
        b2.Context.comm_p2p_attach_local([ctx, other])
        Xr, up, y2 = _table(4096, 8, "offset", "f32", seed=5)
        Xd, yd = ctx.to_device(up), ctx.to_device(y2)
        rc = _raw_refined(ctx, Xd.ptr, b2.F32, yd.ptr, 4096, 8, 8)[0]
        assert rc == E_UNSUPPORTED, rc
        Xd.free(); yd.free()
    finally:
        for c in (ctx, other):
            c.comm_p2p_detach()
        other.close()


def test_estimator_refine_matches_sklearn_and_round_trips(ctx, tmp_path):
    import joblib
    X, y, _ = orc.column_table(300_000, 64, "correlated", seed=92, rho=0.999)
    Xf, yf = X.astype(np.float32), y.astype(np.float32)
    Xr = Xf.astype(np.float64)
    sk = _sk(Xr, yf)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)             # tol 1e-10 may need more than two passes
        est = b2.B200LinearRegression(ctx=ctx, refine=2).fit(Xf, yf)
    plain = b2.B200LinearRegression(ctx=ctx).fit(Xf, yf)
    print(f"[refine] estimator refine=2: {_err(est.coef_, sk.coef_, Xr):.3g} (plain {_err(plain.coef_, sk.coef_, Xr):.3g}) "
          f"passes={est.n_refine_passes_} step={est.refine_step_:.3g}")
    assert _err(est.coef_, sk.coef_, Xr) < 1e-6 and est.n_refine_passes_ >= 1
    assert repr(est) == "B200LinearRegression(refine=2)" and repr(plain) == "B200LinearRegression()"
    path = tmp_path / "model.joblib"
    joblib.dump(est.to_sklearn(), path)
    back = joblib.load(path)
    assert np.array_equal(back.coef_, est.coef_) and back.intercept_ == est.intercept_
    with pytest.raises(ValueError, match="refine"):
        b2.B200LinearRegression(ctx=ctx, refine=1).partial_fit(Xf[:1000], yf[:1000])
    with pytest.raises(ValueError, match="refine"):
        b2.B200LinearRegression(ctx=ctx, refine=1).solve_resident(64)
