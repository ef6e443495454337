"""Every Gram path on the columns real tables have: offset, scaled, integer / 0-1, constant and correlated columns
(oracle.ols_oracle.column_table), against the fp64 oracle of the same rows (fp32- or bf16-rounded as the kernel sees
them), through b2_gram_accumulate and through b2_fit / the estimator.

The kernels' precision depends on |x - c| / sigma (c: the per-column shift) and on the conditioning of the centred
Gram, not on the size of S, so every check here is scale-free (oracle.ols_oracle.stat_error / coef_error):
  * stat:  max |C_ab - Co_ab| / sqrt(Co_aa Co_bb) over the centred second moments of [X y];
  * mean:  max |xbar_j - xbaro_j| / sigma_j;
  * coef:  max |coef_j - coefo_j| * sigma_j (the plain coefficient error for sigma = 1 columns), against
           fit_from_stats of the same kept rows.
The row count is exact and S is symmetric on every path.

Tolerances (largest value measured on one H100 80GB HBM3 at a 400 W power limit -> asserted):
  tensor core, hi + lo operands:  stat 7.5e-6 -> 2e-5, mean 3.4e-8 -> 1e-6, coef 3.8e-5 -> 6e-5
  tensor core, 1.2 M rows:        stat 2.8e-5 -> 1e-4 (fp32 accumulation over full 8192-row drains), coef 4.0e-5 -> 6e-5
  narrow (CUDA-core fp32 FMA):    stat 4.7e-7 -> 2e-6, mean 3.6e-8 -> 1e-6, coef 8.9e-7 -> 1e-5
  SIMT (fp64 products):           stat 3.1e-7 -> 1e-6, mean 5e-16 -> 1e-9, coef 5.8e-7 -> 1e-6 (the fp64 raw statistic
                                  itself cancels at mean / sigma = 1e4, in the oracle as in the kernel)
  single bf16 operand, n = 2 M:   coef 7.4e-5 -> 1e-4 (the contract)
  correlated columns:             coef error <= 1.4e-6 * kappa measured, asserted at 2.5e-6 * kappa
    (kappa: condition number of the centred Gram; DESIGN.md section 2)
With the per-column shift rounded to bf16 for fp32 rows (the earlier kernel), offset columns measured stat 9.9e-4, the
single-operand fit 0.26 and the two-block fit 1.8e-2; with the shift sample dividing by 2048 whatever it skipped, rows
holding NaN on the sample stride measured stat 0.3 (narrow) and 260 (tensor core).
"""
import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc

pytestmark = pytest.mark.gpu

TC, NARROW, SIMT = b2.KERNEL_TCGEN05, b2.KERNEL_NARROW, b2.KERNEL_SIMT

# path id -> (d, storage, kernel).  f32-d128: the fixed-D kernel; d72 / d100 (f32) and d96 (bf16): the runtime-d kernel;
# packed-d24 / 32 / 48: 5, 4 and 2 rows to a 128-wide super-row; rawb-d128: bf16 rows whose raw tile is the MMA's B
# operand; tc-d8: the tensor-core kernel forced on narrow rows; narrow-*: the CUDA-core narrow kernel; simt: the control.
PATHS = {
    "f32-d128": (128, "f32", TC), "f32-d72": (72, "f32", TC), "f32-d100": (100, "f32", TC),
    "packed-d24": (24, "f32", TC), "packed-d32": (32, "f32", TC), "packed-d48": (48, "f32", TC),
    "rawb-d128": (128, "bf16", TC), "bf16-d96": (96, "bf16", TC), "tc-d8": (8, "f32", TC),
    "narrow-d1": (1, "f32", NARROW), "narrow-d4": (4, "f32", NARROW), "narrow-d16": (16, "f32", NARROW),
    "narrow-bf16-d1": (1, "bf16", NARROW), "narrow-bf16-d4": (4, "bf16", NARROW), "narrow-bf16-d16": (16, "bf16", NARROW),
    "simt-d8": (8, "f32", SIMT),
}
# kernel -> (stat, mean, coef) tolerances
TOL = {TC: (2e-5, 1e-6, 6e-5), NARROW: (2e-6, 1e-6, 1e-5), SIMT: (1e-6, 1e-9, 1e-6)}
TC_STAT_MANY_DRAINS = 1e-4      # stat error once every CTA folds several full 8192-row drains (fp32 accumulation)

FAMILIES = ["offset", "scaled-small", "scaled-large", "integer", "constant", "correlated"]


def _table(n, d, family, kind, seed):
    """(rows as the kernel sees them in float64, the array to upload, y as float32)"""
    fam, kw = family, {}
    if family.startswith("scaled"):
        fam, kw = "scaled", {"scale": 1e-3 if family == "scaled-small" else 1e3}
    elif family == "correlated":
        kw = {"rho": 0.5}           # kappa ~ 9: high correlation has its own test below
    X, y, _ = orc.column_table(n, d, fam, seed=seed, bf16=(kind == "bf16"), **kw)
    y = y.astype(np.float32)
    if kind == "bf16":
        up = b2.native.to_bf16_bits(X.astype(np.float32))
        return b2.native.from_bf16_bits(up).astype(np.float64), up, y
    up = X.astype(np.float32)
    return up.astype(np.float64), up, y


def _accumulate(ctx, parts, d, kernel, kind, mask=None, keep=1):
    """b2_gram_accumulate of each (rows, y) in `parts` into one statistic (each call samples its own shift)."""
    ctx.set_kernel(kernel)
    try:
        ctx.gram_reset(d)
        for k, (up, y) in enumerate(parts):
            Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
            md = ctx.to_device(mask) if mask is not None else None
            ctx.gram_accumulate(Xd, yd, md, keep)
            for a in (Xd, yd, md):
                if a is not None:
                    a.free()
        return ctx.gram_export()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)


def _fit(ctx, up, y, kernel, kind, mask=None, keep=1):
    """The estimator's default fit (b2_fit, + the spectral solve when the centred Gram is rank deficient) on device rows."""
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    md = ctx.to_device(mask) if mask is not None else None
    ctx.set_kernel(kernel)
    try:
        est = b2.B200LinearRegression(ctx=ctx).fit(Xd, yd, row_mask=md, mask_keep=keep)
        return est, ctx.gram_export()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        for a in (Xd, yd, md):
            if a is not None:
                a.free()


def _check_stat(S, So, kernel, what, tol_stat=None):
    d = So.shape[0] - 2
    assert S[d, d] == So[d, d], what                          # the row count is exact
    assert np.array_equal(S, S.T), what
    stat, mean = orc.stat_error(S, So)
    tol_stat = tol_stat if tol_stat is not None else TOL[kernel][0]
    tol_mean = TOL[kernel][1]
    assert stat < tol_stat, (what, stat)
    assert mean < tol_mean, (what, mean)


def _check_coef(coef, So, kernel, what, tol=None):
    fo = orc.fit_from_stats(So)
    err = orc.coef_error(coef, fo["coef"], So)
    assert err < (tol if tol is not None else TOL[kernel][2]), (what, err)


def _paths_and_families():
    out = []
    for path, (d, _, _) in PATHS.items():
        for fam in FAMILIES:
            if d == 1 and fam in ("constant", "correlated"):
                continue
            out.append((path, fam))
    return out


@pytest.mark.parametrize("path,family", _paths_and_families())
def test_every_path_on_structured_columns(ctx, path, family):
    d, kind, kernel = PATHS[path]
    n = 100_003
    Xr, up, y = _table(n, d, family, kind, seed=d)
    So = orc.gram_stats(Xr, y)
    # b2_gram_accumulate
    S = _accumulate(ctx, [(up, y)], d, kernel, kind)
    _check_stat(S, So, kernel, "accumulate")
    if family != "constant":
        ctx.gram_import(S)
        coef, _ = ctx.solve()
        _check_coef(coef, So, kernel, "accumulate + solve")
    # b2_fit through the estimator
    est, S2 = _fit(ctx, up, y, kernel, kind)
    _check_stat(S2, So, kernel, "b2_fit")
    _check_coef(est.coef_, So, kernel, "estimator")
    if family == "constant":                  # column 0 never varies: rank d - 1 and a zero coefficient, as sklearn
        assert est.rank_ == d - 1
        assert abs(est.coef_[0]) < 1e-6, est.coef_[0]
    else:
        assert est.rank_ == d


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("keep", [0, 1])
def test_masked_offset_columns(ctx, path, keep):
    d, kind, kernel = PATHS[path]
    n = 70_001
    Xr, up, y = _table(n, d, "offset", kind, seed=100 + d)
    mask = (np.random.RandomState(d + keep).rand(n) < 0.6).astype(np.uint8)
    sel = mask == keep
    So = orc.gram_stats(Xr[sel], y[sel])
    S = _accumulate(ctx, [(up, y)], d, kernel, kind, mask=mask, keep=keep)
    _check_stat(S, So, kernel, "accumulate")
    est, S2 = _fit(ctx, up, y, kernel, kind, mask=mask, keep=keep)
    _check_stat(S2, So, kernel, "b2_fit")
    _check_coef(est.coef_, So, kernel, "estimator")


@pytest.mark.parametrize("path", list(PATHS))
def test_two_accumulates_with_different_shifts(ctx, path):
    """Two blocks whose column means differ by one sigma into one statistic: each call samples and undoes its own c
    (a shift of 10 at the mean 1e5, sigma 10 columns, against the first block's)."""
    d, kind, kernel = PATHS[path]
    Xr, up, y = _table(120_000, d, "offset", kind, seed=200 + d)
    sd = np.sqrt(np.diag(orc.centred_moments(orc.gram_stats(Xr, y))[2])[:d] / Xr.shape[0])
    Xb = Xr[50_000:] + sd
    if kind == "bf16":
        upb = b2.native.to_bf16_bits(Xb.astype(np.float32))
        Xb = b2.native.from_bf16_bits(upb).astype(np.float64)
    else:
        upb = Xb.astype(np.float32)
        Xb = upb.astype(np.float64)
    Xall = np.concatenate([Xr[:50_000], Xb])
    So = orc.gram_stats(Xall, y)
    S = _accumulate(ctx, [(up[:50_000], y[:50_000]), (upb, y[50_000:])], d, kernel, kind)
    _check_stat(S, So, kernel, "two accumulates")
    ctx.gram_import(S)
    coef, _ = ctx.solve()
    _check_coef(coef, So, kernel, "solve")


@pytest.mark.parametrize("kind", ["f32", "bf16"])
def test_offset_columns_over_many_drains(ctx, kind):
    """1.2 M rows at D = 128: more than 132 SMs x 8192 rows, so every CTA drains its fp32 accumulators more than once at
    the default interval (the bf16 raw-operand path drains every 2048 rows)."""
    n, d = 1_200_000, 128
    Xr, up, y = _table(n, d, "offset", kind, seed=31)
    So = orc.gram_stats(Xr, y)
    S = _accumulate(ctx, [(up, y)], d, TC, kind)
    _check_stat(S, So, TC, "accumulate", tol_stat=TC_STAT_MANY_DRAINS)
    est, S2 = _fit(ctx, up, y, TC, kind)
    assert np.array_equal(S, S2)
    _check_coef(est.coef_, So, TC, "estimator")


@pytest.mark.parametrize("kind", ["f32", "bf16"])
def test_single_operand_mode_on_offset_columns(ctx, kind):
    """PRECISION_BF16 (one bf16 operand hi = rn(x - c)): its rounding error is relative to |x - c|, so on offset columns
    it meets the 1e-4 contract at n = 2 M only with a shift that keeps x - c small."""
    n, d = 2_000_000, 128
    Xr, up, y = _table(n, d, "offset", kind, seed=47)
    So = orc.gram_stats(Xr, y)
    ctx.set_precision(b2.PRECISION_BF16)
    try:
        S = _accumulate(ctx, [(up, y)], d, TC, kind)
    finally:
        ctx.set_precision(b2.PRECISION_SPLIT)
    assert S[d, d] == n and np.array_equal(S, S.T)
    ctx.gram_import(S)
    coef, _ = ctx.solve()
    _check_coef(coef, So, TC, "single operand", tol=1e-4)


@pytest.mark.parametrize("path", list(PATHS))
def test_dropped_rows_may_hold_nan(ctx, path):
    """A masked-out row never reaches the statistic, whatever it holds -- including rows the shift sample reads (every
    (n // 2048)-th row): the sample ignores the mask, so it must skip non-finite values."""
    d, kind, kernel = PATHS[path]
    n = 50_001
    Xr, up, y = _table(n, d, "offset", kind, seed=300 + d)
    mask = (np.random.RandomState(3).rand(n) < 0.7).astype(np.uint8)
    mask[:: n // 2048] = 0                          # every sampled row is dropped ...
    drop = np.flatnonzero(mask == 0)
    up = up.copy(); y = y.copy()
    nan_bits, inf_bits = (0x7FC0, 0x7F80) if kind == "bf16" else (np.nan, np.inf)
    up[drop[::3]] = nan_bits                        # ... and many of them hold NaN or Inf
    up[drop[1::3]] = inf_bits
    y[drop[::5]] = np.nan
    sel = mask == 1
    So = orc.gram_stats(Xr[sel], y[sel])
    S = _accumulate(ctx, [(up, y)], d, kernel, kind, mask=mask, keep=1)
    assert np.all(np.isfinite(S))
    _check_stat(S, So, kernel, "accumulate")
    est, S2 = _fit(ctx, up, y, kernel, kind, mask=mask, keep=1)
    _check_stat(S2, So, kernel, "b2_fit")
    _check_coef(est.coef_, So, kernel, "estimator")


@pytest.mark.parametrize("rho", [0.9, 0.99, 0.999])
@pytest.mark.parametrize("path", ["f32-d128", "rawb-d128", "tc-d8"])
def test_correlated_columns_error_grows_with_the_condition_number(ctx, path, rho):
    """The tensor-core operands carry 16 significand bits, so the coefficient error grows with the condition number
    kappa of the centred Gram, whatever the shift: measured on an H100 as <= 2.5e-8 * kappa, asserted at 1e-7 * kappa.
    Past kappa ~ 1e3 this leaves the 1e-4 contract (DESIGN.md section 2); KERNEL_SIMT is exact at any kappa."""
    d, kind, kernel = PATHS[path]
    X, yy, _ = orc.column_table(200_000, d, "correlated", seed=400, rho=rho)
    yy = yy.astype(np.float32)
    if kind == "bf16":
        up = b2.native.to_bf16_bits(X.astype(np.float32))
        Xr = b2.native.from_bf16_bits(up).astype(np.float64)
    else:
        up = X.astype(np.float32)
        Xr = up.astype(np.float64)
    So = orc.gram_stats(Xr, yy)
    kappa = orc.centred_condition(So)
    S = _accumulate(ctx, [(up, yy)], d, kernel, kind)
    assert S[d, d] == So[d, d] and np.array_equal(S, S.T)
    ctx.gram_import(S)
    coef, _ = ctx.solve()
    err = orc.coef_error(coef, orc.fit_from_stats(So)["coef"], So)
    assert err < 2.5e-6 * kappa, (kappa, err)
    exact = _accumulate(ctx, [(up, yy)], d, SIMT, kind)
    ctx.gram_import(exact)
    coef_s, _ = ctx.solve()
    assert orc.coef_error(coef_s, orc.fit_from_stats(So)["coef"], So) < 1e-7
