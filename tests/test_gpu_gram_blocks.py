"""The tensor-core Gram kernel computes hi^T hi only from each warpgroup's own 64 features on (its upper half), drains
only the upper triangle of it, and the fold reads each entry of S from one partial entry.  These tests check that
mapping on tables whose blocks across feature 64 are large and not symmetric by accident:

  * cross-half tables: feature j is correlated with feature j + 64 (d > 64), or with feature j + d / 2 of the same
    original row (packed rows, d <= 64), each pair with its own coefficient, mean and scale; at packed d = 24 and 40 a
    sub-row straddles feature 64 of the super-row;
  * stale partials: a different table (other E width, other variant) runs through the same context first, so a
    reduce or fold that reads a partial entry this launch did not write picks up a wrong value, not a correct one;
  * both operand modes, hi + lo (PRECISION_SPLIT) and one bf16 operand (PRECISION_BF16).

Tolerances: hi + lo as tests/test_gpu_columns.py (stat 2e-5, mean 1e-6, coef 6e-5 or 2.5e-6 * kappa).  One operand
(relative operand error 2^-9 of |x - c|, which reaches 3 sigma here): stat and mean measured up to 1.7e-3 on bf16 rows
(6e-5 on fp32 rows), asserted at 5e-3; coef at 5e-2.  A misplaced block or a stale entry is wrong by O(1).
"""
import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc

pytestmark = pytest.mark.gpu

TC = b2.KERNEL_TCGEN05
N = 60_000

# path id -> (d, storage).  d > 64: the fixed-D (128) and runtime-d kernels; d <= 64: packed rows (pack = 5, 4, 3, 2, 2);
# rawb-d128: bf16 rows whose raw tile is the MMA's B operand
PATHS = {
    "f32-d128": (128, "f32"), "f32-d72": (72, "f32"), "f32-d100": (100, "f32"),
    "packed-d24": (24, "f32"), "packed-d32": (32, "f32"), "packed-d40": (40, "f32"), "packed-d48": (48, "f32"),
    "packed-d64": (64, "f32"), "rawb-d128": (128, "bf16"), "bf16-d96": (96, "bf16"),
}
PRECISIONS = {"split": b2.PRECISION_SPLIT, "bf16": b2.PRECISION_BF16}
TOL = {"split": (2e-5, 1e-6, 6e-5), "bf16": (5e-3, 5e-3, 5e-2)}


def _cross_half_table(n, d, kind, seed):
    """(rows as the kernel sees them in float64, the array to upload, y as float32): x_j = m_j + s_j (z_j + a_j z_p(j))
    with p(j) = j + 64 (d > 64) or j + d / 2 (mod d)."""
    rng = np.random.RandomState(seed)
    z = rng.standard_normal((n, d))
    half = 64 if d > 64 else d // 2
    partner = (np.arange(d) + half) % d
    a = rng.uniform(0.3, 0.9, d) * rng.choice([-1.0, 1.0], d)
    scale = 10.0 ** rng.uniform(-1, 1, d)
    mean = scale * rng.uniform(-3, 3, d)
    X = mean + scale * (z + a * z[:, partner])
    w = rng.standard_normal(d) / scale
    y = (X @ w + rng.standard_normal(n)).astype(np.float32)
    if kind == "bf16":
        up = b2.native.to_bf16_bits(X.astype(np.float32))
        return b2.native.from_bf16_bits(up).astype(np.float64), up, y
    up = X.astype(np.float32)
    return up.astype(np.float64), up, y


def _accumulate(ctx, up, y, d, kind):
    ctx.set_kernel(TC)
    try:
        ctx.gram_reset(d)
        Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
        ctx.gram_accumulate(Xd, yd)
        Xd.free(); yd.free()
        return ctx.gram_export()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)


def _prime(ctx, path):
    """Leave other variants' entries in the per-CTA partials: a hi + lo run with 16 E columns (packed d = 24) and one of
    the fixed-D kernel, on tables unlike the one under test."""
    ctx.set_precision(b2.PRECISION_SPLIT)
    for d, kind in ((24, "f32"), (128, "bf16" if path == "f32-d128" else "f32")):
        _, up, y = _cross_half_table(N, d, kind, seed=900 + d)
        _accumulate(ctx, (1e3 * up).astype(np.float32) if kind == "f32" else up, (1e3 * y).astype(np.float32), d, kind)


@pytest.mark.parametrize("precision", list(PRECISIONS))
@pytest.mark.parametrize("path", list(PATHS))
def test_cross_half_blocks_after_another_table(ctx, path, precision):
    d, kind = PATHS[path]
    Xr, up, y = _cross_half_table(N, d, kind, seed=d + 7)
    So = orc.gram_stats(Xr, y)
    tol_stat, tol_mean, tol_coef = TOL[precision]
    kappa = orc.centred_condition(So)
    fo = orc.fit_from_stats(So)
    try:
        _prime(ctx, path)
        ctx.set_precision(PRECISIONS[precision])
        S = _accumulate(ctx, up, y, d, kind)
        assert S[d, d] == N and np.array_equal(S, S.T)
        stat, mean = orc.stat_error(S, So)
        assert stat < tol_stat and mean < tol_mean, (stat, mean)
        # the estimator's fit (b2_fit) of the same rows, after the priming tables again
        _prime(ctx, path)
        ctx.set_precision(PRECISIONS[precision])
        Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
        ctx.set_kernel(TC)
        est = b2.B200LinearRegression(ctx=ctx).fit(Xd, yd)
        Xd.free(); yd.free()
        S2 = ctx.gram_export()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        ctx.set_precision(b2.PRECISION_SPLIT)
    assert np.array_equal(S, S2)
    err = orc.coef_error(est.coef_, fo["coef"], So)
    assert err < max(tol_coef, 2.5e-6 * kappa if precision == "split" else tol_coef), (kappa, err)
