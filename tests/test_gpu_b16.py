"""bf16-stored D = 128 rows through the tensor-core Gram kernel (csrc/gram_tc.cu, T = bf16: hi + lo operands, or a single
operand) against the fp64 oracle of the SAME bf16-rounded rows.

Tolerances: the statistic within 2e-6 relative, the row count exact, coefficients within 2e-5 (contract 1e-4) in the
default hi+lo mode; the single-operand mode ('bf16-accum') within the 1e-4 contract at large n only (its operand
rounding error falls as 1/sqrt(n)), so small cases check its statistic at the operand precision (2^-8).
"""
import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc

pytestmark = pytest.mark.gpu

COEF_TOL = 2e-5


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), 1e-300))


def _rows(n, seed):
    X, y = orc.generate_dataset(n, 128, seed=seed, dtype=np.float32)
    bits = b2.native.to_bf16_bits(X)
    return bits, b2.native.from_bf16_bits(bits), y


def _accumulate(ctx, bits, y, mask=None, keep=1, ldx=128, precision=None):
    """b2_gram_accumulate through the raw C-ABI (the Python wrapper always passes ldx = d)."""
    n = bits.shape[0]
    if ldx != 128:
        wide = np.zeros((n, ldx), dtype=np.uint16)
        wide[:, :128] = bits
        wide[:, 128:] = 0x7FC0          # NaN padding: must never be read
        bits = wide
    ctx.set_kernel(b2.KERNEL_TCGEN05)
    if precision is not None:
        ctx.set_precision(precision)
    ctx.gram_reset(128)
    Xd = ctx.to_device(bits, "bf16")
    yd = ctx.to_device(y)
    md = ctx.to_device(mask) if mask is not None else None
    lib = b2.native.load()
    rc = lib.b2_gram_accumulate(ctx._h, Xd.ptr, b2.native.BF16, yd.ptr, n, 128, ldx, b2.native.MEM_DEVICE,
                                md.ptr if md is not None else None, int(keep))
    assert rc == 0, b2.native.last_error()
    S = ctx.gram_export()
    for a in (Xd, yd, md):
        if a is not None:
            a.free()
    ctx.set_kernel(b2.KERNEL_AUTO)
    ctx.set_precision(b2.PRECISION_SPLIT)
    return S


@pytest.mark.parametrize("n", [64, 65, 127, 8192 + 17, 100_003, 300_000])
def test_b16_gram_matches_oracle(ctx, n):
    bits, Xr, y = _rows(n, seed=n)
    S = _accumulate(ctx, bits, y)
    So = orc.gram_stats(Xr, y)
    assert S[128, 128] == n
    assert _rel(S[:128, 128], So[:128, 128]) < 1e-6
    assert _rel(S, So) < 2e-6
    assert np.array_equal(S, S.T)
    if n > 1000:
        ctx.gram_import(S)
        coef, _ = ctx.solve()
        assert np.max(np.abs(coef - orc.fit_from_stats(So)["coef"])) < COEF_TOL


@pytest.mark.parametrize("n,keep,ldx", [(70_001, 1, 128), (70_001, 0, 128), (33_333, 1, 136), (8_192, 0, 256)])
def test_b16_mask_equals_gather_and_row_pitch(ctx, n, keep, ldx):
    bits, Xr, y = _rows(n, seed=n + keep)
    mask = (np.random.RandomState(n).rand(n) < 0.8).astype(np.uint8)
    S = _accumulate(ctx, bits, y, mask=mask, keep=keep, ldx=ldx)
    sel = mask == keep
    So = orc.gram_stats(Xr[sel], y[sel])
    assert S[128, 128] == int(sel.sum())
    assert _rel(S, So) < 2e-6
    assert np.array_equal(S, S.T)
    ctx.gram_import(S)
    coef, _ = ctx.solve()
    assert np.max(np.abs(coef - orc.fit_from_stats(So)["coef"])) < COEF_TOL


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_b16_dropped_rows_may_hold_nan(ctx, precision):
    """A masked-out row never reaches the statistic, whatever it holds: dropped rows are zeroed before they become tensor
    core operands (0 * NaN would poison the sums)."""
    n = 50_001
    bits, Xr, y = _rows(n, seed=17)
    mask = (np.random.RandomState(3).rand(n) < 0.7).astype(np.uint8)
    bits = bits.copy(); y = y.copy()
    drop = np.flatnonzero(mask == 0)
    bits[drop[::3]] = 0x7FC0            # NaN rows
    bits[drop[1::3]] = 0x7F80           # +Inf rows
    y[drop[::5]] = np.nan
    prec = b2.PRECISION_SPLIT if precision == "split" else b2.PRECISION_BF16
    S = _accumulate(ctx, bits, y, mask=mask, keep=1, precision=prec)
    assert np.all(np.isfinite(S))
    sel = mask == 1
    So = orc.gram_stats(Xr[sel], y[sel])
    assert S[128, 128] == int(sel.sum())
    assert _rel(S, So) < (2e-6 if precision == "split" else 2e-4)


def test_b16_is_deterministic_and_additive(ctx):
    bits, Xr, y = _rows(150_000, seed=5)
    a = _accumulate(ctx, bits, y)
    b = _accumulate(ctx, bits, y)
    assert np.array_equal(a, b)
    ctx.set_kernel(b2.KERNEL_TCGEN05)
    ctx.gram_reset(128)
    for lo, hi in ((0, 64_000), (64_000, 150_000)):
        Xd, yd = ctx.to_device(bits[lo:hi], "bf16"), ctx.to_device(y[lo:hi])
        ctx.gram_accumulate(Xd, yd)
        Xd.free(); yd.free()
    parts = ctx.gram_export()
    ctx.set_kernel(b2.KERNEL_AUTO)
    assert parts[128, 128] == 150_000
    assert _rel(parts, a) < 2e-6


def test_b16_single_operand_mode(ctx):
    """'bf16-accum' (BASELINE.json configs[1]): one operand hi = rn(x - c); zero-mean rounding error 2^-9 per element."""
    n = 1_000_000
    bits, Xr, y = _rows(n, seed=99)
    S = _accumulate(ctx, bits, y, precision=b2.PRECISION_BF16)
    So = orc.gram_stats(Xr, y)
    assert S[128, 128] == n
    assert np.array_equal(S, S.T)
    ctx.gram_import(S)
    coef, _ = ctx.solve()
    err = np.max(np.abs(coef - orc.fit_from_stats(So)["coef"]))
    assert err < 1e-4, err
    S2 = _accumulate(ctx, bits, y)          # default mode on the same rows
    ctx.gram_import(S2)
    coef2, _ = ctx.solve()
    assert np.max(np.abs(coef2 - orc.fit_from_stats(So)["coef"])) < COEF_TOL


def test_b16_generic_kernel_agrees(ctx, monkeypatch):
    """Rows with a feature count other than 128 stay on the generic kernel; at D = 128 both kernels see the same rows."""
    bits, Xr, y = _rows(90_000, seed=3)
    S = _accumulate(ctx, bits, y)
    ctx.set_kernel(b2.KERNEL_SIMT)
    ctx.gram_reset(128)
    Xd, yd = ctx.to_device(bits, "bf16"), ctx.to_device(y)
    ctx.gram_accumulate(Xd, yd)
    exact = ctx.gram_export()
    Xd.free(); yd.free()
    ctx.set_kernel(b2.KERNEL_AUTO)
    assert _rel(S, exact) < 2e-6
