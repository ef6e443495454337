"""The tensor-core Gram kernel's chunk drains: each drained D1 entry keeps its running fp64 sum in its owner thread's
registers, in the shared slab or in the CTA's partial in L2, and the end of the range writes the on-chip sums to the
partial.  At short drain intervals (every tile, every two tiles) and the default one, on offset and correlated columns:
the statistic is the exact kernel's within the tolerances of test_gpu_parity.py, repeated calls are bit-identical, and
a narrow table after a wide one through the same context reads no stale partial entry."""
import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc

pytestmark = pytest.mark.gpu

SF_TOL = 2e-5        # test_gpu_parity.py: scale-free statistic error of the tensor-core kernel

# (d, storage): the fixed-D kernel, the runtime-d kernel, rows packed 2 and 5 to a super-row, bf16 rows whose raw tile
# is the MMA's B operand
PATHS = [(128, "f32"), (96, "f32"), (64, "f32"), (24, "f32"), (128, "bf16")]


def _table(n, d, family, kind, seed):
    X, y, _ = orc.column_table(n, d, family, seed=seed, bf16=(kind == "bf16"), **({"rho": 0.5} if family == "correlated" else {}))
    y = y.astype(np.float32)
    if kind == "bf16":
        up = b2.native.to_bf16_bits(X.astype(np.float32))
        return b2.native.from_bf16_bits(up).astype(np.float64), up, y
    up = X.astype(np.float32)
    return up.astype(np.float64), up, y


def _gram(ctx, Xd, yd, d, kernel, drain=8192, md=None):
    ctx.set_kernel(kernel)
    ctx.set_drain_rows(drain)
    try:
        ctx.gram_reset(d)
        ctx.gram_accumulate(Xd, yd, md, 1)
        return ctx.gram_export()
    finally:
        ctx.set_drain_rows(8192)
        ctx.set_kernel(b2.KERNEL_AUTO)


@pytest.mark.parametrize("family", ["offset", "correlated"])
@pytest.mark.parametrize("drain", [64, 128, 8192])
@pytest.mark.parametrize("d,kind", PATHS)
def test_drained_statistic_matches_the_exact_kernel(ctx, d, kind, drain, family):
    n = 150_001
    Xr, up, y = _table(n, d, family, kind, seed=7 * d + drain % 101)
    Xd, yd = ctx.to_device(up, kind), ctx.to_device(y)
    try:
        S = _gram(ctx, Xd, yd, d, b2.KERNEL_TCGEN05, drain)
        S_again = _gram(ctx, Xd, yd, d, b2.KERNEL_TCGEN05, drain)
        S_exact = _gram(ctx, Xd, yd, d, b2.KERNEL_SIMT)
    finally:
        Xd.free(); yd.free()
    assert np.array_equal(S, S_again)                      # the same sums in the same order, bit for bit
    assert S[d, d] == n
    assert np.array_equal(S, S.T)
    assert max(orc.stat_error(S, S_exact)) < SF_TOL, (family, drain)
    So = orc.gram_stats(Xr, y)
    ctx.gram_import(S)
    coef, _ = ctx.solve()
    assert orc.coef_error(coef, orc.fit_from_stats(So)["coef"], So) < 6e-5   # test_gpu_columns.py's tensor-core bound


@pytest.mark.parametrize("drain", [64, 8192])
def test_narrow_table_after_a_wide_one_reads_no_stale_entry(drain):
    """A wide launch leaves every partial entry written; a narrow one (fewer feature columns, wider E block) writes and
    reads its own prefix.  Its statistic and fit equal those of a fresh context, bit for bit, masked and not."""
    wide = _table(100_000, 128, "offset", "f32", seed=3)
    narrow = _table(90_011, 20, "correlated", "f32", seed=4)
    mask = (np.random.RandomState(5).rand(90_011) < 0.6).astype(np.uint8)

    def run(c, tables):
        out = []
        for _, up, y in tables:
            Xd, yd, md = c.to_device(up), c.to_device(y), c.to_device(mask) if up.shape[0] == mask.size else None
            try:
                for m in (None, md) if md is not None else (None,):
                    out.append(_gram(c, Xd, yd, up.shape[1], b2.KERNEL_TCGEN05, drain, m))
                    c.set_kernel(b2.KERNEL_TCGEN05)
                    c.set_drain_rows(drain)
                    out.append(np.concatenate([np.atleast_1d(v) for v in c.fit(Xd, yd, row_mask=m)]))
                    c.set_drain_rows(8192)
                    c.set_kernel(b2.KERNEL_AUTO)
            finally:
                for a in (Xd, yd, md):
                    if a is not None:
                        a.free()
        return out

    def in_fresh_context(tables):
        c = b2.Context(0)
        try:
            return run(c, tables)
        finally:
            c.close()

    shared = in_fresh_context([wide, narrow, wide])
    alone_narrow = in_fresh_context([narrow])
    alone_wide = in_fresh_context([wide])
    assert len(shared) == 2 + 4 + 2
    for a, b in zip(shared[2:6], alone_narrow):
        assert np.array_equal(a, b)
    for a, b in zip(shared[6:], alone_wide):
        assert np.array_equal(a, b)
    for a, b in zip(shared[:2], alone_wide):
        assert np.array_equal(a, b)
