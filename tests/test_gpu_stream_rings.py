"""Scoring (b2_score), the residual gradient (b2_residual_moments, b2_fit_refined) and the narrow Gram on the six-stage
bulk-copy ring of b2_ptx.cuh (ring_init / ring_produce) at row counts where every CTA walks many tiles.

Scoring and the gradient share one plan (plan_rows in score.cu, restated by _plan): rows that are contiguous with X, y
and, for d <= 16, the mask 16-byte aligned stream their whole tiles through the ring -- one lane per row for d <= 16
(score_narrow_kernel, grad_narrow_kernel: tiles of 896 / 448 / 224 rows for DP <= 2 / 4 / 8, 16, 2 G CTAs), LPR lanes per
row for wide rows with d % 4 == 0 and 16-byte row pitch (score_tma_kernel, grad_tma_kernel: tiles of sweeps x 15 x 32 / LPR
rows, G CTAs) -- and the rest of the rows go to the direct kernels (score_kernel_rows8 / score_kernel, grad_kernel).
With G SMs, N_LONG = T (18 grid + 5) + T / 2 + 3 rows give every CTA 18 or 19 tiles (three laps of the ring, both
mbarrier parities), then a direct tail.  On device rows at N_LONG, for every narrow DP with and without whole-vector rows
and every (LPR, sweeps) of the plan, with and without a mask and with mask_keep 0 and 1:
  * the ten statistics against oracle.score_stats on the long-double prediction of the kept rows, the row count exact;
  * each kept yhat within one fp32 ulp of the long-double prediction rounded to fp32, dropped rows exactly 0;
  * metrics-only calls (the PLAIN narrow flavour without a mask), predict-only calls and repeated calls bit-identical;
  * labels 0, 1e-35 and 1e31 in chosen tiles, so one call runs both the fast and the exact statistics of the narrow
    kernel;
  * b2_residual_moments against a long-double reference at a perturbed model and at the least-squares solution, with and
    without fit_intercept, m taken from the resident S as load_refine_state forms it;
  * X or y 4 bytes past a 16-byte boundary (the direct flavour; a misaligned mask only for d <= 16) against the same
    references, and every call's launch count against _plan.
Then the edge row counts of each tile size and grid, masks that empty whole tiles and whole CTAs (NaN and +-Inf in every
dropped row) and b2_fit_refined at N_LONG.

The narrow Gram (gram_narrow.cu) accumulates in fp32 and folds every lane's accumulators into fp64 every kNwFlushRows =
2048 rows per lane, i.e. every F = 2048 / RPT tiles of its CTA.  N_FLUSH = T (grid 3F/2 + 5) + 7 rows make every CTA fold
once mid-run and once at the end, with uneven tile counts and 7 rows for the fp64 tail kernel; the statistic is compared
with a float64 one accumulated on the host from the same Philox rows regenerated block by block.  A dropped or doubled
tile moves the exact row count S[d, d].  A stale ring slot swaps rows for rows of the same distribution, which moves the
statistic far less than its bounds, so every narrow width also runs under lap_mask, which makes each tile keep one row
more or fewer than the tile one lap earlier: there a stale slot moves S[d, d] too.

On the CPU: _plan against the sweep table, the tile counts of N_LONG and N_FLUSH at G = 132 and 114, and that each fault
is visible in what the GPU tests compare: for scoring and the gradient, every bound is at least 100x below what a dropped
tile, a tile counted twice or a stale ring slot (the tile one lap earlier) would do; for the narrow Gram, an accumulator
not zeroed at a mid-run flush moves the statistic 100x beyond its bounds and, under lap_mask, a stale slot moves the row
count.  A float32 model of the 2048-row chains shows why bf16 rows lose more than fp32 rows there (see below).

Bounds (worst case over this file measured on one H100 80GB HBM3, 132 SMs, at a 700 W power limit, in brackets):
  * statistics: 1e-12 relative per entry, test_gpu_parity's bound (1.3e-14);
  * yhat: one fp32 ulp (0: every kept prediction was the long-double one rounded to fp32);
  * gradient: GRAD_TOL = 2e-15 of sum_rows |x_j - m_j| (|y| + |b| + sum_k |x_k c_k|) per entry, and of sum (...) and
    sum (...)^2 for sum e and sum e^2: 5x the worst case measured (3.6e-16, at the perturbed model; 2.9e-16 at the
    least-squares solution);
  * b2_fit_refined: test_gpu_refine.REFINED_TOL = 1e-10 (1.0e-16);
  * narrow Gram: raw statistic 1e-6 relative (test_narrow_gram_matches_oracle), oracle.stat_error 2e-5 and the
    coefficients within test_gpu_parity.COEF_TOL = 2e-5.  fp32 rows: raw 2.0e-9, stat_error 4.0e-8, coefficients
    1.7e-8.  bf16 rows: raw 4.4e-7, stat_error 9.0e-6, coefficients 4.5e-6 -- within the bounds, but ~200x the fp32
    rows.  bf16 values sit on a coarse grid, so x - c has the same low bits in every row and the fp32 roundings of a
    2048-row chain have a mean that depends on the shift c (test_bf16_rows_bias_the_fp32_chains: 5e-9 to 2e-6 relative on
    sum v^2 over eight shifts, against a steady ~4e-8 for fp32 values).  These numbers come from one dataset at one SM
    count, not from a bound: the worst case of a 2048-row fp32 chain is 1.2e-4 relative.
Each GPU test prints the worst case it measured (run with -s).
"""
import ctypes as C
import time
from collections import defaultdict, namedtuple

import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from oracle import ols_oracle as orc
from test_gpu_parity import COEF_TOL
from test_gpu_refine import REFINED_TOL

SCORE_TOL = 1e-12                # test_gpu_parity: b2_score statistics against oracle.score_stats
GRAD_TOL = 2e-15                 # b2_residual_moments against the long-double reference (see the module docstring)
RAW_TOL = 1e-6                   # test_gpu_parity.test_narrow_gram_matches_oracle
SF_TOL = 2e-5                    # oracle.stat_error of the narrow Gram
H100_SMS = 132                   # the CPU checks take the H100 SXM's SM count (and 114, the PCIe card's)
DEV = native.MEM_DEVICE
B = 3.0                          # intercept: predictions stay near 3, far from 0 (no cancellation in x.c + b)

# score.cu: the narrow and wide ring geometries
SN_CONSUMERS = 224               # kSnConsumers: 7 consumer warps, one lane per row
TM_WARPS = 15                    # kTmWarps
TM_X_STAGE = 32768               # kTmXStage
TM_TILE_ROWS_MAX = 240           # kTmTileRowsMax
# gram_narrow.cu
NW_FLUSH_ROWS = 2048             # kNwFlushRows

NARROW = [(k, d) for k in ("f32", "bf16") for d in (1, 2, 4, 8, 16, 3, 5, 7, 12, 15)]
WIDE = [("f32", 20), ("f32", 36), ("f32", 68), ("f32", 128), ("bf16", 24), ("bf16", 40), ("bf16", 72), ("bf16", 128)]
WIDTHS = NARROW + WIDE
# (kind, d) -> (LPR, sweeps, tile rows) of the plan (one row per sweep count the plan can produce)
SWEEP_TABLE = {("f32", 20): (2, 1, 240), ("f32", 32): (2, 1, 240), ("f32", 36): (4, 1, 120), ("f32", 64): (4, 1, 120),
               ("f32", 68): (8, 2, 120), ("f32", 72): (8, 1, 60), ("f32", 128): (8, 1, 60),
               ("bf16", 24): (2, 1, 240), ("bf16", 32): (2, 1, 240), ("bf16", 40): (4, 2, 240),
               ("bf16", 64): (4, 2, 240), ("bf16", 72): (8, 3, 180), ("bf16", 88): (8, 3, 180),
               ("bf16", 96): (8, 2, 120), ("bf16", 128): (8, 2, 120)}

Plan = namedtuple("Plan", "flavour T grid whole tail")     # flavour: ("narrow", DP) | ("wide", LPR, sweeps) | ("direct",)


def narrow_dp(d):
    return 1 if d <= 1 else 2 if d <= 2 else 4 if d <= 4 else 8 if d <= 8 else 16


def _plan(n, d, kind, G, xp=0, yp=0, mp=0):
    """plan_rows (score.cu) for contiguous rows (ldx == d): the ring flavour and its tile rows T and grid, the rows of
    whole tiles it streams and the tail left to the direct kernels.  xp, yp, mp: the pointers (None: absent)."""
    es = 4 if kind == "f32" else 2
    a16 = lambda p: p is None or p % 16 == 0
    rows = a16(xp) and a16(yp)
    if rows and d <= 16 and a16(mp):
        dp = narrow_dp(d)
        flavour, T, cap = ("narrow", dp), SN_CONSUMERS * (4 if dp <= 2 else 2 if dp == 4 else 1), 2 * G
    elif rows and d > 16 and d % 4 == 0 and (d * es) % 16 == 0:
        lpr = 2 if d <= 32 else 4 if d <= 64 else 8
        sweep_rows = TM_WARPS * (32 // lpr)
        sweeps = min(TM_X_STAGE // (sweep_rows * d * es), TM_TILE_ROWS_MAX // sweep_rows)
        flavour, T, cap = ("wide", lpr, sweeps), sweeps * sweep_rows, G
    else:
        return Plan(("direct",), 0, 0, 0, n)
    tiles = n // T
    return Plan(flavour, T, min(tiles, cap), tiles * T, n - tiles * T)


def score_launches(p, n):
    """launch_score: the ring and its ordered reduce when there is a whole tile, the direct kernel and its reduce when
    rows are left; b2_score launches nothing for no rows"""
    return 0 if n == 0 else 2 * int(p.whole > 0) + 2 * int(p.tail > 0)


def grad_launches(p, n):
    """launch_grad: as launch_score, but no rows still run the direct kernel (it writes the zero sums)"""
    return 2 * int(p.whole > 0) + 2 * int(p.tail > 0 or n == 0)


def n_long(T, grid):
    return T * (18 * grid + 5) + T // 2 + 3


def nw_geom(d):
    """NwGeom (gram_narrow.cu): (tile rows, CTAs per SM, rows per lane per tile)"""
    dp = narrow_dp(d)
    rpt = 4 if dp <= 2 else 2 if dp == 4 else 1
    lane_rows = 352 // 2 if dp > 8 else 224
    return lane_rows * rpt, (1 if dp > 8 else 2), rpt


def gram_narrow_main_rows(n, d):
    """gram_narrow_main_rows (gram_narrow.cu): the rows of whole narrow tiles; the rest take the fp64 kernel"""
    T = nw_geom(d)[0]
    return n - n % T


def n_flush(d, G):
    T, per_sm, rpt = nw_geom(d)
    F = NW_FLUSH_ROWS // rpt
    return T * (G * per_sm * (3 * F // 2) + 5) + 7


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


# ---- references -----------------------------------------------------------------------------------------------------
def _chunks(n, step=1 << 15):
    return [slice(r, min(r + step, n)) for r in range(0, n, step)]


def predict_ld(Xv, coef, b):
    """the prediction x.coef + b of every row in long double"""
    out = np.empty(len(Xv), np.longdouble)
    c = coef.astype(np.longdouble)[:, None]
    for s in _chunks(len(Xv)):
        out[s] = (Xv[s].T.astype(np.longdouble) * c).sum(axis=0) + np.longdouble(b)
    return out


def residual_sums(Xv, y, coef, b, kept=None, ft=np.longdouble):
    """[sum x_j e (d), sum e, sum e^2] over the kept rows (None: every row) in long double (or ft), e = y - b - x.coef"""
    if kept is not None:
        Xv, y = Xv[kept], y[kept]
    d = Xv.shape[1]
    c = coef.astype(ft)[:, None]
    out = np.zeros(d + 2, ft)
    for s in _chunks(len(Xv)):
        XT = Xv[s].T.astype(ft)                               # (d, rows): the sums over rows run along contiguous memory
        e = y[s].astype(ft) - ft(b) - (XT * c).sum(axis=0)
        out[:d] += (XT * e).sum(axis=1)
        out[d] += e.sum()
        out[d + 1] += (e * e).sum()
    return out


def moments_from(sums, m):
    """b2_residual_moments from residual_sums: sum (x_j - m_j) e = sum x_j e - m_j sum e, then sum e and sum e^2"""
    d = len(m)
    return np.r_[sums[:d] - m.astype(sums.dtype) * sums[d], sums[d:]].astype(np.float64)


def moments_scale(Xv, y, coef, b, m):
    """the scale of each moment over the rows given: sum |x_j - m_j| a, sum a and sum a^2 with
    a = |y| + |b| + sum_k |x_k coef_k|"""
    a = np.abs(y.astype(np.float64)) + abs(b) + np.abs(Xv) @ np.abs(coef)
    return np.r_[np.abs(Xv - m).T @ a, a.sum(), a @ a]


def moments_ref(Xv, y, coef, b, m, ft=np.longdouble):
    """b2_residual_moments over the rows given and the scale of each entry"""
    return moments_from(residual_sums(Xv, y, coef, b, ft=ft), m), moments_scale(Xv, y, coef, b, m)


def grad_err(got, want, scale):
    return float(np.max(np.abs(got - want) / np.maximum(scale, 1e-300))) if scale.size else 0.0


def stats_err(got, want):
    """worst relative difference of the ten statistics; entries that are not finite (max |yhat / y - 1| over y = 0)
    must be equal"""
    fin = np.isfinite(want)
    if not np.array_equal(got[~fin], want[~fin]):
        return float("inf")
    return float(np.max(np.abs(got[fin] - want[fin]) / np.maximum(np.abs(want[fin]), 1e-300)))


def _ord32(v):
    """float32 values as integers in the order of the reals (+0 and -0 both 0): the ulp distance is their difference"""
    k = np.asarray(v, np.float32).view(np.int32).astype(np.int64)
    return np.where(k < 0, -(k & 0x7FFFFFFF), k)


def ulps(got, want32):
    return int(np.max(np.abs(_ord32(got) - _ord32(want32)))) if len(got) else 0


def score_ref(p_ld, y, kept):
    return orc.score_stats(y[kept], p_ld[kept].astype(np.float64))


# ---- data ---------------------------------------------------------------------------------------------------------
class Table:
    """n seeded rows of d features (fp32 or bf16), labels y near the prediction, labels yx with 0, 1e-35 and 1e31 in
    chosen tiles of T rows (and in the tail), a perturbed model.  dropped: rows whose X and y are NaN / +-Inf."""

    def __init__(self, kind, d, n, seed, T, dropped=None):
        rng = np.random.default_rng(seed)
        X = (rng.normal(size=(n, d)) * 0.5).astype(np.float32)
        self.kind, self.d, self.n = kind, d, n
        self.dt = b2.BF16 if kind == "bf16" else b2.F32
        self.up = native.to_bf16_bits(X) if kind == "bf16" else X
        self.Xv = native.from_bf16_bits(self.up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
        self.coef = rng.normal(size=d) * 0.4 / np.sqrt(d)
        self.pcoef = self.coef + rng.normal(size=d) * 0.3 / np.sqrt(d)          # a model far from the fit: g large
        y = (self.Xv @ self.coef + B + rng.normal(size=n) * 0.3).astype(np.float32)
        yx = y.copy()
        if n > 0:
            for t in range(3, n // max(T, 1), 7):
                yx[t * T + np.array([0, 5, 9, 40, 77]) % T] = [0.0, 1e-35, 1e31, -0.0, -1e-35]
            yx[n - 1] = 0.0
        if dropped is not None:
            bad = np.resize(np.float32([np.nan, np.inf, -np.inf]), (int(dropped.sum()), d))
            X[dropped] = bad
            self.up = native.to_bf16_bits(X) if kind == "bf16" else X
            self.Xv[dropped] = bad
            y[dropped] = bad[:, 0]
            yx[dropped] = bad[:, 0]
        self.y = {"y": y, "yx": yx}


class Dev:
    """A Table's rows, both labels and a mask on the device twice: at the allocation (16-byte aligned) and `off` bytes
    past a 16-byte boundary (4 for X and y, 1 for the mask)."""

    def __init__(self, ctx, t, mask):
        self._bufs = []
        self.x = self._put(ctx, t.up, 4)
        self.y = {k: self._put(ctx, v, 4) for k, v in t.y.items()}
        self.m = self._put(ctx, mask, 1) if mask is not None else (None, None)

    def _put(self, ctx, a, off):
        raw = np.ascontiguousarray(a).view(np.uint8).ravel()
        al, mis = ctx.to_device(raw), ctx.to_device(np.r_[np.zeros(off, np.uint8), raw])
        self._bufs += [al, mis]
        return al.ptr, mis.ptr + off

    def free(self):
        for a in self._bufs:
            a.free()


LAYOUTS = {"ring": (0, 0, 0), "x+4": (1, 0, 0), "y+4": (0, 1, 0), "mask+1": (0, 0, 1)}


def _ptrs(dev, layout, ykey, masked):
    xo, yo, mo = LAYOUTS[layout]
    return dev.x[xo], dev.y[ykey][yo], (dev.m[mo] if masked else None)


def _call(ctx, fn, *args):
    before = ctx.launch_count()
    rc = fn(*args)
    assert rc == 0, native.last_error()
    return ctx.launch_count() - before


def run_score(ctx, t, dev, n, layout, ykey, masked, keep, coef, want_yhat=True, with_y=True):
    """b2_score on device rows: (yhat | None, stats | None, launches, plan)"""
    xp, yp, mp = _ptrs(dev, layout, ykey, masked)
    yp = yp if with_y else None
    stats = np.full(10, np.nan) if with_y else None
    yh = ctx.empty((max(n, 1),), "f32") if want_yhat else None
    c = np.ascontiguousarray(coef, np.float64)           # held for the call: the library reads it through its address
    try:
        launches = _call(ctx, native.load().b2_score, ctx._h, xp, t.dt, n, t.d, t.d, DEV, c.ctypes.data, B, yp, mp,
                         keep, yh.ptr if yh is not None else None, stats.ctypes.data if with_y else None)
        yhat = yh.to_host()[:n] if yh is not None else None
    finally:
        if yh is not None:
            yh.free()
    p = _plan(n, t.d, t.kind, ctx.info()["sm_count"], xp, yp, mp)
    assert launches == score_launches(p, n), (layout, n, p, launches)
    return yhat, stats, p


def run_moments(ctx, t, dev, n, layout, masked, keep, coef, b, fit_intercept):
    """b2_residual_moments on device rows (the resident S sets m): (out, plan)"""
    xp, yp, mp = _ptrs(dev, layout, "y", masked)
    out = np.full(t.d + 2, np.nan)
    c = np.ascontiguousarray(coef, np.float64)           # held for the call: the library reads it through its address
    launches = _call(ctx, native.load().b2_residual_moments, ctx._h, xp, t.dt, yp, n, t.d, t.d, DEV, mp, keep,
                     c.ctypes.data, float(b), int(fit_intercept), out.ctypes.data)
    p = _plan(n, t.d, t.kind, ctx.info()["sm_count"], xp, yp, mp)
    assert launches == grad_launches(p, n), (layout, n, p, launches)
    return out, p


def refine_means(S, fit_intercept):
    """m as load_refine_state (b2_api.cu) forms it from the resident S: S[j, d] times 1 / n, 0 without an intercept"""
    d = S.shape[0] - 2
    n = S[d, d]
    inv_n = 1.0 / n if n > 0 else 0.0
    return S[:d, d] * inv_n if fit_intercept else np.zeros(d)


def check_rows(yhat, want32, kept):
    """kept yhat within one fp32 ulp of the long-double prediction, dropped rows exactly 0; the ulps"""
    u = ulps(yhat[kept], want32[kept])
    assert u <= 1, u
    assert np.all(yhat[~kept].view(np.uint32) == 0)
    return u


def _widths_ids(ws):
    return [f"{k}-d{d}" for k, d in ws]


def _ring_plan(kind, d, G, n=1 << 40):
    return _plan(n, d, kind, G)


# ---- (1) long runs: scoring and the gradient against their references, ring against direct ---------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", WIDTHS, ids=_widths_ids(WIDTHS))
def test_long_runs_score_and_gradient(ctx, kind, d):
    G = ctx.info()["sm_count"]
    ring = _ring_plan(kind, d, G)
    n = n_long(ring.T, ring.grid)
    t0 = time.perf_counter()
    t = Table(kind, d, n, seed=10 * d + (7 if kind == "bf16" else 0), T=ring.T)
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    p_ld = predict_ld(t.Xv, t.coef, B)
    p32 = p_ld.astype(np.float32)
    worst = defaultdict(float)
    seen = defaultdict(set)

    def note(k, v):
        worst[k] = max(worst[k], v)

    try:
        p = _plan(n, d, kind, G, *_ptrs(dev, "ring", "y", True))
        assert p.flavour == ring.flavour and p.whole == n - (ring.T // 2 + 3) and p.grid == ring.grid
        for masked, keep in ((False, 1), (True, 1), (True, 0)):
            kept = mask == keep if masked else np.ones(n, bool)
            for ykey in ("y", "yx"):
                want = score_ref(p_ld, t.y[ykey], kept)
                yhat, st, pl = run_score(ctx, t, dev, n, "ring", ykey, masked, keep, t.coef)
                assert pl.flavour[0] != "direct"
                assert st[5] == kept.sum()
                e = stats_err(st, want)
                assert e < SCORE_TOL, (masked, keep, ykey, e, st, want)
                note("stats", e)
                note("yhat ulp", check_rows(yhat, p32, kept))
                again = run_score(ctx, t, dev, n, "ring", ykey, masked, keep, t.coef)
                assert np.array_equal(again[0], yhat) and np.array_equal(again[1], st)
                # metrics only (PLAIN for narrow rows without a mask), predict only
                _, st2, _ = run_score(ctx, t, dev, n, "ring", ykey, masked, keep, t.coef, want_yhat=False)
                assert np.array_equal(st2, st), (masked, keep, ykey)
                yh3, _, _ = run_score(ctx, t, dev, n, "ring", ykey, masked, keep, t.coef, with_y=False)
                assert np.array_equal(yh3.view(np.uint32), yhat.view(np.uint32)), (masked, keep, ykey)
                # X or y off its 16-byte boundary, the mask off its boundary
                for layout in ["x+4", "y+4"] + (["mask+1"] if masked else []):
                    yh_o, st_o, pl = run_score(ctx, t, dev, n, layout, ykey, masked, keep, t.coef)
                    seen["score"].add((layout, pl.flavour[0]))
                    assert st_o[5] == st[5] and stats_err(st_o, want) < SCORE_TOL, (layout, stats_err(st_o, want))
                    note("stats", stats_err(st_o, want))
                    check_rows(yh_o, p32, kept)
                    assert ulps(yh_o, yhat) <= 1
            # the residual moments after a Gram of the same rows made S resident
            mp = dev.m[0] if masked else None
            rc = native.load().b2_gram_reset(ctx._h, d)
            assert rc == 0, native.last_error()
            assert native.load().b2_gram_accumulate(ctx._h, dev.x[0], t.dt, dev.y["y"][0], n, d, d, DEV, mp, keep) == 0
            S = np.empty((d + 2, d + 2))
            assert native.load().b2_gram_export(ctx._h, S.ctypes.data, (C.c_int64 * 1)()) == 0, native.last_error()
            Xk, yk = t.Xv[kept], t.y["y"][kept]
            ls = orc.fit_from_stats(orc.gram_stats(Xk, yk))
            models = {"perturbed": (t.pcoef, B + 0.5), "least squares": (ls["coef"], ls["intercept"])}
            sums = {k: residual_sums(Xk, yk, c, b) for k, (c, b) in models.items()}
            for fi in (1, 0):
                m = refine_means(S, fi)
                for model, (c, b) in models.items():
                    want, scale = moments_from(sums[model], m), moments_scale(Xk, yk, c, b, m)
                    got, pl = run_moments(ctx, t, dev, n, "ring", masked, keep, c, b, fi)
                    assert pl.flavour[0] != "direct"
                    e = grad_err(got, want, scale)
                    assert e < GRAD_TOL, (masked, keep, fi, model, e)
                    note(f"grad {model}", e)
                    again, _ = run_moments(ctx, t, dev, n, "ring", masked, keep, c, b, fi)
                    assert np.array_equal(again, got)
                    for layout in ["x+4", "y+4"] + (["mask+1"] if masked else []):
                        got_o, pl = run_moments(ctx, t, dev, n, layout, masked, keep, c, b, fi)
                        seen["grad"].add((layout, pl.flavour[0]))
                        e = grad_err(got_o, want, scale)
                        assert e < GRAD_TOL, (layout, masked, keep, fi, model, e)
                        note(f"grad {model}", e)
    finally:
        dev.free()
    # X or y off its 16-byte boundary never takes the ring; a misaligned mask only for d <= 16
    for pas, s in seen.items():
        for layout, flavour in s:
            assert (flavour == "direct") == (layout != "mask+1" or d <= 16), (pas, layout, flavour)
    print(f"\n[long {kind} d={d} {ring.flavour} T={ring.T} grid={ring.grid}, n={n}] worst: "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()) + f" ({time.perf_counter() - t0:.1f} s)")


# ---- (2) edge row counts of each tile size and grid ------------------------------------------------------------------
EDGES = [("f32", 1), ("f32", 3), ("bf16", 8), ("f32", 20), ("f32", 36), ("f32", 128), ("bf16", 72)]


def n_edge(T, grid):
    return [0, 1, T - 1, T, T + 1, T * grid, T * grid + 1, 6 * T * grid, T * (6 * grid + 1), T * (6 * grid + 1) + T - 1]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", EDGES, ids=_widths_ids(EDGES))
def test_edge_row_counts(ctx, kind, d):
    G = ctx.info()["sm_count"]
    ring = _ring_plan(kind, d, G)
    sizes = n_edge(ring.T, ring.grid)
    N = max(sizes)
    t = Table(kind, d, N, seed=300 + d, T=ring.T)
    mask = (np.arange(N) % 7 != 3).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    p_ld = predict_ld(t.Xv, t.coef, B)
    p32 = p_ld.astype(np.float32)
    S = orc.gram_stats(t.Xv, t.y["y"])
    ctx.gram_import(S)
    m = refine_means(S, 1)
    worst = defaultdict(float)
    lib = native.load()
    try:
        for n in sizes:
            for masked in (False, True):
                kept = mask[:n] == 1 if masked else np.ones(n, bool)
                if n == 0:      # no rows: zero statistics, no launch, nothing written
                    st = np.full(10, np.nan)
                    yh = ctx.to_device(np.full(4, 7.0, np.float32))
                    try:
                        launches = _call(ctx, lib.b2_score, ctx._h, dev.x[0], t.dt, 0, d, d, DEV, t.coef.ctypes.data,
                                         B, dev.y["y"][0], dev.m[0] if masked else None, 1, yh.ptr, st.ctypes.data)
                        assert launches == 0 and not np.any(st) and np.all(yh.to_host() == 7.0)
                    finally:
                        yh.free()
                else:
                    yhat, st, pl = run_score(ctx, t, dev, n, "ring", "yx", masked, 1, t.coef)
                    assert pl.whole == (n // ring.T) * ring.T and pl.grid == min(n // ring.T, ring.grid)
                    e = stats_err(st, score_ref(p_ld[:n], t.y["yx"][:n], kept))
                    assert e < SCORE_TOL and st[5] == kept.sum(), (n, masked, e)
                    worst["stats"] = max(worst["stats"], e)
                    worst["yhat ulp"] = max(worst["yhat ulp"], check_rows(yhat, p32[:n], kept))
                got, _ = run_moments(ctx, t, dev, n, "ring", masked, 1, t.pcoef, B + 0.5, 1)
                want, scale = moments_ref(t.Xv[:n][kept], t.y["y"][:n][kept], t.pcoef, B + 0.5, m)
                if n == 0:
                    assert not np.any(got)
                e = grad_err(got, want, scale)
                assert e < GRAD_TOL, (n, masked, e)
                worst["grad"] = max(worst["grad"], e)
    finally:
        dev.free()
    print(f"\n[edges {kind} d={d} T={ring.T} grid={ring.grid}, n in {sizes}] worst: "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (3) masks that empty whole tiles and whole CTAs ----------------------------------------------------------------
MASKED = [("f32", 1), ("f32", 8), ("bf16", 12), ("f32", 64), ("bf16", 72)]


def _tile_masks(n, T, grid):
    tile = np.arange(n) // T
    third = (tile % 3 != 2).astype(np.uint8)
    return [("every third tile", third, 1), ("tiles t = 0 mod grid", (tile % grid != 0).astype(np.uint8), 1),
            ("all rows", np.zeros(n, np.uint8), 1), ("mask_keep = 0", third, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", MASKED, ids=_widths_ids(MASKED))
def test_masks_that_empty_tiles(ctx, kind, d):
    G = ctx.info()["sm_count"]
    ring = _ring_plan(kind, d, G)
    n = n_long(ring.T, ring.grid)
    worst = defaultdict(float)
    for label, mask, keep in _tile_masks(n, ring.T, ring.grid):
        kept = mask == keep
        t = Table(kind, d, n, seed=500 + d, T=ring.T, dropped=~kept)
        dev = Dev(ctx, t, mask)
        Xk, yk = t.Xv[kept], t.y["y"][kept]
        S = orc.gram_stats(Xk, yk) if kept.any() else orc.gram_stats(np.zeros((1, d)), np.zeros(1))
        ctx.gram_import(S)
        m = refine_means(S, 1)
        with np.errstate(invalid="ignore"):                 # inf - inf on the dropped rows, which no comparison reads
            p_ld = predict_ld(t.Xv, t.coef, B)
        p32 = p_ld.astype(np.float32)
        try:
            for layout in ("ring", "x+4"):
                for ykey in ("y", "yx"):
                    yhat, st, pl = run_score(ctx, t, dev, n, layout, ykey, True, keep, t.coef)
                    assert (pl.flavour[0] != "direct") == (layout == "ring")
                    want = score_ref(p_ld, t.y[ykey], kept)
                    assert st[5] == kept.sum() and np.all(np.isfinite(st[:9]))
                    e = stats_err(st, want)
                    assert e < SCORE_TOL, (label, layout, ykey, e)
                    worst["stats"] = max(worst["stats"], e)
                    worst["yhat ulp"] = max(worst["yhat ulp"], check_rows(yhat, p32, kept))
                got, _ = run_moments(ctx, t, dev, n, layout, True, keep, t.pcoef, B + 0.5, 1)
                assert np.all(np.isfinite(got))
                want, scale = moments_ref(Xk, yk, t.pcoef, B + 0.5, m)
                e = grad_err(got, want, scale)
                assert e < GRAD_TOL, (label, layout, e)
                worst["grad"] = max(worst["grad"], e)
        finally:
            dev.free()
    print(f"\n[tile masks {kind} d={d} T={ring.T}, n={n}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (4) the refined fit at depth -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", [("f32", 8), ("f32", 64)], ids=["f32-d8", "f32-d64"])
def test_fit_refined_at_depth(ctx, kind, d):
    """b2_fit_refined's residual passes on the ring reach the fp64 least-squares solution of the stored rows"""
    G = ctx.info()["sm_count"]
    ring = _ring_plan(kind, d, G)
    n = n_long(ring.T, ring.grid)
    t = Table(kind, d, n, seed=700 + d, T=ring.T)
    Xd, yd = ctx.to_device(t.up), ctx.to_device(t.y["y"])
    try:
        coef, b, passes, step = ctx.fit_refined(Xd, yd, max_passes=4, tol=1e-13)
    finally:
        Xd.free(); yd.free()
    So = orc.gram_stats(t.Xv, t.y["y"])
    ls = orc.fit_lstsq(t.Xv, t.y["y"])
    e = orc.coef_error(coef, ls["coef"], So)
    print(f"\n[refined {kind} d={d}, n={n}] coef error {e:.2e}, passes {passes}, step {step:.2e}")
    assert passes >= 1 and e < REFINED_TOL, (e, passes, step)
    assert abs(b - ls["intercept"]) < 1e-6 * max(1.0, abs(ls["intercept"]))      # test_gpu_refine's intercept bound


# ---- (5) the narrow Gram across its fp32 -> fp64 flushes ------------------------------------------------------------
FLUSH = [("f32", 1, None), ("f32", 1, "mod 5"), ("f32", 8, None), ("f32", 12, None), ("bf16", 16, None),
         ("bf16", 5, None)] + [(k, d, "lap") for k, d in (("f32", 1), ("f32", 8), ("f32", 12), ("bf16", 16), ("bf16", 5))]


def lap_mask(n, d, G, block=1 << 24):
    """drops row 0 of every narrow-Gram tile in even laps of the six-slot ring and rows 0 and 1 in odd laps (lap = tile
    // (6 grid)): a tile and the tile its CTA streamed through the same slot one lap earlier keep different row counts,
    so a stale slot moves the exact row count S[d, d]"""
    T, per_sm, _ = nw_geom(d)
    lap_tiles = 6 * G * per_sm
    out = np.empty(n, np.uint8)
    for r0 in range(0, n, block):
        r = np.arange(r0, min(r0 + block, n), dtype=np.int64)
        out[r0:r0 + len(r)] = (r % T) > (r // T // lap_tiles) % 2
    return out


def flush_mask(how, n, d, G):
    if how == "mod 5":                              # the reference's 80 / 20 split (stage_1_train_model.py:98-103)
        return (np.arange(n, dtype=np.int64) % 5 != 0).astype(np.uint8)
    return lap_mask(n, d, G) if how == "lap" else None


def _host_gram(ctx, n, d, kind, seed, mask, block=1 << 22):
    """the float64 statistic of the synthetic rows [0, n), regenerated block by block on the device (Philox, counter =
    row index) and accumulated on the host"""
    S = np.zeros((d + 2, d + 2))
    for r0 in range(0, n, block):
        rows = min(block, n - r0)
        X, y = ctx.synth(rows, d, seed=seed, row_offset=r0, kind=kind)
        try:
            Xh, yh = X.to_host(), y.to_host()
        finally:
            X.free(); y.free()
        if kind == "bf16":
            Xh = native.from_bf16_bits(Xh)
        if mask is not None:
            sel = mask[r0:r0 + rows] == 1
            Xh, yh = Xh[sel], yh[sel]
        S += orc.gram_stats(Xh, yh, chunk=1 << 20)
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d,masked", FLUSH, ids=[f"{k}-d{d}" + (f"-{m}" if m else "") for k, d, m in FLUSH])
def test_narrow_gram_across_flushes(ctx, kind, d, masked):
    G = ctx.info()["sm_count"]
    n = n_flush(d, G)
    seed = 4242 + d
    t0 = time.perf_counter()
    X, y = ctx.synth(n, d, seed=seed, kind=kind)
    mask = flush_mask(masked, n, d, G)
    md = ctx.to_device(mask) if masked else None
    out = {}
    try:
        for name, kernel in (("narrow", b2.KERNEL_NARROW), ("again", b2.KERNEL_NARROW), ("auto", b2.KERNEL_AUTO)):
            ctx.set_kernel(kernel)
            ctx.gram_reset(d)
            ctx.gram_accumulate(X, y, md, 1)
            out[name] = ctx.gram_export()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        X.free(); y.free()
        if md is not None:
            md.free()
    t_gpu = time.perf_counter() - t0
    So = _host_gram(ctx, n, d, kind, seed, mask)
    t_host = time.perf_counter() - t0 - t_gpu
    S = out["narrow"]
    assert np.array_equal(out["again"], S) and np.array_equal(out["auto"], S)
    kept = int(mask.sum()) if masked else n
    assert S[d, d] == kept == So[d, d]
    assert np.array_equal(S, S.T)
    e_raw, e_sf = rel(S, So), max(orc.stat_error(S, So))
    ctx.gram_import(S)
    coef, _ = ctx.solve()
    e_coef = float(np.max(np.abs(coef - orc.fit_from_stats(So)["coef"])))
    print(f"\n[narrow Gram {kind} d={d}{' mask ' + masked if masked else ''}, n={n} ({gram_narrow_main_rows(n, d)} on the ring)] "
          f"raw {e_raw:.2e}, stat_error {e_sf:.2e}, coef {e_coef:.2e} (GPU {t_gpu:.1f} s, host reference {t_host:.1f} s)")
    assert e_raw < RAW_TOL and e_sf < SF_TOL and e_coef < COEF_TOL, (e_raw, e_sf, e_coef)


# ---- (6) CPU: the plan, the row counts, and the bounds against the faults they target -------------------------------
def test_plan_reproduces_the_sweep_table():
    G = H100_SMS
    for (kind, d), (lpr, sweeps, T) in SWEEP_TABLE.items():
        p = _plan(1 << 30, d, kind, G)
        assert p.flavour == ("wide", lpr, sweeps) and p.T == T and p.grid == G, (kind, d, p)
    for kind, d in NARROW:
        p = _plan(1 << 30, d, kind, G)
        assert p.flavour == ("narrow", narrow_dp(d)) and p.grid == 2 * G
        assert p.T == {1: 896, 2: 896, 4: 448, 8: 224, 16: 224}[narrow_dp(d)]
    # every sweep count the plan can produce appears among the widths the GPU tests run
    reach = {_plan(1 << 30, d, k, G).flavour for k, d in WIDE}
    every = {_plan(1 << 30, d, k, G).flavour for k in ("f32", "bf16") for d in range(17, 129)} - {("direct",)}
    assert reach == every, every - reach
    # what sends rows to the direct kernels
    assert _plan(10_000, 8, "f32", G, xp=4).flavour == ("direct",)
    assert _plan(10_000, 8, "f32", G, yp=4).flavour == ("direct",)
    assert _plan(10_000, 8, "f32", G, mp=1).flavour == ("direct",)
    assert _plan(10_000, 64, "f32", G, mp=1).flavour == ("wide", 4, 1)
    assert _plan(10_000, 20, "bf16", G).flavour == ("direct",)            # 40-byte rows
    assert _plan(10_000, 18, "f32", G).flavour == ("direct",)             # d % 4 != 0
    assert _plan(100, 128, "f32", G) == Plan(("wide", 8, 1), 60, 1, 60, 40)
    assert score_launches(_plan(0, 8, "f32", G), 0) == 0 and grad_launches(_plan(0, 8, "f32", G), 0) == 2


@pytest.mark.parametrize("G", [H100_SMS, 114])
def test_row_counts_give_the_tile_counts_claimed(G):
    for kind, d in WIDTHS:
        p = _ring_plan(kind, d, G)
        n = n_long(p.T, p.grid)
        q = _plan(n, d, kind, G)
        tiles = q.whole // q.T
        per_cta = np.bincount(np.arange(tiles) % q.grid, minlength=q.grid)
        assert per_cta.min() >= 18 and per_cta.max() > per_cta.min()          # three laps of six slots, uneven
        assert 0 < q.tail < q.T and q.grid == p.grid
        sizes = n_edge(p.T, p.grid)
        assert sizes[7] // p.T == 6 * p.grid and sizes[8] // p.T == 6 * p.grid + 1   # one lap; the first reuse of slot 0
    if G == H100_SMS:
        assert 4.2e6 < n_long(896, 2 * G) < 4.4e6 and 1.4e5 < n_long(60, G) < 1.5e5
    for d in (1, 5, 8, 12, 13, 16):
        T, per_sm, rpt = nw_geom(d)
        F = NW_FLUSH_ROWS // rpt
        n = n_flush(d, G)
        grid = G * per_sm
        tiles = gram_narrow_main_rows(n, d) // T
        assert n - tiles * T == 7
        per_cta = np.bincount(np.arange(tiles) % grid, minlength=grid)
        # every CTA's lanes fold once mid-run (after F tiles) and once at the end, some CTAs one tile more
        assert F < per_cta.min() < per_cta.max() < 2 * F
        if G == H100_SMS:
            assert (1.8e8 < n < 1.85e8) if narrow_dp(d) <= 8 else (7.0e7 < n < 7.2e7)


def _fault(n, T, bad, how, stale):
    """row order of a pass over n rows with tile `bad` dropped, counted twice or replaced by tile `stale`"""
    idx = np.arange(n)
    tile = idx[bad * T:(bad + 1) * T]
    if how == "dropped":
        return np.delete(idx, tile)
    if how == "twice":
        return np.r_[idx, tile]
    out = idx.copy()
    out[bad * T:(bad + 1) * T] = idx[stale * T:(stale + 1) * T]
    return out


@pytest.mark.parametrize("kind,d", [("f32", 1), ("f32", 16), ("bf16", 72), ("f32", 128)],
                         ids=["f32-d1", "f32-d16", "bf16-d72", "f32-d128"])
def test_bounds_see_the_faults(kind, d):
    G = H100_SMS
    ring = _ring_plan(kind, d, G)
    T, grid = ring.T, ring.grid
    n = n_long(T, grid)
    t = Table(kind, d, n, seed=5 + d, T=T)
    bad = 6 * grid + 5                    # a tile of CTA 5 after its first lap of the six slots
    stale = bad - 6 * grid                # the tile that CTA streamed through the same slot one lap earlier
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    kept = mask == 1
    p = predict_ld(t.Xv, t.coef, B).astype(np.float64)
    S = orc.gram_stats(t.Xv[kept], t.y["y"][kept])
    m = refine_means(S, 1)
    ls = orc.fit_from_stats(S)
    moved = {}
    for ykey in ("y", "yx"):
        y = t.y[ykey]
        want = orc.score_stats(y[kept], p[kept])
        for how in ("dropped", "twice", "stale"):
            r = _fault(n, T, bad, how, stale)
            k = kept[r]
            got = orc.score_stats(y[r][k], p[r][k])
            if how == "stale":                 # the stale slot's rows are counted where the tile's should be
                assert got[5] == want[5]
            moved[f"stats {ykey}", how] = stats_err(got, want) / SCORE_TOL
    # yhat: the stale slot's predictions in the tile's rows
    p32 = p.astype(np.float32)
    got = p32.copy()
    got[bad * T:(bad + 1) * T] = p32[stale * T:(stale + 1) * T]
    moved["yhat ulp", "stale"] = ulps(got, p32) / 1
    # the gradient at the least-squares solution (the smallest g) and at the perturbed model
    for model, (c, b) in {"least squares": (ls["coef"], ls["intercept"]), "perturbed": (t.pcoef, B + 0.5)}.items():
        want, scale = moments_ref(t.Xv[kept], t.y["y"][kept], c, b, m, np.float64)   # fp64: the effects are far larger
        for how in ("dropped", "twice", "stale"):
            r = _fault(n, T, bad, how, stale)
            k = kept[r]
            got, _ = moments_ref(t.Xv[r][k], t.y["y"][r][k], c, b, m, np.float64)
            moved[f"grad {model}", how] = grad_err(got, want, scale) / GRAD_TOL
    small = {k: v for k, v in moved.items() if not v >= 100}
    assert not small, small


@pytest.mark.parametrize("d", [1, 8, 16])
def test_flush_bounds_see_an_accumulator_not_zeroed(d):
    """An accumulator not zeroed at the mid-run flush adds every lane's first interval twice: the rows of the first F
    tiles of every CTA (tiles 0 .. grid F - 1).  At N_FLUSH that is a fixed share of the rows; on rows of the synthetic
    distribution that share moves the raw statistic and oracle.stat_error far beyond their bounds.  (A dropped or doubled
    tile moves the row count S[d, d] by T, which the GPU test asserts exactly.)"""
    G = H100_SMS
    T, per_sm, rpt = nw_geom(d)
    F = NW_FLUSH_ROWS // rpt
    n = n_flush(d, G)
    share = G * per_sm * F * T / n
    assert 0.6 < share < 0.7
    X, y = orc.generate_dataset(200_000, d, seed=d, dtype=np.float32)
    So = orc.gram_stats(X, y)
    k = int(round(share * len(X)))
    S = So + orc.gram_stats(X[:k], y[:k])
    assert rel(S, So) / RAW_TOL >= 100 and max(orc.stat_error(S, So)) / SF_TOL >= 100


@pytest.mark.parametrize("G", [H100_SMS, 114])
@pytest.mark.parametrize("d", [1, 5, 8, 12, 16])
def test_lap_mask_makes_a_stale_narrow_slot_move_the_row_count(d, G):
    """A stale slot of the narrow Gram's ring (the tile its CTA streamed one lap earlier, X, y and mask alike) replaces
    rows by rows of the same distribution: on unmasked rows it moves the raw statistic and oracle.stat_error by far less
    than their bounds, so only the lap-masked runs can see it.  Under lap_mask every tile keeps one row more or one row
    fewer than the tile one lap earlier, so the exact S[d, d] check moves by one row for every stale tile."""
    T, per_sm, _ = nw_geom(d)
    grid = G * per_sm
    lap = 6 * grid
    n = min(n_flush(d, G), T * (3 * lap + 1))          # three laps and one tile: the mask repeats every two laps
    kept = lap_mask(n, d, G)[: n // T * T].reshape(-1, T).sum(axis=1)
    assert set(kept.tolist()) == {T - 1, T - 2}
    assert np.all(kept[lap:] != kept[:-lap])
    assert np.all(np.abs(kept[lap:].astype(int) - kept[:-lap]) == 1)


def test_bf16_rows_bias_the_fp32_chains():
    """Why bf16 rows lose more in the narrow Gram's fp32 chains than fp32 rows (gram_narrow.cu), in a float32 model of
    2048-row chains of v^2, v = x - c, at eight shifts c near the column mean.  Values on the bf16 grid share the low
    bits of -c in every row, so the roundings of a chain have a mean that depends on c and the error of the sum swings
    over orders of magnitude with c; fp32 values have random low bits and round without a mean at every c.  (The worst
    case of any 2048-row fp32 chain is 2047 x 2^-24 = 1.2e-4 relative: the 1e-6 and 2e-5 bounds rest on the roundings
    averaging out across lanes.)"""
    rng = np.random.default_rng(1)
    L, lanes = NW_FLUSH_ROWS, 2048
    x = rng.uniform(0, 100, size=(L, lanes)).astype(np.float32)
    rows = {"f32": x, "bf16": native.from_bf16_bits(native.to_bf16_bits(x))}
    bias, err = defaultdict(list), defaultdict(list)
    for c in rng.uniform(49, 51, 8).astype(np.float32):
        for kind, X in rows.items():
            v = X - c                                       # exact in fp32: the kernel's shifted values
            s2 = np.zeros(lanes, np.float32)
            for i in range(L):
                s2 += v[i] * v[i]
            e = s2.astype(np.float64) - (v.astype(np.float64) ** 2).sum(axis=0)
            bias[kind].append(abs(e.mean()) / e.std())      # the mean rounding against the lane-to-lane spread
            err[kind].append(abs(e.sum()) / (v.astype(np.float64) ** 2).sum())
    assert max(bias["f32"]) < 0.2 and max(err["f32"]) < 1e-7, (bias["f32"], err["f32"])
    assert max(bias["bf16"]) > 1.0 and max(err["bf16"]) > 1e-6, (bias["bf16"], err["bf16"])
    assert max(err["bf16"]) > 100 * min(err["bf16"]), err["bf16"]
