"""The fp64 tensor-core passes on the 32-row tile ring of b2_dmma.cuh that hold a Hessian-sized sum in registers for
the whole launch -- multinomial_kernel (b2_multinomial_pass / b2_multinomial_line_search), svm_kernel (b2_svm_pass) and
class_scatter_kernel (b2_class_scatter) -- at row counts where every CTA walks many tiles: each slot of the three-stage
ring is refilled across several laps, the register-resident accumulators of D = 128 (up to six 16 x 16 blocks per warp)
sum over many tiles, and svm_kernel's staging tile of rows that changed side is carried from tile to tile.

The row counts, layouts and launch rule are test_gpu_tile_passes's (n_long, n_edge, _layouts, _ring, _launches): each
call's launch count must match the flavour _ring predicts, at whole tiles the ring and the direct flavour must return
the same bits (tile_grid gives tile i to the same CTA in both), with a tail they agree within the bound.

  * long runs against the references of the passes' own suites (test_gpu_multinomial._reference /
    _reference_ladder, test_gpu_svm._reference, test_gpu_lda._reference), ring against direct on the same rows;
  * the multinomial class-pair grid: K = 3, 11, 12, 15, 16, 32 (22, 2, 1, 1, 1 and 1 row slices on 132 SMs; 136 and
    528 CTAs of one slice at K = 16 and 32, a second wave);
  * svm_kernel's staging tile on integer rows where sum sigma z z^T is exact: 0, 1, 17, 31 and 32 changed rows per
    tile, 1 and 32 in alternate tiles (33 staged: a flush and one row carried), changed rows only in the last tile of
    each CTA or only in the direct tail; dH equals numpy bit for bit;
  * the within-class scatter on integer rows, dyadic means and dyadic weights: S_w equals numpy bit for bit;
  * the edge row counts, masks that empty whole tiles and whole CTAs (NaN and +-Inf in X and y of every dropped row),
    small calls after large ones through one context (stale per-CTA partials), host rows over three staging blocks;
  * on the CPU, that each bound is at least 100x below what a dropped tile, a tile counted twice or a stale ring slot
    would do to the compared quantity.

Bounds are the passes' suites' PASS_TOL = 1e-13: multinomial loss, gradient, each Hessian block and each ladder step
relative to its largest entry; SVM loss and gradient relative to their largest entry and dH relative to
max |Gram of the active rows| + max |dH|; the scatter per entry relative to sum w |u_i u_j|.  Counts equal.  The longer
chains stay within them.  Worst case over this file, measured on one H100 80GB HBM3 (132 SMs) at a 700 W power limit:
  * multinomial 2.8e-14 (D = 17, K = 16: one row slice, each of 136 CTAs over all 2382 tiles); 1.8e-14 on host rows,
    1.2e-14 over the long runs;
  * SVM 1.5e-14 (host rows, three staging blocks); 1.0e-14 with masks that empty tiles;
  * scatter 2.3e-15 (fp32, D = 20, long run).
The whole file took 200 s there, most of it in the numpy references.  Each GPU test prints the worst case it measured
(run with -s).
"""
import types
from collections import defaultdict

import numpy as np
import pytest

from bodywork_mlops_demo_b200 import _native as native
from test_gpu_lda import PASS_TOL as SCATTER_TOL
from test_gpu_lda import _reference as scatter_reference
from test_gpu_multinomial import PASS_TOL as MN_TOL
from test_gpu_multinomial import _reference as mn_reference
from test_gpu_multinomial import _reference_ladder as mn_reference_ladder
from test_gpu_ridge_classifier_cv import Rows as ClassRows
from test_gpu_ridge_classifier_cv import call as ridge_classifier_loo
from test_gpu_svm import PASS_TOL as SVM_TOL
from test_gpu_svm import _reference as svm_reference
from test_gpu_svm import rel as svm_rel
from test_gpu_tile_passes import (CLASSES, H100_SMS, TILE, WIDTHS, Dev, Layout, Table, _call, _fault_rows, _launches,
                                  _layouts, _ring, _same, _tile_masks, n_edge, n_long, rel, run_classify, run_glm)

DEV = native.MEM_DEVICE
HINGE, EPS = native.SVM_SQUARED_HINGE, native.SVM_SQUARED_EPSILON
STEPS = 21
POS = 7.0                            # Table's positive binary label: the squared hinge's positive label
EPS_PARAM = 0.4
MODES = ("hess", "grad", "ladder")


# ---- data -------------------------------------------------------------------------------------------------------------
def mn_classes(K):
    return CLASSES[K] if K in CLASSES else np.arange(K, dtype=np.float32) * 5 - 20


def add_labels(t, ks, seed, dropped=None):
    """labels of K classes in t.y[f"cls{K}"] (Table has 2, 3 and 32): a few rows of no class, NaN and -inf, the dropped
    rows NaN / +-Inf.  Call before Dev."""
    rng = np.random.default_rng(seed)
    for K in ks:
        if f"cls{K}" in t.y:
            continue
        y = mn_classes(K)[rng.integers(0, K, size=t.n)]
        if t.n > 64:
            y[rng.choice(t.n, 6, replace=False)] = 99.0
            y[rng.choice(t.n, 2, replace=False)] = [np.nan, -np.inf]
        if dropped is not None:
            y[dropped] = np.resize(np.float32([np.nan, np.inf, -np.inf]), int(dropped.sum()))
        t.y[f"cls{K}"] = y


def mn_model(K, d, seed):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(K, d + 1)) * 3.0 / np.sqrt(d), rng.normal(size=(K, d + 1)) * 2.0 / np.sqrt(d)


def svm_model(d, seed):
    """(w0, b0) the accepted point and (w1, b1) the trial point"""
    rng = np.random.default_rng(seed)
    w0 = rng.normal(size=d) * 0.4 / np.sqrt(d)
    return (w0, 0.3), (w0 + rng.normal(size=d) * 0.3 / np.sqrt(d), -0.2)


def scatter_means(t, n, kept, K, seed):
    rng = np.random.default_rng(seed)
    X, y = t.Xv[:n][kept], t.y[f"cls{K}"][:n][kept]
    m = np.array([X[y == c].mean(axis=0) if np.any(y == c) else np.zeros(t.d) for c in CLASSES[K]])
    return m + rng.normal(size=m.shape) * 1e-3


def kept_rows(n, mask, keep):
    return np.ones(n, bool) if mask is None else mask[:n] == keep


# ---- the passes on device rows: (outputs, ring) ----------------------------------------------------------------------
def run_mn(ctx, L, n, masked, K, coef, step, fi, mode, mem=DEV, xp=None, yp=None, mp=None):
    """one multinomial call in `mode` (Hessian, gradient only, ladder); the outputs as the reference's dict"""
    lib, d, cl = native.load(), L.d, mn_classes(K)
    xp = L.xp if xp is None else xp
    yp = L.yp[f"cls{K}"] if yp is None else yp
    mp = L.mask(masked) if mp is None else mp
    args = (ctx._h, xp, L.dt, yp, n, d, d, mem, mp, L.keep, cl.ctypes.data, K, coef.ctypes.data)
    if mode == "ladder":
        lad = np.empty(STEPS)
        launches = _call(ctx, lib.b2_multinomial_line_search, *args, step.ctypes.data, STEPS, lad.ctypes.data)
        got = {"ladder": lad}
    else:
        sums = np.empty(5 + K * (d + 1))
        H = np.empty((K, K, d + 1, d + 1)) if mode == "hess" else None
        launches = _call(ctx, lib.b2_multinomial_pass, *args, int(fi), sums.ctypes.data,
                         None if H is None else H.ctypes.data)
        got = dict(zip(("loss", "kept", "unmatched", "nonfinite", "correct"), sums[:5]))
        got["grad"], got["hessian"] = sums[5:].reshape(K, d + 1), H
    ring = _ring(xp, yp, mp, d, d, L.es)
    if mem == DEV:
        assert launches == _launches(n, ring, 2), (L.name, n, K, mode, launches)
    return got, ring, launches


def mn_ref(t, n, mask, keep, K, coef, step, fi):
    """the multinomial sums and ladder over the kept rows"""
    kept = kept_rows(n, mask, keep)
    X, y, cl = t.Xv[:n][kept], t.y[f"cls{K}"][:n][kept], mn_classes(K)
    d = t.d
    if not kept.any():
        return {"loss": 0.0, "kept": 0.0, "unmatched": 0.0, "nonfinite": 0.0, "correct": 0.0,
                "grad": np.zeros((K, d + 1)), "hessian": np.zeros((K, K, d + 1, d + 1)), "ladder": np.zeros(STEPS)}
    want = mn_reference(X, y, cl, coef, fi, None)
    want["ladder"] = mn_reference_ladder(X, y, cl, coef, step, None)
    return want


def mn_counts(got, want):
    return [k for k in ("kept", "unmatched", "nonfinite", "correct") if k in got and got[k] != want[k]]


def mn_err(got, want):
    """test_gpu_multinomial's comparison: loss, gradient, each Hessian block and each ladder step relative to its largest
    entry"""
    if "ladder" in got:
        return max(rel(got["ladder"][s], want["ladder"][s]) for s in range(STEPS))
    errs = [rel(got["loss"], want["loss"]), rel(got["grad"], want["grad"])]
    H = got.get("hessian")
    if H is not None:
        K = H.shape[0]
        errs += [rel(H[a, c], want["hessian"][a, c]) for a in range(K) for c in range(K)]
    return max(errs)


def mn_check(got, want):
    """counts equal, every Hessian block bitwise symmetric and equal to its mirror, the error within MN_TOL"""
    assert not mn_counts(got, want), mn_counts(got, want)
    H = got.get("hessian")
    if H is not None:
        assert all(np.array_equal(H[a, c], H[a, c].T) and np.array_equal(H[a, c], H[c, a])
                   for a in range(H.shape[0]) for c in range(H.shape[0]))
    err = mn_err(got, want)
    assert err < MN_TOL, err
    return err


def run_svm(ctx, L, n, masked, ykey, loss, frm, to, hess, mem=DEV, xp=None, yp=None, mp=None):
    lib, d = native.load(), L.d
    xp = L.xp if xp is None else xp
    yp = L.yp[ykey] if yp is None else yp
    mp = L.mask(masked) if mp is None else mp
    param = POS if loss == HINGE else EPS_PARAM
    sums = np.empty(d + 8)
    H = np.empty((d + 1, d + 1)) if hess else None
    wf, bf = frm if frm is not None else (None, 0.0)
    w, b = to
    launches = _call(ctx, lib.b2_svm_pass, ctx._h, xp, L.dt, yp, n, d, d, mem, mp, L.keep, loss, float(param),
                     None if wf is None else wf.ctypes.data, float(bf), w.ctypes.data, float(b), 1,
                     sums.ctypes.data, None if H is None else H.ctypes.data)
    ring = _ring(xp, yp, mp, d, d, L.es)
    if mem == DEV:
        assert launches == _launches(n, ring, 2), (L.name, n, hess, launches)
    got = {"loss": sums[0], "counts": sums[1:7], "grad": sums[7:], "dH": H}
    return got, ring, launches


def svm_ref(t, n, mask, keep, ykey, loss, frm, to):
    kept = kept_rows(n, mask, keep)
    wf, bf = frm if frm is not None else (None, 0.0)
    param = POS if loss == HINGE else EPS_PARAM
    return svm_reference(t.Xv[:n], t.y[ykey][:n], loss, param, wf, bf, to[0], to[1], kept)


def svm_err(got, want):
    """test_gpu_svm's comparison: loss and gradient relative to their largest entry, dH relative to max |Gram of the
    active rows| + max |dH|"""
    err = max(svm_rel(got["loss"], want["loss"]), svm_rel(got["grad"], want["grad"]))
    if got["dH"] is not None:
        assert np.array_equal(got["dH"], got["dH"].T)
        err = max(err, svm_rel(got["dH"], want["dH"], scale=np.max(np.abs(want["gram"]), initial=0.0) +
                               np.max(np.abs(want["dH"]), initial=0.0)))
    return err


def svm_check(got, want):
    assert list(got["counts"]) == [float(c) for c in want["counts"]], (got["counts"], want["counts"])
    err = svm_err(got, want)
    assert err < SVM_TOL, err
    return err


def run_scatter(ctx, L, n, masked, K, means, weights, mem=DEV, xp=None, yp=None, mp=None):
    lib, d, cl = native.load(), L.d, CLASSES[K]
    xp = L.xp if xp is None else xp
    yp = L.yp[f"cls{K}"] if yp is None else yp
    mp = L.mask(masked) if mp is None else mp
    S, counts = np.full((d, d), np.nan), np.full(3, np.nan)
    launches = _call(ctx, lib.b2_class_scatter, ctx._h, xp, L.dt, yp, n, d, d, mem, mp, L.keep, cl.ctypes.data, K,
                     means.ctypes.data, None if weights is None else weights.ctypes.data, S.ctypes.data,
                     counts.ctypes.data)
    ring = _ring(xp, yp, mp, d, d, L.es)
    if mem == DEV:
        assert launches == _launches(n, ring, 2), (L.name, n, K, launches)
    return {"S": S, "counts": counts}, ring, launches


def scatter_ref(t, n, mask, keep, K, means, weights):
    S, B, counts = scatter_reference(t.Xv[:n], t.y[f"cls{K}"][:n], kept_rows(n, mask, keep), CLASSES[K], means, weights)
    return {"S": S, "B": B, "counts": counts}


def scatter_err(got, want):
    """test_gpu_lda's comparison: every entry relative to sum w |u_i u_j|"""
    return float(np.max(np.abs(got["S"] - want["S"]) / np.maximum(want["B"], 1e-300))) if want["S"].size else 0.0


def scatter_check(got, want):
    assert list(got["counts"]) == want["counts"], (got["counts"], want["counts"])
    assert np.array_equal(got["S"], got["S"].T)
    err = scatter_err(got, want)
    assert err < SCATTER_TOL, err
    return err


# ---- (1) long runs against the references, ring against direct on the same rows ---------------------------------------
def _long(run, lay, names, n, whole, want, check, ring_rows=True):
    """the pass on the aligned layout at n (against the reference, repeated bit for bit) and at whole tiles, then on
    every other layout: bit-identical at whole tiles, within the bound at n.  ring_rows: the width streams through the
    ring when aligned.  The worst error and the (layout, ring) pairs."""
    base, worst, seen = {}, 0.0, set()
    for nn in (n, whole):
        base[nn], ring = run(lay["ring"], nn)
        assert ring == ring_rows
        assert _same(run(lay["ring"], nn)[0], base[nn]), nn
    worst = check(base[n], want)
    for name in names[1:]:
        for nn in (n, whole):
            other, ring = run(lay[name], nn)
            seen.add((name, ring))
            if nn == whole:
                assert _same(other, base[whole]), (name, ring)
            else:
                worst = max(worst, check(other, want))
    return worst, seen


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", WIDTHS, ids=[f"{k}-d{d}" for k, d in WIDTHS])
def test_long_runs_against_reference_and_ring_against_direct(ctx, kind, d):
    G = ctx.info()["sm_count"]
    n = n_long(G)
    whole = n // TILE * TILE
    t = Table(kind, d, n, seed=700 + 100 * d + (7 if kind == "bf16" else 0))
    add_labels(t, (10,), seed=d)
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    lay = _layouts(dev, with_mask=True)
    worst, rings = defaultdict(float), defaultdict(set)

    def note(group, res):
        worst[group] = max(worst[group], res[0])
        rings[group] |= res[1]

    try:
        for masked in (False, True):
            m = mask if masked else None
            names = ["ring", "x+4", "y+4"] + (["mask+1"] if masked else [])
            # multinomial: K = 3 with an intercept unmasked, K = 10 without one masked, in all three modes
            K, fi = (10, False) if masked else (3, True)
            coef, step = mn_model(K, d, seed=K + d)
            want = mn_ref(t, n, m, 1, K, coef, step, fi)
            for mode in MODES:
                note("multinomial", _long(lambda L, nn: run_mn(ctx, L, nn, masked, K, coef, step, fi, mode)[:2],
                                          lay, names, n, whole, want, mn_check))
            # the SVM pass: both losses, from none and from an accepted point, with and without the Hessian
            w_from, w_to = svm_model(d, seed=d)
            for loss, ykey in ((HINGE, "bin"), (EPS, "reg")):
                for frm in (None, w_from):
                    want = svm_ref(t, n, m, 1, ykey, loss, frm, w_to)
                    for hess in (True, False):
                        note("svm", _long(lambda L, nn: run_svm(ctx, L, nn, masked, ykey, loss, frm, w_to, hess)[:2],
                                          lay, names, n, whole, want, svm_check))
            # the within-class scatter: K = 2 and 32, weights none and random
            for K in (2, 32):
                means = scatter_means(t, n, kept_rows(n, m, 1), K, seed=K)
                for weights in (None, np.random.default_rng(K).uniform(0.1, 3.0, size=K)):
                    want = scatter_ref(t, n, m, 1, K, means, weights)
                    note("scatter", _long(lambda L, nn: run_scatter(ctx, L, nn, masked, K, means, weights)[:2],
                                          lay, names, n, whole, want, scatter_check))
    finally:
        dev.free()
    # X or y off its 16-byte boundary never takes the ring; a misaligned mask only for d > 16
    for pas, seen in rings.items():
        for name, ring in seen:
            assert ring == (name == "mask+1" and d > 16), (pas, name, ring)
    print(f"\n[long {kind} d={d}, n={n}, G={G}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (2) the multinomial class-pair grid -----------------------------------------------------------------------------
PAIR_CASES = [(d, K) for d in (17, 128) for K in (3, 11, 12, 15, 16, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("d,K", PAIR_CASES, ids=[f"d{d}-K{K}" for d, K in PAIR_CASES])
def test_multinomial_class_pair_grid(ctx, d, K):
    """slices x K (K + 1) / 2 pairs: K = 3 and 11 give several row slices, K >= 12 one slice whose CTAs each walk every
    tile (K = 16 and 32: more CTAs than SMs).  D = 17 rows (68 bytes) take the direct flavour in every layout.  The
    reference costs K^2 d^2 n, so at D = 128 the K >= 12 cases, where one slice walks every tile at any n, run 41 tiles
    and a tail."""
    G = ctx.info()["sm_count"]
    n = n_long(G) if d == 17 or K < 12 else TILE * 41 + 17
    whole = n // TILE * TILE
    pairs = K * (K + 1) // 2
    slices = min(-(-n // TILE), max(G // pairs, 1))
    t = Table("f32", d, n, seed=900 + K + d)
    add_labels(t, (K,), seed=K)
    mask = (np.arange(n) % 7 != 3).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    lay = _layouts(dev, with_mask=False)
    coef, step = mn_model(K, d, seed=K * d)
    worst = 0.0
    try:
        for masked, fi in ((False, True), (True, False)):
            m = mask if masked else None
            want = mn_ref(t, n, m, 1, K, coef, step, fi)
            for mode in MODES:
                res = _long(lambda L, nn: run_mn(ctx, L, nn, masked, K, coef, step, fi, mode)[:2], lay,
                            ["ring", "x+4"], n, whole, want, mn_check, ring_rows=d % 4 == 0)
                worst = max(worst, res[0])
    finally:
        dev.free()
    print(f"\n[class pairs d={d} K={K}, n={n}, {slices} slice(s) x {pairs} pairs] worst {worst:.2e}")


# ---- (3) svm_kernel's staging tile, exact --------------------------------------------------------------------------
def _exact_svm_rows(n, d, changed, seed):
    """integer rows in [-3, 3] whose last feature c is +1 (enters: active at `to` only), -1 (leaves) or 0 (active at
    both) for the squared hinge at label +1, from w_from = (2^-9 s, +4) to w_to = (2^-9 s', -4), no intercept: every
    eta, and every sum of sigma z z^T, is exact in fp64"""
    rng = np.random.default_rng(seed)
    X = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    sign = np.where(rng.uniform(size=n) < 0.5, 1.0, -1.0)
    X[:, d - 1] = np.where(changed, sign, 0.0)
    small = lambda: np.r_[rng.integers(-1, 2, size=d - 1) / 512.0, 0.0]   # |x . small| <= 3 (d - 1) / 512 < 1
    wf, wt = small(), small()
    wf[d - 1], wt[d - 1] = 4.0, -4.0
    return X, (wf, 0.0), (wt, 0.0)


def _staging_patterns(n, G):
    idx = np.arange(n)
    tile, r = idx // TILE, idx % TILE
    whole_tiles = n // TILE
    last = tile >= whole_tiles - min(whole_tiles, G)          # the last tile of each CTA of the ring launch (Hessian)
    return {"none": np.zeros(n, bool), "1 per tile": r == 7, "17 per tile": r < 17, "31 per tile": r != 0,
            "every row": np.ones(n, bool), "1 and 32 in alternate tiles": (tile % 2 == 1) | (r == 3),
            "last tile of each CTA": last & (tile < whole_tiles), "direct tail only": tile >= whole_tiles}


@pytest.mark.gpu
@pytest.mark.parametrize("d", [8, 128])
def test_svm_staging_tile_exact(ctx, d):
    G = ctx.info()["sm_count"]
    n = n_long(G)
    t = Table("f32", d, n, seed=40 + d)
    y = np.ones(n, np.float32)
    patterns = _staging_patterns(n, G)
    for label, changed in patterns.items():
        X, frm, to = _exact_svm_rows(n, d, changed, seed=d)
        t.up, t.Xv, t.y = X, X.astype(np.float64), {"one": y}
        want = svm_reference(t.Xv, y, HINGE, 1.0, frm[0], 0.0, to[0], 0.0, np.ones(n, bool))
        enter, leave = int(np.sum(changed & (X[:, d - 1] > 0))), int(np.sum(changed & (X[:, d - 1] < 0)))
        assert (want["counts"][2], want["counts"][3]) == (enter, leave), label
        dev = Dev(ctx, t, None)
        lay = _layouts(dev, with_mask=False)
        try:
            for name in ("ring", "x+4"):
                L = lay[name]
                sums, H = np.empty(d + 8), np.empty((d + 1, d + 1))
                launches = _call(ctx, native.load().b2_svm_pass, ctx._h, L.xp, L.dt, L.yp["one"], n, d, d, DEV, None,
                                 1, HINGE, 1.0, frm[0].ctypes.data, 0.0, to[0].ctypes.data, 0.0, 1, sums.ctypes.data,
                                 H.ctypes.data)
                assert launches == _launches(n, name == "ring", 2)
                svm_check({"loss": sums[0], "counts": sums[1:7], "grad": sums[7:], "dH": H}, want)
                assert np.array_equal(H, want["dH"]), (label, name, float(np.max(np.abs(H - want["dH"]))))
        finally:
            dev.free()
    print(f"\n[svm staging d={d}, n={n}] dH bit-identical to numpy in {len(patterns)} patterns x 2 layouts")


# ---- (4) the within-class scatter, exact ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_scatter_exact(ctx):
    """integer rows, means in quarters and weights in quarters: every u, w u and sum w u u^T is exact in fp64"""
    G = ctx.info()["sm_count"]
    n, d, K = n_long(G), 128, 32
    t = Table("f32", d, n, seed=61)
    rng = np.random.default_rng(61)
    X = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    t.up, t.Xv = X, X.astype(np.float64)
    means = rng.integers(-4, 5, size=(K, d)) / 4.0
    weights = rng.integers(1, 8, size=K) / 4.0
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    lay = _layouts(dev, with_mask=False)
    try:
        for masked in (False, True):
            m = mask if masked else None
            want = scatter_ref(t, n, m, 1, K, means, weights)
            for name in ("ring", "x+4"):
                got, ring, _ = run_scatter(ctx, lay[name], n, masked, K, means, weights)
                assert ring == (name == "ring")
                assert list(got["counts"]) == want["counts"]
                assert np.array_equal(got["S"], want["S"]), (name, masked, float(np.max(np.abs(got["S"] - want["S"]))))
    finally:
        dev.free()
    print(f"\n[scatter exact d={d} K={K}, n={n}] S_w bit-identical to numpy")


# ---- (5) edge row counts --------------------------------------------------------------------------------------------
def _all_passes(ctx, t, L, n, masked, m, keep, worst, ring_expected=None):
    """every pass of this file on one layout: multinomial K = 3 in its three modes, the squared hinge from an accepted
    point with and without the Hessian, the scatter at K = 32 with weights; each against its reference"""
    d = t.d
    coef, step = mn_model(3, d, seed=d)
    want = mn_ref(t, n, m, keep, 3, coef, step, True)
    outs = []
    for mode in MODES:
        got, ring, _ = run_mn(ctx, L, n, masked, 3, coef, step, True, mode)
        worst["multinomial"] = max(worst["multinomial"], mn_check(got, want))
        outs.append((ring, got))
    w_from, w_to = svm_model(d, seed=d)
    want = svm_ref(t, n, m, keep, "bin", HINGE, w_from, w_to)
    for hess in (True, False):
        got, ring, _ = run_svm(ctx, L, n, masked, "bin", HINGE, w_from, w_to, hess)
        worst["svm"] = max(worst["svm"], svm_check(got, want))
        outs.append((ring, got))
    means = scatter_means(t, n, kept_rows(n, m, keep), 32, seed=5)
    weights = np.random.default_rng(5).uniform(0.1, 3.0, size=32)
    want = scatter_ref(t, n, m, keep, 32, means, weights)
    got, ring, _ = run_scatter(ctx, L, n, masked, 32, means, weights)
    worst["scatter"] = max(worst["scatter"], scatter_check(got, want))
    outs.append((ring, got))
    for ring, got in outs:
        assert ring_expected is None or ring == ring_expected
        for k, v in got.items():
            assert v is None or np.all(np.isfinite(v)), k
    return outs


EDGES = [("f32", 8), ("f32", 128), ("bf16", 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d", EDGES, ids=[f"{k}-d{d}" for k, d in EDGES])
def test_edge_row_counts(ctx, kind, d):
    G = ctx.info()["sm_count"]
    sizes = n_edge(G)
    t = Table(kind, d, max(sizes), seed=800 + d)
    mask = (np.arange(t.n) % 7 != 3).astype(np.uint8)
    dev = Dev(ctx, t, mask)
    L = Layout(dev, "ring")
    worst = defaultdict(float)
    try:
        for n in sizes:
            for masked in (False, True):
                m = mask[:n] if masked else None
                outs = _all_passes(ctx, t, L, n, masked, m, 1, worst)
                if n == 0:         # no rows: zero sums, Hessian, ladder and counts
                    for _, got in outs:
                        for k, v in got.items():
                            assert v is None or not np.any(v), (k, v)
    finally:
        dev.free()
    print(f"\n[edges {kind} d={d}, n in {sizes}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (6) masks that empty whole tiles and whole CTAs ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("d", [8, 64])
def test_masks_that_empty_tiles(ctx, d):
    G = ctx.info()["sm_count"]
    n = n_long(G)
    worst = defaultdict(float)
    for label, mask, keep in _tile_masks(n, G):
        kept = mask == keep
        t = Table("f32", d, n, seed=500 + d, dropped=~kept)
        dev = Dev(ctx, t, mask, keep)
        lay = _layouts(dev, with_mask=False)
        try:
            for name in ("ring", "x+4"):
                _all_passes(ctx, t, lay[name], n, True, mask, keep, worst, ring_expected=name == "ring")
        finally:
            dev.free()
    print(f"\n[tile masks f32 d={d}, n={n}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (7) small calls after large ones through one context ------------------------------------------------------------
@pytest.mark.gpu
def test_small_calls_after_large_ones(ctx):
    """mn_part only grows and glm_part is shared, at different pitches, by the SVM, GLM, logistic, classify and
    leave-one-out passes: a smaller call must write every entry its reduce reads"""
    G = ctx.info()["sm_count"]
    n_big, n_small = TILE * 5 + 17, n_long(G)
    big = Table("f32", 128, max(n_big, TILE * (3 * G + 1)), seed=31)
    small = Table("f32", 8, n_small, seed=32)
    mask = (np.arange(n_small) % 5 != 2).astype(np.uint8)
    dbig, dsmall = Dev(ctx, big, None), Dev(ctx, small, mask)
    Lb, Ls = Layout(dbig, "ring"), Layout(dsmall, "ring")
    rows = ClassRows("f32", 96, TILE * (3 * G + 1), 3, seed=33)
    drows = Dev(ctx, rows, rows.mask)
    worst = defaultdict(float)
    try:
        # multinomial: K = 32 at D = 128 with the Hessian, then K = 3 at D = 8 in every mode
        coef, step = mn_model(32, 128, seed=1)
        got, _, _ = run_mn(ctx, Lb, n_big, False, 32, coef, step, True, "hess")
        worst["multinomial"] = mn_check(got, mn_ref(big, n_big, None, 1, 32, coef, step, True))
        coef, step = mn_model(3, 8, seed=2)
        for masked in (False, True):
            want = mn_ref(small, n_small, mask if masked else None, 1, 3, coef, step, True)
            for mode in MODES:
                got, _, _ = run_mn(ctx, Ls, n_small, masked, 3, coef, step, True, mode)
                worst["multinomial"] = max(worst["multinomial"], mn_check(got, want))
        # scatter: K = 32 at D = 128, then K = 2 at D = 8
        n_sc = big.n
        means = scatter_means(big, n_sc, np.ones(n_sc, bool), 32, seed=3)
        got, _, _ = run_scatter(ctx, Lb, n_sc, False, 32, means, None)
        worst["scatter"] = scatter_check(got, scatter_ref(big, n_sc, None, 1, 32, means, None))
        means = scatter_means(small, n_small, mask == 1, 2, seed=4)
        got, _, _ = run_scatter(ctx, Ls, n_small, True, 2, means, None)
        worst["scatter"] = max(worst["scatter"], scatter_check(got, scatter_ref(small, n_small, mask, 1, 2, means,
                                                                                None)))
        # the SVM pass with the Hessian after every other writer of glm_part at a larger d
        w_from, w_to = svm_model(8, seed=8)
        want = svm_ref(small, n_small, mask, 1, "bin", HINGE, w_from, w_to)
        writers = [lambda: run_glm(ctx, big, Lb, big.n, False, "log p=1.5"),
                   lambda: run_classify(ctx, big, Lb, big.n, False, 32, True),
                   lambda: ridge_classifier_loo(ctx, Layout(drows, "ring"), rows, rows.n,
                                                np.array([0.1, 1.0, 10.0]), True)]
        for write in writers:
            write()
            got, _, _ = run_svm(ctx, Ls, n_small, True, "bin", HINGE, w_from, w_to, True)
            worst["svm"] = max(worst["svm"], svm_check(got, want))
    finally:
        for dv in (dbig, dsmall, drows):
            dv.free()
    print("\n[small after large] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (8) host rows across staging blocks ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_host_rows(ctx):
    """three staging blocks of 262 144 rows and a tail at D = 128 with a mask, from pageable host memory: each block
    is one call of the device launcher, so the launches are those of each block's rows"""
    d, n, blk = 128, 2 * (1 << 18) + 4321, 1 << 18
    t = Table("f32", d, n, seed=88)
    mask = (np.arange(n) % 7 != 3).astype(np.uint8)
    kept = mask == 1
    L = types.SimpleNamespace(d=d, dt=t.dt, es=t.es, keep=1, name="host", xp=t.up.ctypes.data,
                              mask=lambda masked: mask.ctypes.data)
    host = dict(mem=native.MEM_HOST, xp=t.up.ctypes.data, mp=mask.ctypes.data)
    launches = sum(_launches(min(blk, n - r0), True, 2) for r0 in range(0, n, blk))
    worst = {}
    coef, step = mn_model(3, d, seed=3)
    want = mn_ref(t, n, mask, 1, 3, coef, step, True)
    worst["multinomial"] = 0.0
    for mode in MODES:
        got, _, nl = run_mn(ctx, L, n, True, 3, coef, step, True, mode, yp=t.y["cls3"].ctypes.data, **host)
        assert nl == launches, (mode, nl, launches)
        worst["multinomial"] = max(worst["multinomial"], mn_check(got, want))
    w_from, w_to = svm_model(d, seed=d)
    want = svm_ref(t, n, mask, 1, "bin", HINGE, w_from, w_to)
    got, _, nl = run_svm(ctx, L, n, True, "bin", HINGE, w_from, w_to, True, yp=t.y["bin"].ctypes.data, **host)
    assert nl == launches
    worst["svm"] = svm_check(got, want)
    means = scatter_means(t, n, kept, 32, seed=9)
    weights = np.random.default_rng(9).uniform(0.1, 3.0, size=32)
    got, _, nl = run_scatter(ctx, L, n, True, 32, means, weights, yp=t.y["cls32"].ctypes.data, **host)
    assert nl == launches
    worst["scatter"] = scatter_check(got, scatter_ref(t, n, mask, 1, 32, means, weights))
    print(f"\n[host rows, 3 staging blocks, d={d}] worst: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---- (9) the bounds see the faults this file targets (CPU) ----------------------------------------------------------
def _faults(n, grid):
    """the row order of the pass with one tile dropped, counted twice, or replaced by the tile its CTA streamed through
    the same ring slot three tiles earlier (grid: the CTAs that stride over the tiles)"""
    bad = 3 * grid + 5
    stale = np.arange(n)
    stale[bad * TILE:(bad + 1) * TILE] = np.arange((bad - 3 * grid) * TILE, (bad - 3 * grid + 1) * TILE)
    return {"dropped": _fault_rows(n, bad, "dropped"), "twice": _fault_rows(n, bad, "twice"), "stale": stale}


def _view(t, r):
    f = Table.__new__(Table)
    f.__dict__.update(t.__dict__)
    f.Xv, f.y, f.n = t.Xv[r], {k: v[r] for k, v in t.y.items()}, len(r)
    return f


@pytest.mark.parametrize("G", [H100_SMS, 114])
def test_bounds_see_the_faults(G):
    n, d = n_long(G), 16
    t = Table("f32", d, n, seed=5)
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    moved = {}
    coef, step = mn_model(3, d, seed=1)
    w_from, w_to = svm_model(d, seed=2)
    means = scatter_means(t, n, mask == 1, 32, seed=3)
    weights = np.random.default_rng(3).uniform(0.1, 3.0, size=32)
    mn_want = mn_ref(t, n, mask, 1, 3, coef, step, True)
    svm_want = {loss: svm_ref(t, n, mask, 1, ykey, loss, w_from, w_to) for loss, ykey in ((HINGE, "bin"),
                                                                                          (EPS, "reg"))}
    sc_want = scatter_ref(t, n, mask, 1, 32, means, weights)
    # the CTAs striding over the tiles: multinomial one per SM (gradient, ladder) and G // 6 slices (Hessian at K = 3),
    # the SVM pass two per SM without the Hessian and one with it, the scatter one per SM
    for grid in sorted({G, G // 6, 2 * G}):
        for how, r in _faults(n, grid).items():
            f = _view(t, r)
            fm = mask[r]
            got = mn_ref(f, f.n, fm, 1, 3, coef, step, True)
            moved["multinomial sums", grid, how] = mn_err({k: got[k] for k in ("loss", "grad", "hessian")},
                                                          mn_want) / MN_TOL
            moved["multinomial ladder", grid, how] = mn_err({"ladder": got["ladder"]}, mn_want) / MN_TOL
            for loss, ykey in ((HINGE, "bin"), (EPS, "reg")):
                moved[f"svm {loss}", grid, how] = svm_err(svm_ref(f, f.n, fm, 1, ykey, loss, w_from, w_to),
                                                          svm_want[loss]) / SVM_TOL
            moved["scatter", grid, how] = scatter_err(scatter_ref(f, f.n, fm, 1, 32, means, weights),
                                                      sc_want) / SCATTER_TOL
    small = {k: v for k, v in moved.items() if not v >= 100}
    assert not small, small
    # the exact designs: any fault changes the sum
    X, frm, to = _exact_svm_rows(n, d, _staging_patterns(n, G)["1 per tile"], seed=d)
    y = np.ones(n)
    ex = svm_reference(X.astype(np.float64), y, HINGE, 1.0, frm[0], 0.0, to[0], 0.0, np.ones(n, bool))["dH"]
    rng = np.random.default_rng(6)
    Xs = rng.integers(-3, 4, size=(n, d)).astype(np.float64)
    ys = t.y["cls32"]
    sm, sw = rng.integers(-4, 5, size=(32, d)) / 4.0, rng.integers(1, 8, size=32) / 4.0
    sc = scatter_reference(Xs, ys, mask == 1, CLASSES[32], sm, sw)[0]
    for grid in sorted({G, 2 * G}):
        for how, r in _faults(n, grid).items():
            dH = svm_reference(X[r].astype(np.float64), y[r], HINGE, 1.0, frm[0], 0.0, to[0], 0.0,
                               np.ones(len(r), bool))["dH"]
            assert not np.array_equal(dH, ex), (grid, how)
            assert not np.array_equal(scatter_reference(Xs[r], ys[r], mask[r] == 1, CLASSES[32], sm, sw)[0], sc)
