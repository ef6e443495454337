"""LogisticRegression on the H100: the passes (b2_logistic_pass, b2_logistic_line_search) against scikit-learn's
HalfBinomialLoss on float64 copies of the same rounded rows, on every row layout and with eta in every branch of
log1pexp; b2_label_scan and b2_logistic_predict against numpy; the estimator against scikit-learn's
LogisticRegression(solver="newton-cholesky") on float64 copies of the rows.  Each test prints the worst case it measured
(run with -s).

Bounds:
  * the pass sums (loss, gradient, Hessian, every ladder entry), relative to the largest entry of each: 3e-14, the bound
    of the GLM passes (the same row loop and reduce); the counts are equal and repeated calls bit-identical;
  * decision against a correctly rounded dot product: 4e-16 relative to the largest entry; probabilities against
    scipy's expit of the returned decision: 4e-16; against expit of the exact dot product they inherit eta's error
    through dp/deta = p (1 - p) <= 1/4 (up to 2.2e-15 measured at |eta| ~ 70); labels equal wherever |eta| > 1e-9;
  * the estimator against scikit-learn, 16 384 x 24: coef_ / intercept_ relative 1.8e-14 (the GLM estimators' bound),
    equal n_iter_, the same warnings, score equal to accuracy_score.
"""
import io
import math
import warnings

import joblib
import numpy as np
import pytest
from scipy.special import expit
from sklearn import linear_model
from sklearn.metrics import accuracy_score

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from test_logistic_driver import LABELS, NumpyLogisticContext, make_data

pytestmark = pytest.mark.gpu

E_ARG, E_UNSUPPORTED = -1, -6
PASS_TOL = 3e-14
PRED_TOL = 4e-16
COEF_TOL = 1.8e-14
REF = NumpyLogisticContext()
NEG, POS = 3.0, 7.0


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def _rows(n, d, seed, kind):
    """(stored rows with 3 spare columns, their float64 values, y (labels 3 / 7, a few others), coef, b, step)"""
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d + 3)) * 0.5).astype(np.float32)
    up = b2.native.to_bf16_bits(X) if kind == "bf16" else X
    Xv = b2.native.from_bf16_bits(up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
    coef = rng.normal(size=d)
    coef *= 30.0 / np.linalg.norm(coef)             # eta ~ N(0.5, 15): every branch of log1pexp, |eta| > 40 included
    eta = Xv[:, :d] @ coef + 0.5
    y = np.where(rng.uniform(size=n) < expit(eta), POS, NEG).astype(np.float32)
    y[[11, 12]] = 5.0                                # neither label
    y[13] = np.nan
    y[14] = np.inf
    step = rng.normal(size=d) * 2.0 / np.sqrt(d)
    return up, Xv, y, coef, 0.5, step


def _raw_pass(ctx, ptr, dt, yp, n, d, ldx, mk, mp, coef, b, hess):
    sums = np.empty(d + 9)
    H = np.empty((d + 1, d + 1)) if hess else None
    rc = native.load().b2_logistic_pass(ctx._h, ptr, dt, yp, n, d, ldx, mk, mp, 1, NEG, POS, coef.ctypes.data, b, 1,
                                        sums.ctypes.data, H.ctypes.data if hess else None)
    assert rc == 0, native.last_error()
    return sums, H


def _raw_ladder(ctx, ptr, dt, yp, n, d, ldx, mk, mp, coef, b, step, db):
    out = np.empty(21)
    rc = native.load().b2_logistic_line_search(ctx._h, ptr, dt, yp, n, d, ldx, mk, mp, 1, NEG, POS, coef.ctypes.data,
                                               b, step.ctypes.data, db, 21, out.ctypes.data)
    assert rc == 0, native.last_error()
    return out


def _check_sums(sums, H, want, d):
    got = dict(zip(("loss", "const", "sum_y", "kept", "y_out_of_range", "h_nonpos", "y_nonfinite"), sums[:7]))
    got["correct"] = sums[8 + d]
    for k in ("sum_y", "kept", "y_out_of_range", "h_nonpos", "y_nonfinite", "correct"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert got["const"] == 0.0
    errs = [rel(got["loss"], want["loss"]), rel(sums[7:8 + d], want["grad"])]
    if H is not None:
        assert np.array_equal(H, H.T)
        errs.append(rel(H, want["hessian"]))
    return max(errs)


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128])
def test_pass_sums_every_layout(ctx, kind, d):
    n = 4133                                         # ring tiles, then a partial tile on the direct kernel
    up, Xv, y, coef, b, step = _rows(n, d, 20 + d, kind)
    eta = Xv[:, :d] @ coef + b
    for lo, hi in ((-np.inf, -37), (-37, -2), (-2, 18), (18, 33.3), (40, np.inf)):
        assert np.any((eta > lo) & (eta <= hi)), (lo, hi)
    dt = b2.BF16 if kind == "bf16" else b2.F32
    es = 2 if kind == "bf16" else 4
    mask = (np.arange(n) % 5 != 2).astype(np.uint8)
    cont = np.ascontiguousarray(up[:, :d])
    Xd, yd, md = ctx.to_device(cont, kind), ctx.to_device(y), ctx.to_device(mask)
    Xs = ctx.to_device(np.ascontiguousarray(up), kind)         # ldx = d + 3, starting one element in
    worst = 0.0
    try:
        layouts = [("host", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, None, Xv[:, :d], None),
                   ("device", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, None, Xv[:, :d], None),
                   ("strided", Xs.ptr + es, yd.ptr, d + 3, native.MEM_DEVICE, None, Xv[:, 1:d + 1], None),
                   ("device masked", Xd.ptr, yd.ptr, d, native.MEM_DEVICE, md.ptr, Xv[:, :d], mask),
                   ("host masked", cont.ctypes.data, y.ctypes.data, d, native.MEM_HOST, mask.ctypes.data, Xv[:, :d],
                    mask)]
        for name, xp, yp, ldx, mk, mp, Xref, mref in layouts:
            want = REF.logistic_pass(Xref, y, coef, b, NEG, POS, row_mask=mref, hessian=True)
            sums, H = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, coef, b, True)
            err = _check_sums(sums, H, want, d)
            sums2, H2 = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, coef, b, True)
            assert np.array_equal(sums, sums2) and np.array_equal(H, H2), name
            sums3, _ = _raw_pass(ctx, xp, dt, yp, n, d, ldx, mk, mp, coef, b, False)
            assert np.array_equal(sums, sums3), name      # the Hessian does not touch the other sums
            lw = REF.logistic_line_search(Xref, y, coef, b, step, -0.3, NEG, POS, row_mask=mref)
            ladder = _raw_ladder(ctx, xp, dt, yp, n, d, ldx, mk, mp, coef, b, step, -0.3)
            assert np.array_equal(ladder, _raw_ladder(ctx, xp, dt, yp, n, d, ldx, mk, mp, coef, b, step, -0.3))
            err = max(err, max(rel(ladder[k], lw[k]) for k in range(21)))
            assert err < PASS_TOL, (name, err)
            worst = max(worst, err)
    finally:
        for a in (Xd, yd, md, Xs):
            a.free()
    print(f"\n[logistic pass {kind} d={d}] worst relative difference {worst:.2e}")


def _np_scan(y, mask, keep):
    k = y if mask is None else y[mask == keep]
    fin = k[np.isfinite(k)]
    lo, hi = (float(fin.min()), float(fin.max())) if fin.size else (np.nan, np.nan)
    return [float(k.size), float(np.sum(~np.isfinite(k))), float(np.sum(fin != np.rint(fin))), lo, hi,
            float(np.sum(k == lo)), float(np.sum(k == hi))]


def test_label_scan_matches_numpy(ctx):
    rng = np.random.default_rng(3)
    n = 1_000_003
    cases = {"two": rng.choice(np.float32([-1.0, 4.0]), n), "one": np.full(n, 2.0, np.float32),
             "three": rng.choice(np.float32([0.0, 1.0, 2.0]), n),
             "continuous": rng.normal(size=n).astype(np.float32), "negative zero": rng.choice(np.float32([-0.0, 1.0]), n)}
    special = cases["two"].copy()
    special[[5, 77]] = np.nan
    special[900] = np.inf
    special[901] = -np.inf
    special[902] = 2.5
    cases["nan inf fraction"] = special
    cases["all nan"] = np.full(100, np.nan, np.float32)
    mask = (np.arange(n) % 7 != 3).astype(np.uint8)
    for name, y in cases.items():
        yd = ctx.to_device(y)
        m = mask[:y.size]
        md = ctx.to_device(m)
        try:
            for mk, keep in ((None, 1), (m, 1), (m, 0)):
                got = ctx.label_scan(yd, md if mk is not None else None, keep)
                want = _np_scan(y, mk, keep)
                got = [got[k] for k in ("kept", "nonfinite", "nonintegral", "min", "max", "n_min", "n_max")]
                assert np.array_equal(np.array(got), np.array(want), equal_nan=True), (name, keep, got, want)
        finally:
            yd.free(); md.free()
    empty, none = ctx.to_device(np.zeros(4, np.float32)), ctx.to_device(np.zeros(4, np.uint8))
    try:
        st = ctx.label_scan(empty, none, 1)
        assert st["kept"] == 0 and np.isnan(st["min"]) and st["n_min"] == 0
    finally:
        empty.free(); none.free()


@pytest.mark.parametrize("kind", ["f32", "bf16"])
@pytest.mark.parametrize("d", [1, 8, 33, 128])
def test_predict_every_layout(ctx, kind, d):
    n = 300_007                                      # host rows: two staging blocks and a tail
    up, Xv, _, coef, b, _ = _rows(n, d, 40 + d, kind)
    dt = b2.BF16 if kind == "bf16" else b2.F32
    es = 2 if kind == "bf16" else 4
    cont = np.ascontiguousarray(up[:, :d])
    Xd = ctx.to_device(cont, kind)
    Xs = ctx.to_device(np.ascontiguousarray(up), kind)
    lib = native.load()
    worst = 0.0
    try:
        for name, xp, ldx, mk, Xref in (("host", cont.ctypes.data, d, native.MEM_HOST, Xv[:, :d]),
                                        ("device", Xd.ptr, d, native.MEM_DEVICE, Xv[:, :d]),
                                        ("strided", Xs.ptr + es, d + 3, native.MEM_DEVICE, Xv[:, 1:d + 1])):
            eta = np.array([math.fsum(r) for r in Xref * coef]) + b if d > 1 else Xref[:, 0] * coef[0] + b
            p = expit(eta)
            if mk == native.MEM_HOST:
                dec, pr, lab = np.empty(n), np.empty((n, 2)), np.empty(n, np.float32)
                ptrs = (dec.ctypes.data, pr.ctypes.data, lab.ctypes.data)
            else:
                bufs = (ctx.empty((n,), "f64"), ctx.empty((n, 2), "f64"), ctx.empty((n,), "f32"))
                ptrs = tuple(a.ptr for a in bufs)
            rc = lib.b2_logistic_predict(ctx._h, xp, dt, n, d, ldx, mk, coef.ctypes.data, b, NEG, POS, *ptrs)
            assert rc == 0, native.last_error()
            if mk != native.MEM_HOST:
                dec, pr, lab = (a.to_host() for a in bufs)
                for a in bufs:
                    a.free()
            q = expit(dec)
            err = max(rel(dec, eta), rel(pr, np.stack([1 - q, q], axis=1)))
            bound = 0.25 * PRED_TOL * np.max(np.abs(eta)) + PRED_TOL
            assert rel(pr, np.stack([1 - p, p], axis=1)) < bound, name
            sure = np.abs(eta) > 1e-9
            assert np.array_equal(lab[sure], np.where(eta > 0, POS, NEG).astype(np.float32)[sure]), name
            assert err < PRED_TOL, (name, err)
            worst = max(worst, err)
        only = ctx.logistic_predict(cont[:1000], coef, b, proba=True)            # one output alone
        assert list(only) == ["proba"] and only["proba"].shape == (1000, 2)
    finally:
        Xd.free(); Xs.free()
    print(f"\n[logistic predict {kind} d={d}] worst relative difference {worst:.2e}")


CASES = [dict(C=C, fit_intercept=fi) for C in (1e-2, 1.0, 1e4, np.inf) for fi in (True, False)]


def _fit_both(ctx, X, y, **kw):
    ours = b2.B200LogisticRegression(ctx=ctx, **kw)
    ref = linear_model.LogisticRegression(solver="newton-cholesky", **kw)
    with warnings.catch_warnings(record=True) as w_ours:
        warnings.simplefilter("always")
        ours.fit(X.astype(np.float32), y)
    with warnings.catch_warnings(record=True) as w_ref:
        warnings.simplefilter("always")
        ref.fit(X, y)
    assert [w.category for w in w_ours] == [w.category for w in w_ref]
    assert np.array_equal(ours.n_iter_, ref.n_iter_) and np.array_equal(ours.classes_, ref.classes_)
    return ours, ref


@pytest.mark.parametrize("kw", CASES, ids=[f"C={c['C']}-intercept={c['fit_intercept']}" for c in CASES])
def test_estimator_matches_sklearn(ctx, kw):
    X, t = make_data(n=16_384, d=24, seed=7)
    ours, ref = _fit_both(ctx, X, t, **kw)
    err = rel(np.r_[ours.coef_[0], ours.intercept_], np.r_[ref.coef_[0], ref.intercept_])
    assert err < COEF_TOL, err
    X32 = X.astype(np.float32)
    assert np.array_equal(ours.predict(X32), ref.predict(X))
    perr = rel(ours.predict_proba(X32), ref.predict_proba(X))
    assert perr < COEF_TOL, perr
    assert ours.score(X32, t) == accuracy_score(t, ref.predict(X))
    print(f"\n[logistic {kw}] n_iter {ours.n_iter_[0]}, coef {err:.2e}, proba {perr:.2e}")


@pytest.mark.parametrize("labels", list(LABELS), ids=list(LABELS))
def test_labels_masks_warm_start_and_joblib(ctx, labels):
    X, t = make_data(n=16_384, d=24, seed=8)
    y = LABELS[labels][t]
    mask = (np.arange(len(t)) % 4 != 1).astype(np.uint8)
    X32 = X.astype(np.float32)
    Xn = X32.copy()
    Xn[mask == 0, 3] = np.nan
    ref = linear_model.LogisticRegression(solver="newton-cholesky").fit(X[mask == 1], y[mask == 1])
    ours = b2.B200LogisticRegression(ctx=ctx).fit(Xn, y, row_mask=mask)
    err = rel(np.r_[ours.coef_[0], ours.intercept_], np.r_[ref.coef_[0], ref.intercept_])
    assert np.array_equal(ours.n_iter_, ref.n_iter_) and err < COEF_TOL, err
    assert np.array_equal(ours.classes_, ref.classes_)
    assert ours.score(Xn, y, row_mask=mask) == accuracy_score(y[mask == 1], ref.predict(X[mask == 1]))
    # warm start from a two-iteration fit
    w_ours = b2.B200LogisticRegression(ctx=ctx, warm_start=True, max_iter=2, C=10.0)
    w_ref = linear_model.LogisticRegression(solver="newton-cholesky", warm_start=True, max_iter=2, C=10.0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        w_ours.fit(X32, y)
        w_ref.fit(X, y)
    w_ours.max_iter = w_ref.max_iter = 100
    w_ours.fit(X32[:12_000], y[:12_000])
    w_ref.fit(X[:12_000], y[:12_000])
    werr = rel(np.r_[w_ours.coef_[0], w_ours.intercept_], np.r_[w_ref.coef_[0], w_ref.intercept_])
    assert np.array_equal(w_ours.n_iter_, w_ref.n_iter_) and werr < COEF_TOL, werr
    buf = io.BytesIO()
    joblib.dump(ours.to_sklearn(), buf)
    buf.seek(0)
    sk = joblib.load(buf)
    assert rel(sk.predict_proba(X32.astype(np.float64)), ours.predict_proba(X32)) < COEF_TOL
    assert np.array_equal(sk.predict(X32.astype(np.float64)), ours.predict(X32))
    print(f"\n[logistic labels {labels}] masked coef {err:.2e}, warm start {werr:.2e}")


@pytest.mark.parametrize("case", ["collinear", "separable"])
def test_unpenalised_hard_cases(ctx, case):
    X, t = make_data(n=16_384, d=24, seed=9, collinear=case == "collinear", scale=40.0 if case == "separable" else 1.0)
    ours, ref = _fit_both(ctx, X, t, C=np.inf)
    X32 = X.astype(np.float32)
    agree = float(np.mean(ours.predict(X32) == ref.predict(X)))
    assert agree > 0.999, agree
    print(f"\n[logistic {case}] n_iter {ours.n_iter_[0]}, predict agreement {agree}")


def test_device_rows_and_device_labels(ctx):
    """1 M x 128: float64 host columns through upload_columns, fp32 labels on the device."""
    rng = np.random.default_rng(13)
    n, d = 1_000_000, 128
    X = rng.normal(size=(n, d)).astype(np.float32).astype(np.float64)
    beta = rng.normal(size=d) * 0.1
    y = np.where(rng.uniform(size=n) < expit(X @ beta - 0.2), 2.0, -1.0).astype(np.float32)
    Xd = ctx.upload_columns([X[:, j] for j in range(d)])
    yd = ctx.to_device(y)
    try:
        ours = b2.B200LogisticRegression(ctx=ctx).fit(Xd, yd)
        ref = linear_model.LogisticRegression(solver="newton-cholesky").fit(X, y)
        err = rel(np.r_[ours.coef_[0], ours.intercept_], np.r_[ref.coef_[0], ref.intercept_])
        assert ours.classes_.dtype == np.float32 and np.array_equal(ours.classes_, ref.classes_)
        assert np.array_equal(ours.n_iter_, ref.n_iter_) and err < COEF_TOL, err
        lab, pr, dec = ours.predict(Xd), ours.predict_proba(Xd), ours.decision_function(Xd)
        assert isinstance(lab, b2.DeviceArray) and lab.kind == "f32" and pr.shape == (n, 2) and dec.kind == "f64"
        assert np.array_equal(lab.to_host(), ref.predict(X).astype(np.float32))
        assert rel(pr.to_host(), ref.predict_proba(X)) < COEF_TOL
        assert ours.score(Xd, yd) == accuracy_score(y, ref.predict(X))
        for a in (lab, pr, dec):
            a.free()
    finally:
        Xd.free(); yd.free()
    print(f"\n[logistic 1M x 128 device rows] n_iter {ours.n_iter_[0]}, coef {err:.2e}")


def test_refusals_and_errors(ctx):
    X, t = make_data(n=1000, d=4)
    X32 = X.astype(np.float32)
    with pytest.raises(ValueError, match="multinomial"):
        b2.B200LogisticRegression(ctx=ctx).fit(X32, np.arange(1000) % 3)
    yd = ctx.to_device((np.arange(1000) % 3).astype(np.float32))
    Xd = ctx.to_device(X32)
    try:
        with pytest.raises(ValueError, match="multinomial"):
            b2.B200LogisticRegression(ctx=ctx).fit(Xd, yd)
    finally:
        yd.free(); Xd.free()
    y32, coef, o = t.astype(np.float32), np.zeros(4), np.zeros(16)
    lib = native.load()
    args = (ctx._h, X32.ctypes.data, b2.F32, y32.ctypes.data, 1000, 4, 4, native.MEM_HOST, None, 1)
    assert lib.b2_logistic_pass(*args, 0.0, 0.0, coef.ctypes.data, 0.0, 1, o.ctypes.data, None) == E_ARG
    assert lib.b2_logistic_pass(*args, 0.0, 0.1, coef.ctypes.data, 0.0, 1, o.ctypes.data, None) == E_ARG   # not fp32
    assert lib.b2_logistic_pass(*args, 0.0, float("nan"), coef.ctypes.data, 0.0, 1, o.ctypes.data, None) == E_ARG
    assert lib.b2_logistic_pass(*args, 0.0, 1.0, coef.ctypes.data, 0.0, 1, None, None) == E_ARG
    assert lib.b2_logistic_line_search(*args, 0.0, 1.0, coef.ctypes.data, 0.0, coef.ctypes.data, 0.0, 22,
                                       o.ctypes.data) == E_ARG
    assert lib.b2_logistic_predict(ctx._h, X32.ctypes.data, b2.F32, 1000, 4, 4, native.MEM_HOST, coef.ctypes.data, 0.0,
                                   0.0, 1.0, None, None, None) == E_ARG
    assert lib.b2_label_scan(ctx._h, None, 10, None, 1, o.ctypes.data) == E_ARG
    other = b2.Context(0)
    try:
        b2.Context.comm_p2p_attach_local([ctx, other])
        assert lib.b2_logistic_pass(*args, 0.0, 1.0, coef.ctypes.data, 0.0, 1, o.ctypes.data, None) == E_UNSUPPORTED
        assert lib.b2_label_scan(ctx._h, y32.ctypes.data, 10, None, 1, o.ctypes.data) == E_UNSUPPORTED
    finally:
        for c in (ctx, other):
            c.comm_p2p_detach()
        other.close()
