"""RidgeClassifierCV on the H100: b2_ridge_classifier_loo (the leave-one-out pass with T targets) against the numpy
oracle (tests/loo_classes_oracle.py) on the same rounded rows, against b2_ridge_loo for two classes, and the estimator
against scikit-learn's RidgeClassifierCV.

Tolerances (asserted; run with -s for the worst case each test measured):
  * on the exact fp64 (SIMT) Gram path, against the oracle of the same rows, with and without an intercept: mse relative
    1e-10, cv max |difference| / max |cv| 1e-9 (DESIGN section 6's bounds), the model at the chosen alpha 1e-9, correct
    counts and best equal; repeated calls bit-identical;
  * every layout (fp32 / bf16; ring, misaligned X or y, masked, host rows) with many tiles per CTA and a direct tail,
    K in {2, 3, 10, 32}, A in {1, 3, 13, 64}: the same bounds; kept / unmatched / non-finite counts equal, also with
    labels outside the classes;
  * two classes, scoring None: b2_ridge_loo on y = +-1 of the same rows within 1e-12 (mse) and 1e-11 (cv);
  * the estimator on KERNEL_SIMT against scikit-learn: alpha_ and predict equal, best_score_ and coefficients 1e-12
    relative; on the default tensor-core Gram, alpha_ equal on well-separated grids and coefficients within 1e-5;
  * 1 M x 128 float64 host columns with ten fp32 device labels: alpha_ equal, predict agreement >= 0.9999.
"""
import ctypes as C

import numpy as np
import pytest
from sklearn.linear_model import RidgeClassifierCV

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import _native as native
from loo_classes_oracle import ridge_classifier_loo
from test_gpu_tile_passes import TILE, Dev, _layouts, n_long

pytestmark = pytest.mark.gpu

MSE_TOL, CV_TOL = 1e-10, 1e-9
KA = [(2, 1), (3, 3), (10, 13), (32, 64)]


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)) if b.size else 0.0


def alphas_of(A):
    return np.logspace(-2, 3, A) if A > 1 else np.array([1.0])


class Rows:
    """n rows (fp32 or bf16, the values the kernels read as float64 in Xv), fp32 labels of K classes in y["cls"]
    (a few kept rows of no class, NaN and -inf where unmatched=True), their class indices and a mask."""

    def __init__(self, kind, d, n, K, seed, unmatched=False):
        rng = np.random.default_rng(seed)
        X = (rng.normal(size=(n, d)) * 0.5 + 0.25).astype(np.float32)
        self.kind, self.d, self.n, self.K = kind, d, n, K
        self.dt, self.es = (b2.BF16, 2) if kind == "bf16" else (b2.F32, 4)
        self.up = native.to_bf16_bits(X) if kind == "bf16" else X
        self.Xv = native.from_bf16_bits(self.up).astype(np.float64) if kind == "bf16" else X.astype(np.float64)
        self.classes = (np.arange(K) * 3 - 7).astype(np.float32)
        k = np.argmax(self.Xv @ rng.normal(size=(d, K)) + rng.normal(0.0, 1.0, size=(n, K)), axis=1)
        k[: min(K, n)] = np.arange(min(K, n))
        y = self.classes[k].copy()
        if unmatched and n > 64:
            bad = rng.choice(np.arange(K, n), 4, replace=False)
            y[bad] = [99.0, 0.5, np.nan, -np.inf]
            k[bad] = -1
        self.k, self.y = k, {"cls": y.astype(np.float32)}
        self.mask = (rng.uniform(size=n) < 0.8).astype(np.uint8)
        self.mask[:K] = 1


def oracle(t, n, alphas, masked, scoring=None, fit_intercept=True):
    with np.errstate(invalid="ignore", divide="ignore"):
        return ridge_classifier_loo(t.Xv[:n], t.k[:n], t.K, alphas, mask=t.mask[:n] if masked else None,
                                    fit_intercept=fit_intercept, scoring=scoring)


def call(ctx, L, t, n, alphas, masked, scoring=native.LOO_SQUARED, fit_intercept=True):
    """b2_ridge_classifier_loo on a layout's device pointers: the outputs, with cv on the host"""
    lib, d, T, A = native.load(), t.d, 1 if t.K == 2 else t.K, alphas.size
    cvd = ctx.empty((max(n, 1), T, A), "f64")
    mse, correct, coef, b0, counts = np.empty(A), np.empty(A), np.empty((T, d)), np.empty(T), np.empty(3)
    best = np.zeros(1, np.int32)
    try:
        rc = lib.b2_ridge_classifier_loo(ctx._h, L.xp, L.dt, L.yp["cls"], n, d, d, native.MEM_DEVICE, L.mask(masked),
                                         1, t.classes.ctypes.data, t.K, alphas.ctypes.data, A, int(fit_intercept),
                                         scoring, mse.ctypes.data, correct.ctypes.data, cvd.ptr,
                                         best.ctypes.data_as(C.POINTER(C.c_int)), coef.ctypes.data, b0.ctypes.data, counts.ctypes.data)
        assert rc == 0, native.last_error()
        cv = cvd.to_host()[:n]
    finally:
        cvd.free()
    return {"mse": mse, "correct": correct, "cv": cv, "best": int(best[0]), "coef": coef, "intercept": b0,
            "counts": counts}


def check(got, want, t, n, masked, what):
    keep = t.mask[:n] == 1 if masked else np.ones(n, bool)
    e_mse, e_cv = rel(got["mse"], want["mse"]), rel(got["cv"][keep], want["cv"])
    assert e_mse <= MSE_TOL and e_cv <= CV_TOL, f"{what}: mse {e_mse:.3e}, cv {e_cv:.3e}"
    assert np.all(np.isnan(got["cv"][~keep]))
    assert np.array_equal(got["correct"], want["correct"]), what
    assert got["best"] == want["best"], what
    kept = keep.sum()
    ys = t.y["cls"][:n][keep]
    assert got["counts"][0] == kept and got["counts"][1] == np.sum(~np.isin(ys, t.classes))
    assert got["counts"][2] == np.sum(~np.isfinite(ys))
    return e_mse, e_cv


@pytest.mark.parametrize("fit_intercept", [True, False])
@pytest.mark.parametrize("d", [1, 2, 7, 8, 9, 16, 17, 33, 64, 127, 128])
def test_pass_matches_the_oracle_on_the_exact_gram(ctx, d, fit_intercept):
    """with an intercept: the centred class sums, ybar_k = 2 n_k / n - 1 and h0 = 1 / n; without: the uncentred sums,
    the right-hand sides 2 s_k - s, ybar = 0 and h0 = 0"""
    t = Rows("f32", d, 3000 + d, 3, seed=d)
    dev = Dev(ctx, t, t.mask)
    L = _layouts(dev, True)["ring"]
    ctx.set_kernel(b2.KERNEL_SIMT)
    fi = fit_intercept
    try:
        worst = [0.0, 0.0]
        for scoring, name in ((native.LOO_SQUARED, None), (native.LOO_ACCURACY, "accuracy")):
            for masked in (False, True):
                al = alphas_of(5)
                got = call(ctx, L, t, t.n, al, masked, scoring, fit_intercept=fi)
                want = oracle(t, t.n, al, masked, name, fit_intercept=fi)
                e = check(got, want, t, t.n, masked, f"D = {d}, intercept {fi}")
                assert rel(got["coef"], want["coef"]) <= CV_TOL
                if fi:
                    assert rel(got["intercept"], want["intercept"]) <= CV_TOL
                else:
                    assert np.all(got["intercept"] == 0.0)
                worst = [max(worst[0], e[0]), max(worst[1], e[1])]
                again = call(ctx, L, t, t.n, al, masked, scoring, fit_intercept=fi)
                for key in ("mse", "correct", "cv", "coef", "intercept"):
                    assert np.array_equal(again[key], got[key], equal_nan=True), key
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        dev.free()
    print(f"\nD = {d}, intercept {fi}: worst mse {worst[0]:.3e}, cv {worst[1]:.3e}")


@pytest.mark.parametrize("K,A", KA)
@pytest.mark.parametrize("kind,d", [("f32", 8), ("f32", 24), ("f32", 128), ("bf16", 24), ("bf16", 128)])
def test_every_layout_with_many_tiles_per_cta(ctx, kind, d, K, A):
    n = n_long(ctx.info()["sm_count"])
    t = Rows(kind, d, n, K, seed=K * 1000 + d)
    dev = Dev(ctx, t, t.mask)
    al = alphas_of(A)
    worst = [0.0, 0.0]
    ctx.set_kernel(b2.KERNEL_SIMT)
    try:
        for name, L in _layouts(dev, True).items():
            for masked in ((False, True) if name == "ring" else (name == "mask+1",)):
                for rows in (n, TILE * (n // TILE)):
                    scoring = native.LOO_ACCURACY if masked else native.LOO_SQUARED
                    got = call(ctx, L, t, rows, al, masked, scoring)
                    want = oracle(t, rows, al, masked, "accuracy" if masked else None)
                    e = check(got, want, t, rows, masked, f"{kind} D = {d} K = {K} A = {A} {name} n = {rows}")
                    worst = [max(worst[0], e[0]), max(worst[1], e[1])]
        # host rows: the staging ring, cv through the per-row output blocks (several blocks at T A = 2048)
        res = ctx.ridge_classifier_loo(t.up, t.y["cls"], t.classes, al, t.mask, 1, store_cv=True)
        want = oracle(t, n, al, True)
        host = {"mse": res["mse"], "correct": res["correct"], "cv": res["cv"], "best": res["best"],
                "counts": np.array([res["kept"], res["unmatched"], res["nonfinite"]])}
        e = check(host, want, t, n, True, f"{kind} D = {d} K = {K} A = {A} host rows")
        worst = [max(worst[0], e[0]), max(worst[1], e[1])]
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
        dev.free()
    print(f"\n{kind} D = {d} K = {K} A = {A}: worst mse {worst[0]:.3e}, cv {worst[1]:.3e}")


@pytest.mark.parametrize("K", [2, 10])
def test_counts_of_labels_outside_the_classes(ctx, K):
    """kept rows whose y is no class (99, 0.5, NaN, -inf) are counted; the estimator refuses such labels before the
    call, and the error is RidgeClassifierCV's only when every kept row has a class"""
    t = Rows("f32", 16, 5000, K, seed=K, unmatched=True)
    dev = Dev(ctx, t, t.mask)
    try:
        for masked in (False, True):
            got = call(ctx, _layouts(dev, True)["ring"], t, t.n, alphas_of(3), masked)
            keep = t.mask == 1 if masked else np.ones(t.n, bool)
            ys = t.y["cls"][keep]
            assert got["counts"].tolist() == [keep.sum(), np.sum(~np.isin(ys, t.classes)), np.sum(~np.isfinite(ys))]
            assert np.all(np.isfinite(got["mse"])) and np.all(np.isnan(got["cv"][~keep]))
    finally:
        dev.free()


def test_two_classes_match_the_single_target_ridge_loo(ctx):
    t = Rows("f32", 20, 20000, 2, seed=5)
    al = alphas_of(13)
    ctx.set_kernel(b2.KERNEL_SIMT)
    try:
        Xd, yd = ctx.to_device(t.up), ctx.to_device(t.y["cls"])
        ypm = ctx.to_device(np.where(t.k == 1, 1.0, -1.0).astype(np.float32))
        res = ctx.ridge_classifier_loo(Xd, yd, t.classes, al, store_cv=True)
        mse, best, _, _, cv = ctx.ridge_loo(Xd, ypm, al, store_cv=True)
        cvc, cvr = res["cv"].to_host()[:, 0, :], cv.to_host()
        for a in (Xd, yd, ypm, res["cv"], cv):
            a.free()
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
    e_mse, e_cv = rel(res["mse"], mse), rel(cvc, cvr)
    print(f"\nK = 2 against b2_ridge_loo: mse {e_mse:.3e}, cv {e_cv:.3e}")
    assert res["best"] == best and e_mse <= 1e-12 and e_cv <= 1e-11


def _sk_data(n, d, K, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32).astype(np.float64)
    k = np.argmax(X @ rng.normal(size=(d, K)) + rng.normal(0.0, 2.0, size=(n, K)), axis=1)
    k[:K] = np.arange(K)
    return X, k


@pytest.mark.parametrize("scoring", [None, "accuracy"])
@pytest.mark.parametrize("K", [2, 3, 10, 32])
def test_estimator_matches_sklearn_on_the_exact_gram(ctx, K, scoring):
    X, y = _sk_data(4000, 24, K, seed=K)
    al = (0.01, 1.0, 30.0, 1000.0)
    ctx.set_kernel(b2.KERNEL_SIMT)
    try:
        ours = b2.B200RidgeClassifierCV(alphas=al, scoring=scoring, ctx=ctx).fit(X, y)
        pred = ours.predict(X)
    finally:
        ctx.set_kernel(b2.KERNEL_AUTO)
    ref = RidgeClassifierCV(alphas=al, scoring=scoring).fit(X, y)
    e_s = abs(ours.best_score_ - ref.best_score_) / abs(ref.best_score_)
    e_c = rel(ours.coef_, ref.coef_)
    print(f"\nK = {K} {scoring}: best_score_ {e_s:.3e}, coef {e_c:.3e}")
    assert ours.alpha_ == ref.alpha_ and np.array_equal(pred, ref.predict(X))
    assert e_s <= 1e-12 and e_c <= 1e-12


@pytest.mark.parametrize("K", [3, 10])
def test_estimator_on_the_tensor_core_gram(ctx, K):
    X, y = _sk_data(50000, 64, K, seed=100 + K)
    al = (1e-2, 1e2, 1e4, 1e6)
    ours = b2.B200RidgeClassifierCV(alphas=al, ctx=ctx, store_cv_results=True).fit(X, y)
    ref = RidgeClassifierCV(alphas=al, store_cv_results=True).fit(X, y)
    e_c, e_cv = rel(ours.coef_, ref.coef_), rel(ours.cv_results_, ref.cv_results_)
    print(f"\nK = {K} tensor-core Gram: coef {e_c:.3e}, cv {e_cv:.3e}")
    assert ours.alpha_ == ref.alpha_ and e_c <= 1e-5 and e_cv <= 1e-5
    assert np.mean(ours.predict(X) == ref.predict(X)) >= 0.999


def test_million_rows_from_float64_columns_with_device_labels(ctx):
    n, d, K = 1_000_000, 128, 10
    X, k = _sk_data(n, d, K, seed=7)
    labels = (np.arange(K) * 2.0 + 1.0).astype(np.float32)
    Xd = ctx.upload_columns([X[:, j] for j in range(d)])
    yd = ctx.to_device(labels[k])
    try:
        ours = b2.B200RidgeClassifierCV(alphas=(1.0, 1e3, 1e5), ctx=ctx).fit(Xd, yd)
        pred = ours.predict(Xd).to_host()
    finally:
        Xd.free()
        yd.free()
    ref = RidgeClassifierCV(alphas=(1.0, 1e3, 1e5)).fit(X, labels[k])
    agree = float(np.mean(pred == ref.predict(X)))
    print(f"\n1 M x 128, ten device labels: alpha_ {ours.alpha_} / {ref.alpha_}, predict agreement {agree:.6f}")
    assert ours.alpha_ == ref.alpha_ and np.array_equal(ours.classes_, labels) and agree >= 0.9999
