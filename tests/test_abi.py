"""CPU-side checks: the C-ABI library loads and exports every symbol include/b2gram.h declares,
fails loudly without a GPU, and the host logic (split mask, metrics algebra, artefact layout) matches
the oracle.  No compute call is made here."""
import ctypes
import io
import os
import re

import numpy as np
import pytest

import bodywork_mlops_demo_b200 as b2
from bodywork_mlops_demo_b200 import stage_1_train_model as s1
from oracle import ols_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "b2gram.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(b2.native.lib_path())
    declared = _header_symbols()
    assert len(declared) >= 30
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/b2gram.h but not exported"
    # and the Python binding table covers the header one to one
    assert sorted(b2.native.EXPORTED_SYMBOLS) == declared


def _header_prototypes():
    """name -> list of parameter type strings, parsed from include/b2gram.h"""
    text = open(os.path.join(ROOT, "include", "b2gram.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(?:int|const char\s*\*)\s+(b2_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        params = [p.strip() for p in m.group(2).split(",")]
        if params == ["void"]:
            params = []
        protos[m.group(1)] = params
    return protos


def _ctype_class(param: str) -> str:
    """coarse class of a C parameter: what the ctypes argtype must be compatible with"""
    ptype = re.sub(r"\b[a-zA-Z_][a-zA-Z0-9_]*$", "", param).strip()       # drop the parameter name
    if "*" in ptype:
        return "pointer"
    if "double" in ptype:
        return "double"
    if "int64_t" in ptype or "uint64_t" in ptype or "size_t" in ptype:
        return "int64"
    return "int32"


def test_ctypes_signatures_match_the_header_prototypes():
    """Arity and coarse type class (pointer / 64-bit / 32-bit / double) of every binding == the C prototype."""
    import ctypes as C
    protos = _header_prototypes()
    assert sorted(protos) == sorted(b2.native.EXPORTED_SYMBOLS)
    for name, (_res, args) in b2.native._SIGNATURES.items():
        params = protos[name]
        assert len(params) == len(args), f"{name}: header has {len(params)} parameters, binding {len(args)}"
        for param, ctype in zip(params, args):
            want = _ctype_class(param)
            if want == "pointer":
                ok = ctype in (C.c_void_p, C.c_char_p) or hasattr(ctype, "contents") or issubclass(ctype, C._Pointer)
            elif want == "double":
                ok = ctype is C.c_double
            elif want == "int64":
                ok = C.sizeof(ctype) == 8 and ctype not in (C.c_double,)
            else:
                ok = C.sizeof(ctype) == 4 and ctype is not C.c_float
            assert ok, f"{name}: parameter '{param}' bound as {ctype}"


def test_abi_version_and_error_string():
    lib = b2.native.load()
    assert lib.b2_abi_version() == 2
    assert isinstance(b2.native.last_error(), str)


def test_no_cpu_fallback_without_gpu():
    if b2.native.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        b2.Context(0)
    with pytest.raises(RuntimeError):
        s1.model_metrics(np.ones(4), np.ones(4))


def test_plain_c_client_builds_against_the_header_and_refuses_to_run_on_the_cpu(c_client):
    """The boundary is C: a C99 translation unit with only include/b2gram.h links against the library, and without
    a GPU the fit fails with the library's error text (exit 3) rather than falling back to host arithmetic."""
    import subprocess
    proc = subprocess.run([c_client], capture_output=True, text=True, timeout=120)
    if b2.native.device_count() > 0:
        assert proc.returncode == 0, proc.stdout + proc.stderr
    else:
        assert proc.returncode == 3, proc.stdout + proc.stderr
        assert "no CPU fallback" in proc.stdout


def test_library_has_hopper_native_sass():
    """wgmma / TMA must be in the shipped binary, compiled for sm_90a."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", b2.native.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    # wgmma from shared-memory descriptors with register accumulators, the warpgroup register split and TMA tensor loads
    # (gram_tc), TMA bulk copies (gram_narrow, score kernels), mbarrier try_wait pipelines
    # and, for bf16-stored D = 128 rows, the raw swizzled TMA tile as an MN-major (transposed) B operand
    for mnemonic in ("HGMMA.64x144x16.F32.BF16", "HGMMA.64x128x16.F32.BF16", ".tnspB", "WARPGROUP.ARRIVE", "USETMAXREG",
                     "UTMALDG", "UBLKCP", "SYNCS.PHASECHK.TRANS64.TRYWAIT"):
        assert mnemonic in sass, mnemonic


def test_split_mask_restates_numpys_legacy_generator_bit_for_bit():
    """b2_split_mask (host C: MT19937 + Fisher-Yates with prefetched swap partners) == RandomState(seed).permutation(n)
    for block boundaries of the generator (624 words), rejection-heavy sizes (just above a power of two) and seeds."""
    for n, seed in ((2, 42), (3, 42), (624, 42), (625, 42), (1025, 42), (65_537, 42), (200_003, 0), (77_777, 2 ** 31 + 5)):
        n_test = int(np.ceil(0.2 * n))
        perm = np.random.RandomState(seed).permutation(n)
        want = np.ones(n, np.uint8); want[perm[:n_test]] = 0
        assert np.array_equal(s1.split_mask(n, seed=seed), want), (n, seed)
    lib = b2.native.load()
    assert lib.b2_split_mask(0, 0, 42, None) == -1 and "b2_split_mask" in b2.native.last_error()


def test_split_mask_cache_round_trip(tmp_path, monkeypatch):
    monkeypatch.setenv("B2_CACHE_DIR", str(tmp_path))
    a = s1.split_mask(12_345)
    assert (tmp_path / "split-mask-n12345-t0.2-s42.u8").stat().st_size == 12_345
    assert np.array_equal(s1.split_mask(12_345), a) and np.array_equal(s1.split_mask_async(12_345).result(), a)


@pytest.mark.parametrize("n", [5, 57, 1440, 10_001])
def test_split_mask_equals_reference_split(golden_dir, n):
    g = np.load(os.path.join(golden_dir, f"sk_split_n{n}.npz"))
    mask = s1.split_mask(n)
    assert np.array_equal(np.sort(np.flatnonzero(mask == 1)), np.sort(g["train"]))
    assert np.array_equal(np.sort(np.flatnonzero(mask == 0)), np.sort(g["test"]))
    tr, te = orc.split_indices(n)
    assert set(np.flatnonzero(mask == 1)) == set(tr) and set(np.flatnonzero(mask == 0)) == set(te)


def test_metrics_from_stats_matches_reference_metrics(golden_dir):
    g = np.load(os.path.join(golden_dir, "ref_model_metrics.npz"))
    stats = orc.score_stats(g["y"], g["p"])
    mape, r2, mx = s1.metrics_from_stats(stats)
    assert mape == pytest.approx(float(g["MAPE"]), rel=1e-12)
    assert r2 == pytest.approx(float(g["r_squared"]), rel=1e-10)
    assert mx == pytest.approx(float(g["max_residual"]), rel=1e-14)


def test_metrics_edge_cases():
    # constant y, perfect prediction -> r2 == 1 (sklearn force_finite); imperfect -> 0
    y = np.full(10, 3.0)
    assert s1.metrics_from_stats(orc.score_stats(y, y))[1] == 1.0
    assert s1.metrics_from_stats(orc.score_stats(y, y + 1))[1] == 0.0
    with pytest.raises(RuntimeError):
        s1.metrics_from_stats(np.zeros(6))


def test_bf16_bit_conversion_round_to_nearest_even():
    x = np.array([1.0, 1.00390625, 1.01171875, -3.14159, 0.0, 65504.0, 1e-20], dtype=np.float32)
    bits = b2.native.to_bf16_bits(x)
    back = b2.native.from_bf16_bits(bits)
    assert back[0] == 1.0 and back[4] == 0.0
    assert np.all(np.abs(back - x) <= np.abs(x) * 2.0 ** -8)
    assert back[1] == 1.0            # 1 + 2^-8 ties to even (down)
    assert back[2] == np.float32(1.015625)  # 1 + 3*2^-8 ties to even (up)


def test_sklearn_artefact_layout_and_stage2_contract(tmp_path):
    """The estimator we dump must behave exactly like the reference's for stage_2_serve_model.py:65,78,79."""
    import joblib
    from sklearn.linear_model import LinearRegression
    est = b2.B200LinearRegression()
    est.coef_ = np.array([0.5, -0.25]); est.intercept_ = np.float64(1.5)
    est.rank_ = 2; est.singular_ = np.array([3.0, 1.0]); est.n_features_in_ = 2
    reg = est.to_sklearn()
    assert type(reg) is LinearRegression and str(reg) == "LinearRegression()"
    path = tmp_path / "regressor-2021-04-08.joblib"
    joblib.dump(reg, path)
    loaded = joblib.load(io.BytesIO(path.read_bytes()))
    X = np.array([[50.0, 2.0]], ndmin=2)
    assert loaded.predict(X)[0] == pytest.approx(0.5 * 50 - 0.25 * 2 + 1.5)
    ref = LinearRegression().fit(np.random.RandomState(0).rand(20, 2), np.random.RandomState(1).rand(20))
    assert set(vars(ref)) == set(vars(loaded))  # same attribute set as a genuinely fitted estimator
    assert loaded.coef_.dtype == np.float64 and loaded.coef_.shape == (2,)


def test_feature_columns_and_dataset_loader(tmp_path):
    import pandas as pd
    folder = tmp_path / "datasets"
    folder.mkdir()
    for day, n in (("2021-04-09", 3), ("2021-04-08", 2)):
        pd.DataFrame({"date": [day] * n, "y": np.arange(n, dtype=float), "X": np.arange(n, dtype=float)}) \
            .to_csv(folder / f"regression-dataset-{day}.csv", index=False)
    data, newest = s1.download_latest_dataset(str(tmp_path))
    assert str(newest) == "2021-04-09" and len(data) == 5
    assert list(data["date"])[:2] == ["2021-04-08"] * 2   # oldest tranche first
    assert s1.feature_columns(data) == ["X"]
    assert s1.feature_columns(pd.DataFrame({"y": [1], "X10": [1], "X2": [1]})) == ["X2", "X10"]
    with pytest.raises(RuntimeError):
        s1.download_latest_dataset(str(tmp_path / "missing"))


def test_service_test_metrics_algebra_matches_stage_4_definitions():
    """stage_4's record (APE mean, Pearson 'r_squared', max APE) from the ten reductions == direct evaluation."""
    import datetime as dt
    from bodywork_mlops_demo_b200 import stage_2_scoring as s2
    rng = np.random.RandomState(3)
    label = rng.uniform(5, 80, 1317)
    score = label * (1 + rng.normal(0, 0.3, 1317))
    rec = s2.test_metrics_from_stats(orc.score_stats(label, score), dt.date(2021, 4, 8), 0.00822)
    want = orc.service_test_metrics(label, score)
    assert list(rec.columns) == ["date", "MAPE", "r_squared", "max_residual", "mean_response_time"]
    assert rec["MAPE"].iloc[0] == pytest.approx(want["MAPE"], rel=1e-12)
    assert rec["r_squared"].iloc[0] == pytest.approx(want["r_squared"], rel=1e-10)
    assert rec["max_residual"].iloc[0] == pytest.approx(want["max_residual"], rel=1e-12)
    import pandas as pd
    df = pd.DataFrame({"score": score, "label": label})          # the reference's own pandas expressions
    assert rec["r_squared"].iloc[0] == pytest.approx(df.score.corr(df.label), rel=1e-10)


def test_pack_columns_gathers_and_converts_like_numpy():
    """b2_pack_columns (host only): strided float64 / float32 columns -> np.stack(columns, 1).astype(float32), bit for bit,
    across the thread split (n above and below the 4 096-row single-thread cut, not a multiple of 64) -- the gather
    b2_upload_columns runs on the way to the device."""
    rng = np.random.RandomState(0)
    for n, d, dtype in ((1, 1, np.float64), (100, 3, np.float64), (5000, 7, np.float32), (70_001, 128, np.float64),
                        (33_333, 17, np.float64)):
        block = (rng.rand(d, n) * 100 - 50).astype(dtype)              # pandas: one (d, n) block, contiguous columns
        cols = [block[j] for j in range(d)]
        if d >= 3:
            cols[1] = (rng.rand(2 * n) * 100).astype(dtype)[::2]           # a strided column
            cols[2] = np.asfortranarray(rng.rand(n, 2).astype(dtype))[:, 1]
        got = b2.native.pack_columns(cols)
        assert got.dtype == np.float32 and got.shape == (n, d)
        assert np.array_equal(got, np.stack(cols, axis=1).astype(np.float32)), (n, d)
    # row-major float64 matrix (the estimator's view list), reversed rows (negative stride), a broadcast column (stride 0),
    # non-finite and out-of-float32-range values: the conversion is numpy's, element by element
    X = rng.rand(9001, 20) * 1e3
    X[5, 3], X[6, 3], X[7, 3], X[8, 3], X[9, 3] = np.nan, np.inf, -np.inf, 1e300, -1e-300
    cols = [X[:, j] for j in range(20)]
    cols[4] = X[::-1, 4]
    cols[5] = np.broadcast_to(np.float64(2.5), (9001,))
    with np.errstate(over="ignore"):
        want = np.stack(cols, axis=1).astype(np.float32)
    assert np.array_equal(b2.native.pack_columns(cols), want, equal_nan=True)
    with pytest.raises(RuntimeError):
        b2.native.pack_columns([np.zeros(4), np.zeros(5)])
    with pytest.raises(RuntimeError):
        b2.native.pack_columns([np.zeros(4, np.int32)])
