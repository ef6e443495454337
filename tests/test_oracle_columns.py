"""CPU tests of the structured column tables and the scale-free statistic error (oracle.ols_oracle): what the GPU column
tests (tests/test_gpu_columns.py) measure the kernels with."""
import numpy as np
import pytest
from sklearn.linear_model import LinearRegression

from oracle import ols_oracle as orc


def _rel(a, b):
    """The relative error the GPU tests used before the scale-free one: max |S - So| / max |So|."""
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), 1e-300))


def _perturb_centred(S, a, b, delta):
    """S whose centred moment C_ab (and C_ba) is moved by delta, its sums and row count unchanged."""
    out = S.copy()
    out[a, b] += delta
    if a != b:
        out[b, a] += delta
    return out


def test_stat_error_ignores_a_common_offset():
    """The same centred error reads the same on rows with mean 50 and on the same rows moved by 1e4."""
    X, y = orc.generate_dataset(20_000, 8, seed=1)
    errs = []
    for off in (0.0, 1e4):
        So = orc.gram_stats(X + off, y)
        Co = orc.centred_moments(So)[2]
        S = _perturb_centred(So, 2, 5, 3e-5 * np.sqrt(Co[2, 2] * Co[5, 5]))
        stat, mean = orc.stat_error(S, So)
        assert mean == 0.0
        errs.append(stat)
    assert errs[0] == pytest.approx(3e-5, rel=1e-6)
    assert errs[1] == pytest.approx(3e-5, rel=1e-3)     # fp64 centring of S at mean 1e4 cancels ~ eps * (1e4 / 29)^2
    assert orc.stat_error(orc.gram_stats(X + 1e4, y), orc.gram_stats(X + 1e4, y)) == (0.0, 0.0)


def test_stat_error_catches_what_the_relative_error_of_s_accepts():
    """At D = 128 max |S| is sum y^2 ~ 1e7 n while a centred variance is ~ 833 n: a 1e-4 error in one centred entry is
    invisible to _rel(S, So) < 2e-6 and plain in the scale-free error."""
    X, y = orc.generate_dataset(20_000, 128, seed=2)
    So = orc.gram_stats(X, y)
    Co = orc.centred_moments(So)[2]
    S = _perturb_centred(So, 7, 7, 1e-4 * Co[7, 7])
    assert _rel(S, So) < 2e-6
    stat, _ = orc.stat_error(S, So)
    assert stat == pytest.approx(1e-4, rel=1e-6)
    # a wrong column sum (the mean of feature 3 off by 1e-4 sigma) moves the mean error
    n = So[128, 128]
    S2 = So.copy()
    delta = 1e-4 * np.sqrt(Co[3, 3] / n) * n
    S2[3, 128] += delta
    S2[128, 3] += delta
    assert _rel(S2, So) < 2e-6
    assert orc.stat_error(S2, So)[1] == pytest.approx(1e-4, rel=1e-3)


def test_stat_error_of_a_constant_column_is_finite():
    X, y, sigma = orc.column_table(5000, 6, "constant", seed=3)
    assert sigma[0] == 0.0 and np.all(X[:, 0] == orc.CONSTANT_VALUE)
    So = orc.gram_stats(X, y)
    assert orc.centred_moments(So)[2][0, 0] == 0.0                  # exact in fp64: 2021.5^2 has 24 significant bits
    stat, mean = orc.stat_error(So * (1 + 1e-15), So)
    assert np.isfinite(stat) and np.isfinite(mean)


@pytest.mark.parametrize("family,kw", [("offset", {}), ("offset", {"bf16": True}), ("scaled", {"scale": 1e-3}),
                                       ("scaled", {"scale": 1e3}), ("integer", {}), ("constant", {}),
                                       ("correlated", {"rho": 0.99})])
def test_column_tables_have_the_stated_shape(family, kw):
    n, d = 40_000, 16
    X, y, sigma = orc.column_table(n, d, family, seed=5, **kw)
    again = orc.column_table(n, d, family, seed=5, **kw)
    assert np.array_equal(X, again[0]) and np.array_equal(y, again[1])        # seeded
    assert X.dtype == np.float64 and X.shape == (n, d) and X.flags.c_contiguous
    live = sigma > 0
    np.testing.assert_allclose(X.std(axis=0)[live], sigma[live], rtol=0.05)
    if family == "offset" and kw.get("bf16"):
        assert np.all(sigma >= 2 * orc.bf16_spacing(X.mean(axis=0)) * 0.99)   # rows rounded to bf16 still vary
    if family == "scaled":
        assert np.any(X.mean(axis=0) > sigma) and np.any(X.mean(axis=0) < -sigma)
    if family == "integer":
        assert np.array_equal(X, np.round(X)) and set(np.unique(X[:, 1])) <= {0.0, 1.0}
    if family == "correlated":
        r = np.corrcoef(X[:, :8], rowvar=False)[np.triu_indices(8, 1)]
        np.testing.assert_allclose(r, 0.99, atol=2e-3)
    # every varying column moves y: the fit recovers a coefficient of |beta_j sigma_j| in [0.5, 2] (N(0, 1) noise)
    fo = orc.fit_from_stats(orc.gram_stats(X, y))
    ref = LinearRegression().fit(X, y)
    assert fo["rank"] == ref.rank_ == (d - 1 if family == "constant" else d)
    std_coef = np.abs(fo["coef"] * sigma)[live]
    assert np.all(std_coef > 0.4) and np.all(std_coef < 2.2)
    if family == "constant":
        assert abs(fo["coef"][0]) < 1e-6 and abs(ref.coef_[0]) < 1e-6     # fp64 rounding of S_0j ~ eps * 2021.5 * 1e5


def test_centred_condition_of_correlated_blocks():
    """Blocks of 8 columns with pairwise rho: kappa = (1 + 7 rho) / (1 - rho)."""
    for rho in (0.9, 0.99, 0.999):
        X, y, _ = orc.column_table(200_000, 8, "correlated", seed=7, rho=rho)
        kappa = orc.centred_condition(orc.gram_stats(X, y))
        assert kappa == pytest.approx((1 + 7 * rho) / (1 - rho), rel=0.1)


def test_coef_error_is_in_units_of_one_standard_deviation():
    X, y, sigma = orc.column_table(10_000, 5, "scaled", seed=9, scale=1e3)
    So = orc.gram_stats(X, y)
    fo = orc.fit_from_stats(So)
    moved = fo["coef"].copy()
    moved[4] += 1e-4 / sigma[4]
    assert orc.coef_error(moved, fo["coef"], So) == pytest.approx(1e-4, rel=0.05)
