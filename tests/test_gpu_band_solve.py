"""K4 on the device: glio_band_solve's L and x bit-identical to tests/band_solve_reference.py (whose factor and forward half are the
scalar host path's, tests/test_band_solve_reference.py) over sizes, half bandwidths up to GLIO_BAND_MAX_HB, n <= hb and diagonals
scaled over 1e-12 .. 1e12; failure on indefinite and NaN bands; the argument checks; run-to-run determinism."""
import numpy as np
import pytest

from tests import band_solve_reference as br

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


@pytest.fixture(scope="module")
def ctx(api):
    c = api.Context(0)
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _check(ctx, n, hb, scale, seed):
    rng = np.random.default_rng(seed)
    band = br.random_spd_band(n, hb, rng, scale)
    b = rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)
    L_ref, _, x_ref, ok_ref = br.band_cholesky_solve(band, b)
    assert ok_ref
    L, x, ok = ctx.band_solve(band, b)
    assert ok
    assert np.array_equal(_bits(L), _bits(L_ref)), f"L differs at {np.argwhere(_bits(L) != _bits(L_ref))[:5].tolist()}"
    assert np.array_equal(_bits(x), _bits(x_ref)), f"x differs at {np.flatnonzero(_bits(x) != _bits(x_ref))[:5].tolist()}"


@pytest.mark.parametrize("scale", [0, 6])
@pytest.mark.parametrize("hb", [0, 1, 5, 41, 104, 160])
@pytest.mark.parametrize("n", [1, 2, 7, 1200])
def test_band_solve_bit_identical_to_reference(ctx, n, hb, scale):
    _check(ctx, n, hb, scale, seed=n * 1000 + hb * 10 + scale)


@pytest.mark.parametrize("hb", [0, 41, 104, 160])
def test_band_solve_bit_identical_to_reference_level1_size(ctx, hb):
    # n of the level-1 batch problem at the sample run's K = 3 457 (15 columns per keyframe)
    _check(ctx, 51855, hb, 6, seed=hb)


def test_band_solve_is_deterministic(ctx):
    rng = np.random.default_rng(5)
    band = br.random_spd_band(20742, 41, rng, 3)
    b = rng.standard_normal(20742)
    L1, x1, ok1 = ctx.band_solve(band, b)
    L2, x2, ok2 = ctx.band_solve(band, b)
    assert ok1 and ok2
    assert np.array_equal(_bits(L1), _bits(L2)) and np.array_equal(_bits(x1), _bits(x2))


@pytest.mark.parametrize("case", ["negative_diagonal", "indefinite", "nan_diagonal", "nan_off", "nan_rhs", "inf_rhs"])
def test_band_solve_fails_like_the_host(ctx, case):
    rng = np.random.default_rng(6)
    n, hb = 500, 41
    band = br.random_spd_band(n, hb, rng)
    b = np.ones(n)
    if case == "negative_diagonal":
        band[300, hb] = -band[300, hb]
    elif case == "indefinite":
        band[301, hb - 1] = 10.0 * band[301, hb]
    elif case == "nan_diagonal":
        band[250, hb] = np.nan
    elif case == "nan_off":
        band[250, hb - 7] = np.nan
    elif case == "nan_rhs":
        b[100] = np.nan
    else:
        b[100] = np.inf
    assert not br.band_cholesky_solve(band, b)[3]
    _, _, ok = ctx.band_solve(band, b)
    assert not ok
    _check(ctx, n, hb, 0, seed=7)          # the context solves the next system as usual


def test_band_solve_arguments(api, ctx):
    rng = np.random.default_rng(8)
    with pytest.raises(api.GlioError, match="GLIO_BAND_MAX_HB"):
        ctx.band_solve(br.random_spd_band(400, api.BAND_MAX_HB + 1, rng), np.ones(400))
    with pytest.raises(api.GlioError, match="n > 0"):
        ctx.band_solve(np.zeros((0, 5)), np.zeros(0))
    _check(ctx, 400, api.BAND_MAX_HB, 6, seed=9)


def test_band_solve_kernel_is_profiled(ctx):
    rng = np.random.default_rng(10)
    band = br.random_spd_band(300, 20, rng)
    ctx.lib_profile(True)
    before = ctx.launch_count
    ctx.band_solve(band, np.ones(300))
    prof = ctx.lib_profile_read()
    ctx.lib_profile(False)
    assert ctx.launch_count == before + 1
    assert prof["k_band_chol_solve"][1] == 1 and prof["k_band_chol_solve"][0] > 0.0
