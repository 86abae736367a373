"""tests/band_bcr_reference.py, the numpy restatement of the block cyclic reduction that the GPU tests hold glio_band_solve_bcr to:
its x meets the normwise backward-error bound scipy's banded Cholesky meets on the same bands, for one to many blocks and sizes
around block multiples; it fails on an indefinite band and on a NaN diagonal in any block; it never reads the layout's j < 0
slots."""
import numpy as np
import pytest
import scipy.linalg

from tests import band_bcr_reference as bcr
from tests import band_solve_reference as br

HBS = [0, 1, 5, 41, 104, 160, 194, 256]
BOUND = 1e-14


def sizes(hb):
    """n around block multiples: one block short, one block, one row into the next, two and three blocks, and 2^k blocks +- 1
    for a few k (the levels' odd counts and the last block's neighbours change there)"""
    b = bcr.block_size(hb)
    return sorted({b - 1, b, b + 1, 2 * b, 2 * b + 1, 3 * b, 4 * b - 1, 4 * b + 1, 8 * b - 1, 16 * b + 1} - {0})


def _scipy_solve(band, rhs):
    n, w = band.shape
    hb = w - 1
    ab = np.zeros((w, n))
    for d in range(min(w, n)):
        ab[d, :n - d] = band[d:, hb - d]
    return scipy.linalg.solveh_banded(ab, rhs, lower=True)


def _check(band, rhs):
    x, ok = bcr.bcr_solve(band, rhs)
    assert ok
    e = bcr.backward_error(band, x, rhs)
    es = bcr.backward_error(band, _scipy_solve(band, rhs), rhs)
    assert e <= BOUND and es <= BOUND, (e, es)
    return x


@pytest.mark.parametrize("scale_exp", [0.0, 6.0])
@pytest.mark.parametrize("hb", HBS)
def test_backward_error_over_block_multiples(hb, scale_exp):
    rng = np.random.default_rng([hb, int(scale_exp)])
    for n in sizes(hb):
        band = br.random_spd_band(n, hb, rng, scale_exp=scale_exp)
        _check(band, rng.normal(size=n))


@pytest.mark.parametrize("nt,span", [(6, 6), (15, 6), (15, 12), (15, 16)])
def test_backward_error_on_block_bands(nt, span):
    rng = np.random.default_rng([nt, span])
    for K in (span + 1, 3 * (span + 1) + 1, 40, 200):
        band = br.block_band(K, nt, span, rng)
        _check(band, rng.normal(size=band.shape[0]))


@pytest.mark.parametrize("hb", [104, 194, 256])
def test_backward_error_at_full_size(hb):
    """n = 51 855: the level-1 system of the 3 457-keyframe sample run"""
    rng = np.random.default_rng(hb)
    n = 51855
    band = br.random_spd_band(n, hb, rng)
    _check(band, rng.normal(size=n))


def test_small_cases_equal_dense_solve():
    rng = np.random.default_rng(5)
    for hb, n in ((0, 1), (0, 33), (1, 2), (5, 31), (5, 32), (5, 33), (5, 65), (5, 97), (41, 100)):
        band = br.random_spd_band(n, hb, rng)
        rhs = rng.normal(size=n)
        x, ok = bcr.bcr_solve(band, rhs)
        xd = np.linalg.solve(br.band_to_dense(np.where(np.isnan(band), 0.0, band)), rhs)
        assert ok and np.max(np.abs(x - xd)) <= 1e-12 * np.max(np.abs(xd))


@pytest.mark.parametrize("hb", [5, 41, 194])
def test_fails_on_indefinite_band_and_nan_diagonal(hb):
    rng = np.random.default_rng(hb + 1)
    b = bcr.block_size(hb)
    n = 5 * b + 3
    band = br.random_spd_band(n, hb, rng)
    rhs = rng.normal(size=n)
    for row in (0, 2 * b + 7, n - 1):                # first, middle and last block
        bad = band.copy(); bad[row, hb] = -abs(bad[row, hb]) * 1e3
        assert not bcr.bcr_solve(bad, rhs)[1]
        bad = band.copy(); bad[row, hb] = np.nan
        assert not bcr.bcr_solve(bad, rhs)[1]


def test_never_reads_slots_before_column_zero():
    rng = np.random.default_rng(9)
    for hb, n in ((41, 30), (104, 300), (256, 600)):
        band = br.random_spd_band(n, hb, rng)
        rhs = rng.normal(size=n)
        assert np.isnan(band[0, 0]) or hb == 0
        x, ok = bcr.bcr_solve(band, rhs)
        x0, ok0 = bcr.bcr_solve(np.where(np.isnan(band), 0.0, band), rhs)
        assert ok and ok0 and np.array_equal(x.view(np.uint64), x0.view(np.uint64))


def test_flop_count_follows_the_blocks():
    """one block: b^3/3 + 3 b^2; the count grows like 6 n b^2 for many blocks"""
    assert bcr.flops(10, 5) == 32 ** 3 / 3 + 3 * 32 * 32
    n, hb = 51855, 104
    b = bcr.block_size(hb)
    assert 4 * n * b * b < bcr.flops(n, hb) < 8 * n * b * b
