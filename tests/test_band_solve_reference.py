"""tests/band_solve_reference.py, the numpy restatement of K4's operation order that the GPU tests hold glio_band_solve to: its
factor and forward half equal a literal transliteration of detail::cholesky_solve_scalar (solver.cpp) bit for bit, its solution
is within the backward-error bound of scipy's banded Cholesky solve, and it fails where the host path fails."""
import math

import numpy as np
import pytest
import scipy.linalg

from tests import band_solve_reference as br


def _scalar_host(band, b):
    """cholesky_solve_scalar's factor and forward solve, statement for statement, on a flat copy of the band (Python floats
    are IEEE doubles; nothing is fused)"""
    n, w = band.shape
    hb = w - 1
    a = [float(v) for v in band.reshape(-1)]
    col = [0.0] * (hb + 2)
    for j in range(n):
        d = a[j * w + hb]
        if not (d > 0.0) or not math.isfinite(d):
            return None, None
        l = math.sqrt(d)
        a[j * w + hb] = l
        m = min(hb, n - 1 - j)
        linv = 1.0 / l
        for t in range(1, m + 1):
            e = (j + t) * w + hb - t
            a[e] *= linv
            col[t] = a[e]
        for t in range(1, m + 1):
            ri = (j + t) * w + hb - t + 1
            c = col[t]
            for u in range(t):
                a[ri + u] -= c * col[1 + u]
    x = [0.0] * n
    for i in range(n):
        ri = i * w + hb - i
        s = float(b[i])
        for k in range(max(0, i - hb), i):
            s -= a[ri + k] * x[k]
        x[i] = s / a[ri + i]
    return np.array(a).reshape(n, w), np.array(x)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("n,hb,scale", [(1, 0, 0), (2, 1, 0), (7, 1, 3), (7, 5, 6), (12, 5, 6), (30, 6, 0), (40, 11, 6),
                                        (3, 5, 0), (5, 4, 6), (64, 17, 2)])
def test_factor_and_forward_equal_the_scalar_host_path(n, hb, scale):
    rng = np.random.default_rng(1000 * n + hb)
    band = br.random_spd_band(n, hb, rng, scale)
    b = rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)
    L_host, y_host = _scalar_host(band, b)
    L, y, x, ok = br.band_cholesky_solve(band, b)
    assert ok
    assert np.array_equal(_bits(L), _bits(L_host))          # NaN slots (j < 0) are untouched on both sides
    assert np.array_equal(_bits(y), _bits(y_host))


@pytest.mark.parametrize("n,hb,scale", [(50, 3, 0), (400, 41, 0), (300, 104, 0), (200, 12, 6), (1000, 29, 3)])
def test_solution_within_backward_error_bound(n, hb, scale):
    rng = np.random.default_rng(7 * n + hb)
    band = br.random_spd_band(n, hb, rng, scale)
    b = rng.standard_normal(n)
    L, y, x, ok = br.band_cholesky_solve(band, b)
    assert ok
    # scipy's upper-form band: ab[hb + i - j, j] = A[i, j] for i <= j
    ab = np.zeros((hb + 1, n))
    for k in range(hb + 1):                      # ab row hb - k: the k-th super-diagonal, A[j - k, j] = band[j, hb - k]
        ab[hb - k, k:] = band[k:, hb - k]
    x_sp = scipy.linalg.solveh_banded(ab, b)
    A = br.band_to_dense(np.nan_to_num(band))
    absA = np.abs(A)

    def componentwise_backward_error(z):
        return np.max(np.abs(b - A @ z) / (absA @ np.abs(z) + np.abs(b)))

    # Cholesky is componentwise backward stable: |dA| <= gamma_(hb+1) |L||L^T|, and with a diagonally dominant A,
    # |L||L^T| stays within a small multiple of |A|; (4 (hb + 2) eps) covers the factor, both substitutions and the check itself
    bound = 4 * (hb + 2) * np.finfo(float).eps
    assert componentwise_backward_error(x) <= bound
    assert componentwise_backward_error(x_sp) <= bound
    assert np.max(np.abs(x - x_sp)) <= 1e-9 * np.max(np.abs(x_sp))


def test_fails_on_an_indefinite_band():
    rng = np.random.default_rng(3)
    band = br.random_spd_band(40, 6, rng)
    band[20, 6] = -band[20, 6]                   # a negative diagonal entry: some pivot at or before column 20 is not positive
    assert not br.band_cholesky_solve(band, np.ones(40))[3]
    ind = br.random_spd_band(40, 6, rng)
    ind[25, 5] = 10.0 * ind[25, 6]               # |A_25,24| far above sqrt(A_25,25 A_24,24): indefinite, diagonal positive
    assert not br.band_cholesky_solve(ind, np.ones(40))[3]


@pytest.mark.parametrize("where", ["diagonal", "off", "rhs"])
def test_fails_on_a_nan_entry(where):
    rng = np.random.default_rng(4)
    band = br.random_spd_band(30, 4, rng)
    b = np.ones(30)
    if where == "diagonal":
        band[17, 4] = np.nan
    elif where == "off":
        band[17, 2] = np.nan
    else:
        b[9] = np.nan
    assert not br.band_cholesky_solve(band, b)[3]
