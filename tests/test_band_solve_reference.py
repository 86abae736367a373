"""tests/band_solve_reference.py, the numpy restatement of K4's operation order that the GPU tests hold glio_band_solve to: its
factor and forward half equal a literal transliteration of detail::cholesky_solve_scalar (solver.cpp) bit for bit, its solution
is within the backward-error bound of scipy's banded Cholesky solve, and it fails where the host path fails.  The compiled
cholesky_solve_scalar (tests/cpp/band_chol_dump.cpp) gives its L and y bit for bit, and band_symv, the order of k_band_symv, is
within the a-priori bound of a longdouble product."""
import math
import os

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


def _host_backward(L, y):
    """cholesky_solve_scalar's backward substitution, statement for statement: dot form, ascending k"""
    n, w = L.shape
    hb = w - 1
    x = [0.0] * n
    for i in range(n - 1, -1, -1):
        s = float(y[i])
        for k in range(i + 1, min(n, i + hb + 1)):
            s -= float(L[k, hb - k + i]) * x[k]
        x[i] = s / float(L[i, hb])
    return np.array(x)


def _compiled_fixtures():
    """(name, band, b): the ring-edge sizes of K4 over its half bandwidths, bands shaped like the batch normal equations (whole zero
    blocks, empty speed-bias columns), a system that fails at its last pivot and one that fails at its first"""
    out = []
    for hb in (0, 1, 7, 8, 9, 41, 104, 160):
        sizes = br.ring_edge_sizes(hb)
        for n in sorted({sizes[0], sizes[8], sizes[17], *sizes[-3:]}):
            rng = np.random.default_rng([hb, n])
            out.append((f"ring hb={hb} n={n}", br.random_spd_band(n, hb, rng, 6), rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)))
    for K, nt, span in ((40, 6, 6), (12, 15, 6), (7, 15, 2)):
        rng = np.random.default_rng([K, nt, span])
        out.append((f"blocks K={K} nt={nt}", br.block_band(K, nt, span, rng), rng.standard_normal(K * nt)))
    rng = np.random.default_rng(77)
    last = br.random_spd_band(60, 9, rng); last[59, 9] = -last[59, 9]
    first = br.random_spd_band(60, 9, rng); first[0, 9] = 0.0
    out += [("fails at n-1", last, np.ones(60)), ("fails at 0", first, np.ones(60))]
    return out


def test_compiled_scalar_host_path_equals_the_reference(tmp_path):
    """the compiled detail::cholesky_solve_scalar (libglio_b200.so), not a transliteration of it: its L is band_cholesky_solve's bit
    for bit, and its x is its own dot-form back-substitution applied to band_cholesky_solve's y, bit for bit"""
    import struct
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, "glio_b200")
    exe = str(tmp_path / "band_chol_dump")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", os.path.join(root, "tests", "cpp", "band_chol_dump.cpp"), "-o", exe,
                           "-L", lib, "-lglio_b200", "-Wl,-rpath," + lib,
                           "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    fixtures = _compiled_fixtures()
    blob = b"".join(struct.pack("<ii", *band.shape[:1], band.shape[1] - 1) + band.astype("<f8").tobytes() + b.astype("<f8").tobytes()
                    for _, band, b in fixtures)
    out = subprocess.run([exe], input=blob, capture_output=True, check=True).stdout
    pos = 0
    for name, band, b in fixtures:
        n, w = band.shape
        ok = struct.unpack_from("<i", out, pos)[0]; pos += 4
        L_host = np.frombuffer(out, "<f8", n * w, pos).reshape(n, w); pos += 8 * n * w
        x_host = np.frombuffer(out, "<f8", n, pos); pos += 8 * n
        L, y, x, ok_ref = br.band_cholesky_solve(band, b)
        assert bool(ok) == ok_ref, name
        if not ok_ref:
            continue
        assert np.array_equal(_bits(L_host), _bits(L)), f"{name}: L differs at {np.argwhere(_bits(L_host) != _bits(L))[:5].tolist()}"
        assert np.array_equal(_bits(x_host), _bits(_host_backward(L, y))), f"{name}: y differs"
    assert pos == len(out)
    assert sum(not br.band_cholesky_solve(band, b)[3] for _, band, b in fixtures) == 2


@pytest.mark.parametrize("n,hb", [(1, 0), (2, 1), (3, 5), (40, 0), (257, 5), (300, 104), (500, 160)])
def test_band_symv_within_a_priori_bound(n, hb):
    """band_symv (k_band_symv's order) against a longdouble product, within (2hb+1) 2^-53 sum |Hs_ij| |x_j| per row, with scales
    and x spanning 1e-150 .. 1e150; band_scale and band_shift against their dense definitions"""
    rng = np.random.default_rng([n, hb])
    H = br.random_spd_band(n, hb, rng)
    s = 10.0 ** rng.uniform(-150, 150, n)
    x = rng.uniform(-1.0, 1.0, n) * 10.0 ** rng.uniform(-3, 3, n) / s         # spans 1e-150 .. 1e150, Hs x stays finite
    Hs, hs_diag = br.band_scale(H, s)
    y = br.band_symv(Hs, x)
    D = br.band_to_dense(Hs)
    ld = D.astype(np.longdouble) @ x.astype(np.longdouble)
    mag = np.abs(D) @ np.abs(x)
    assert np.all(np.isfinite(y)) and np.all(mag > 0)
    assert np.all(np.abs(y.astype(np.longdouble) - ld) <= (2 * hb + 1) * 2.0 ** -53 * mag.astype(np.longdouble))
    dense = br.band_to_dense(np.nan_to_num(H))
    assert np.allclose(D, (s[:, None] * dense) * s[None, :], rtol=4 * np.finfo(float).eps, atol=np.finfo(float).tiny)
    assert np.array_equal(hs_diag, np.diag(D))
    v = 10.0 ** rng.uniform(-100, 100, n)
    A = br.band_shift(Hs, v)
    assert np.array_equal(A[:, :-1], Hs[:, :-1]) and np.array_equal(A[:, -1], Hs[:, -1] + v * v)


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
