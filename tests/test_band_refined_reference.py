"""tests/band_refined_reference.py, the extended-precision reference the BCR edge tests hold the device to: its refined x is the
50-digit solution to the last bits up to kappa = 1e12; its condition estimate tracks numpy's; its generators reach their condition
numbers, and the indefinite ones are indefinite with positive definite diagonal blocks; and the numpy restatement of block cyclic
reduction (tests/band_bcr_reference.py) meets the backward- and forward-error bars of tests/test_gpu_band_bcr_edges.py on them,
which calibrates those bars before any device run."""
import mpmath
import numpy as np
import pytest

from tests import band_bcr_reference as bcr
from tests import band_refined_reference as rr
from tests import band_solve_reference as br

KAPPAS = [1.0, 1e4, 1e8, 1e12]


def bars(hb):
    """(backward bar, forward bar per unit kappa): 4 (b + 2) eps, b BCR's block size"""
    c = 4 * (bcr.block_size(hb) + 2) * rr.EPS
    return c, c


def make(kind, n, hb, rng, kappa):
    """a factor_band or gauge_band of condition number about kappa"""
    if kind == "factor":
        return rr.factor_band(n, hb, rng, np.log10(kappa) / 2)
    A = rr.gauge_band(n, hb, rng, 0.0)
    A[:, hb] += max(rr.norm1(A), 1.0) / kappa
    return A


def _dense(band):
    return br.band_to_dense(np.nan_to_num(band))


@pytest.mark.parametrize("kind", ["factor", "gauge"])
@pytest.mark.parametrize("kappa", [1e2, 1e6, 1e9, 1e12])
def test_refined_solve_equals_50_digit_solve(kind, kappa):
    rng = np.random.default_rng([int(np.log10(kappa)), len(kind)])
    mpmath.mp.dps = 50
    for n, hb in ((1, 0), (7, 3), (40, 1), (64, 31), (120, 5)):
        A = make(kind, n, hb, rng, kappa)
        b = rng.normal(size=n)
        x, converged = rr.refined_solve(A, b)
        assert converged, (n, hb)
        xm = mpmath.lu_solve(mpmath.matrix(_dense(A).tolist()), mpmath.matrix(b.tolist()))
        xm = np.array([float(v) for v in xm])
        err = np.max(np.abs(x - xm)) / np.max(np.abs(xm))
        assert err <= 2 * np.finfo(float).eps, (n, hb, err)


@pytest.mark.parametrize("kind", ["factor", "gauge"])
def test_cond_estimate_tracks_numpy(kind):
    rng = np.random.default_rng(len(kind))
    for n, hb in ((1, 0), (2, 1), (50, 0), (300, 5), (1000, 41), (2000, 129)):
        for kappa in KAPPAS:
            A = make(kind, n, hb, rng, kappa)
            est, ref = rr.cond_estimate(A), np.linalg.cond(_dense(A))
            assert ref / 10 <= est <= ref * 10, (n, hb, kappa, est, ref)


@pytest.mark.parametrize("kind", ["factor", "gauge"])
def test_generators_reach_their_condition_numbers(kind):
    """factor_band within a factor 9 of the target, gauge_band within a factor 2 (either way, up to the estimate's own error)"""
    rng = np.random.default_rng(len(kind) + 1)
    lo, hi = (1 / 9, 9) if kind == "factor" else (1 / 2, 2)
    for n, hb in ((64, 1), (500, 33), (2000, 225)):
        for kappa in KAPPAS:
            A = make(kind, n, hb, rng, kappa)
            assert not np.any(np.isnan(A[:, hb])) and np.all(np.isnan(A[0, :hb]))
            k = np.linalg.cond(_dense(A))
            assert kappa * lo <= k <= max(kappa * hi, 2.0), (n, hb, kappa, k)
            if kind == "factor" and kappa >= 1e4:   # not diagonally dominant (a gauge band is, weakly: a Laplacian plus delta I)
                D = _dense(A)
                assert np.any(2 * np.abs(np.diag(D)) < np.abs(D).sum(axis=1)), (n, hb, kappa)


@pytest.mark.parametrize("where", rr.SCHUR_WHERE)
@pytest.mark.parametrize("hb", [1, 5, 33, 64])
def test_schur_indefinite_bands(hb, where):
    """lambda_min < 0 (clearly: far beyond 100 n eps ||A||) with every diagonal block positive definite; K4's order and BCR's
    restatement both fail, BCR's at the level schur_pair names (its Cholesky of the blocks eliminated before succeeds)"""
    rng = np.random.default_rng([hb, len(where)])
    b = bcr.block_size(hb)
    for n in (5 * b + 1, 8 * b - 1):
        A = rr.schur_indefinite_band(n, hb, rng, where)
        D = _dense(A)
        lam = np.linalg.eigvalsh(D)[0]
        assert lam < -100 * n * rr.EPS * rr.norm1(A), (n, lam)
        for k in range(-(-n // b)):
            blk = D[k * b:(k + 1) * b, k * b:(k + 1) * b]
            assert np.linalg.eigvalsh(blk)[0] > 0, (n, k)
        rhs = rng.normal(size=n)
        assert not bcr.bcr_solve(A, rhs)[1]
        assert not br.band_cholesky_solve(A, rhs)[3]
        p, level = rr.schur_pair(where)
        # the blocks BCR eliminates before the failing one: every odd block (level 0), then the levels below `level`; their
        # principal submatrix is positive definite, and adding the failing block p makes it indefinite
        before = [k for k in range(1, -(-n // b)) if level is None or (k & -k) < (1 << level)]
        rows = np.concatenate([np.arange(k * b, min(n, (k + 1) * b)) for k in before])
        assert np.linalg.eigvalsh(D[np.ix_(rows, rows)])[0] > 0
        rows_p = np.sort(np.concatenate([rows, np.arange(p * b, (p + 1) * b)]))
        assert np.linalg.eigvalsh(D[np.ix_(rows_p, rows_p)])[0] < 0


@pytest.mark.parametrize("kind", ["factor", "gauge"])
@pytest.mark.parametrize("hb", [0, 1, 33, 129, 256])
def test_bcr_restatement_meets_the_bars(kind, hb):
    """the numpy block cyclic reduction: backward error <= 4 (b+2) eps and forward error <= 4 (b+2) eps kappa against
    refined_solve, over the sizes and condition numbers of the device tests"""
    from tests.test_band_bcr_reference import sizes
    rng = np.random.default_rng([hb, len(kind), 2])
    back, fwd = bars(hb)
    for n in sorted({1, 2, max(hb, 1), hb + 1} | set(sizes(hb))):
        for kappa in KAPPAS:
            A = make(kind, n, hb, rng, kappa)
            rhs = rng.normal(size=n)
            x, ok = bcr.bcr_solve(A, rhs)
            xr, conv = rr.refined_solve(A, rhs)
            k = rr.cond_estimate(A)
            assert ok and conv, (n, kappa)
            assert rr.backward_error(A, x, rhs) <= back, (n, kappa)
            assert np.max(np.abs(x - xr)) <= fwd * k * np.max(np.abs(xr)), (n, kappa)


def test_backward_error_in_longdouble():
    """the residual is formed in longdouble: a perturbation of one ulp in x shows, and the exact solution of a diagonal band is 0"""
    A = np.array([[2.0], [4.0], [8.0]])
    b = np.array([1.0, 1.0, 1.0])
    assert rr.backward_error(A, b / A[:, 0], b) == 0.0
    x = b / A[:, 0]
    x[0] = np.nextafter(x[0], 1.0)
    assert 0.0 < rr.backward_error(A, x, b) < 1e-15
