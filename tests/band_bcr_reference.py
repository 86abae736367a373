"""numpy restatement of the band solve by block cyclic reduction (glio_b200/csrc/bcr.cu, glio_band_solve_bcr, GLIO_FACTOR_BCR).

The band is an (n, hb+1) float64 array in glio_batch_solve's layout: entry (i, j), i-hb <= j <= i, at band[i, j-i+hb].
  - Blocks of b = 32 * ceil(max(hb, 1) / 32) rows (block_size), m = ceil(n / b); block i covers rows [i b, (i+1) b).  The rows past
    n are padded with an identity diagonal and a zero right-hand side.  D_i is the diagonal block, E_i = A[block i+1, block i], r_i
    the right-hand side.  Only slots with j >= 0 are read.
  - Level l (s = 2^l) holds the blocks 0, s, 2s, ... < m in the original numbering.  Its odd blocks k (k / s odd) are eliminated:
    D_k = L L^T, Ut = E_(k-s)^T L^-T, Vt = E_k L^-T (when k+s < m), w = L^-1 r_k.  Then every even block j is updated, left
    neighbour first: D_j -= Vt_(j-s) Vt_(j-s)^T, D_j -= Ut_(j+s) Ut_(j+s)^T, r_j -= Vt_(j-s) w_(j-s), r_j -= Ut_(j+s) w_(j+s), and
    E_j = -Vt_(j+s) Ut_(j+s)^T when j+2s < m.  When s >= m, block 0 is factored and solved.
  - Back-substitution in reverse level order: x_k = L^-T (w_k - Ut_k^T x_(k-s) - Vt_k^T x_(k+s)).
  - Failure: a block Cholesky that meets a pivot that is not positive and finite, or a non-finite x.
The block order is the device's; the dense work inside a block (numpy's Cholesky, triangular solves and products) sums in another
order, so the device is held to this reference by a tolerance, not bit for bit.
"""
import numpy as np
import scipy.linalg


def block_size(hb):
    return 32 * ((max(hb, 1) + 31) // 32)


def gather(band, rhs):
    """-> (D (m, b, b) symmetric, E (m, b, b), r (m, b), b); reads only the slots with j >= 0"""
    n, w = band.shape
    hb = w - 1
    b = block_size(hb)
    m = -(-n // b)
    D = np.zeros((m, b, b)); E = np.zeros((m, b, b)); r = np.zeros((m, b))
    r.reshape(-1)[:n] = rhs
    i = np.arange(n)
    for d in range(hb + 1):                          # entry (i, i-d)
        ii = i[i >= d]
        jj = ii - d
        val = band[ii, hb - d]
        ki, p, kj, q = ii // b, ii % b, jj // b, jj % b
        same = ki == kj
        D[ki[same], p[same], q[same]] = val[same]
        D[kj[same], q[same], p[same]] = val[same]
        E[kj[~same], p[~same], q[~same]] = val[~same]
    pad = np.arange(n, m * b)
    D[pad // b, pad % b, pad % b] = 1.0
    return D, E, r, b


def _chol(A):
    """lower Cholesky factor, or None when a pivot is not positive and finite"""
    if not np.all(np.isfinite(A)):
        return None
    try:
        L = np.linalg.cholesky(A)
    except np.linalg.LinAlgError:
        return None
    return L if np.all(np.isfinite(L)) and np.all(np.diag(L) > 0) else None


def _rsolve(L, M):
    """M L^-T (row solves y L^T = M_row)"""
    return scipy.linalg.solve_triangular(L, M.T, lower=True, check_finite=False).T


def bcr_solve(band, rhs):
    """-> (x, ok).  On failure x is None."""
    band = np.asarray(band, np.float64)
    n = band.shape[0]
    D, E, r, b = gather(band, np.asarray(rhs, np.float64).reshape(n))
    m = D.shape[0]
    U = np.zeros_like(D)
    s = 1
    while s < m:
        for k in range(s, m, 2 * s):
            L = _chol(D[k])
            if L is None:
                return None, False
            D[k] = L
            U[k] = _rsolve(L, E[k - s].T)
            if k + s < m:
                E[k] = _rsolve(L, E[k])
            r[k] = scipy.linalg.solve_triangular(L, r[k], lower=True, check_finite=False)
        for j in range(0, m, 2 * s):
            lft, rgt = j - s, j + s
            if lft >= 0:
                D[j] = D[j] - E[lft] @ E[lft].T
            if rgt < m:
                D[j] = D[j] - U[rgt] @ U[rgt].T
            if lft >= 0:
                r[j] = r[j] - E[lft] @ r[lft]
            if rgt < m:
                r[j] = r[j] - U[rgt] @ r[rgt]
            if j + 2 * s < m:
                E[j] = -(E[rgt] @ U[rgt].T)
        s *= 2
    L = _chol(D[0])
    if L is None:
        return None, False
    X = np.zeros((m, b))
    X[0] = scipy.linalg.solve_triangular(L, scipy.linalg.solve_triangular(L, r[0], lower=True, check_finite=False), lower=True,
                                         trans="T", check_finite=False)
    s //= 2
    while s >= 1:
        for k in range(s, m, 2 * s):
            t = r[k] - U[k].T @ X[k - s]
            if k + s < m:
                t = t - E[k].T @ X[k + s]
            X[k] = scipy.linalg.solve_triangular(D[k], t, lower=True, trans="T", check_finite=False)
        s //= 2
    x = X.reshape(-1)[:n].copy()
    return x, bool(np.all(np.isfinite(x)))


def flops(n, hb):
    """the floating-point operations of one device factor-and-solve, counted from its kernels' useful work: per eliminated block a
    Cholesky (b^3 / 3), the row solves of Ut, Vt and w (b^2 each row), the updates of its even neighbours (b^3 per symmetric block
    product, 2 b^3 per coupling product, 2 b^2 per right-hand-side product) and its back-substitution (2 b^2 per neighbour and b^2)"""
    b = block_size(hb)
    m = -(-n // b)
    f = 0.0
    s = 1
    while s < m:
        for k in range(s, m, 2 * s):
            nbr = 1 + (k + s < m)
            f += b ** 3 / 3 + (nbr * b + 1) * b * b            # potrf, trsm
            f += nbr * (b ** 3 + 2 * b * b)                     # the neighbours' D and r updates
            f += 2 * b ** 3 if k + s < m else 0.0               # the new coupling
            f += nbr * 2 * b * b + b * b                        # back-substitution
        s *= 2
    return f + b ** 3 / 3 + 3 * b * b


def backward_error(band, x, rhs):
    """||A x - b||_inf / (||A||_inf ||x||_inf + ||b||_inf) for the symmetric band"""
    from tests.band_solve_reference import band_symv
    band = np.asarray(band, np.float64)
    n, w = band.shape
    hb = w - 1
    Hs = np.where(np.isnan(band), 0.0, band)
    res = band_symv(Hs, x) - rhs
    absrow = band_symv(np.abs(Hs), np.ones(n))
    return float(np.max(np.abs(res)) / (np.max(absrow) * np.max(np.abs(x)) + np.max(np.abs(rhs))))
