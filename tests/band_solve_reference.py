"""numpy restatement of K4 (glio_b200/csrc/band.cu, glio_band_solve): the band Cholesky factor-and-solve in exactly the device's
operation order, so the GPU tests can ask for bit-identical L and x.

The band is an (n, hb+1) float64 array in glio_batch_solve's layout: entry (i, j), i-hb <= j <= i, at band[i, j-i+hb].
  - Factorisation, right-looking, column j: l = sqrt(a_jj), linv = 1.0 / l, L_(j+t, j) = a_(j+t, j) * linv, then every trailing
    entry a_(j+t, j+1+u), 0 <= u < t <= min(hb, n-1-j), becomes a_(j+t, j+1+u) - L_(j+t, j) * L_(j+1+u, j).  An entry therefore
    receives its updates in ascending column order, one rounded product and one rounded difference each: the order of
    detail::cholesky_solve_scalar (solver.cpp).
  - Forward half, fused into the sweep: y_j = s_j / l, then s_(j+t) = s_(j+t) - L_(j+t, j) * y_j, s starting at b: the scalar
    forward solve's order.
  - Backward half, axpy form over descending rows: x_i = s_i / L_ii, then s_k = s_k - L_(i, k) * x_i for k = i-1 .. i-hb, s
    starting at y.
  - Failure: a pivot that is not positive and finite, or a non-finite x.
numpy's float64 +, -, *, / and sqrt are IEEE round-to-nearest and never fused, so each statement below is the device's rounding.
"""
import functools

import numpy as np


@functools.lru_cache(maxsize=None)
def _triangle(m):
    """(t, u) with 0 <= u < t <= m, as index arrays"""
    t = np.repeat(np.arange(1, m + 1), np.arange(1, m + 1))
    u = np.concatenate([np.arange(k) for k in range(1, m + 1)]) if m else np.zeros(0, np.int64)
    return t, u


def band_cholesky_solve(band, b):
    """-> (L, y, x, ok): L the factored band (a copy), y the forward half, x the solution.  On failure ok is False and the
    arrays hold partial results, as glio_band_solve's do (not the same ones)."""
    a = np.array(band, dtype=np.float64, copy=True)
    n, w = a.shape
    hb = w - 1
    s = np.array(b, dtype=np.float64, copy=True)
    y = np.zeros(n)
    for j in range(n):
        d = a[j, hb]
        if not (d > 0.0) or not np.isfinite(d):
            return a, y, y.copy(), False
        l = np.sqrt(d)
        linv = 1.0 / l
        a[j, hb] = l
        y[j] = s[j] / l
        m = min(hb, n - 1 - j)
        if m == 0:
            continue
        t = np.arange(1, m + 1)
        v = a[j + t, hb - t] * linv
        a[j + t, hb - t] = v
        s[j + t] = s[j + t] - v * y[j]
        tt, uu = _triangle(m)
        a[j + tt, hb + 1 + uu - tt] = a[j + tt, hb + 1 + uu - tt] - v[tt - 1] * v[uu]
    s = y.copy()
    x = np.zeros(n)
    for i in range(n - 1, -1, -1):
        x[i] = s[i] / a[i, hb]
        m = min(hb, i)
        if m:
            t = np.arange(1, m + 1)
            s[i - t] = s[i - t] - a[i, hb - t] * x[i]
    return a, y, x, bool(np.all(np.isfinite(x)))


def _offsets(n, hb):
    """(i, j) index grids of the band layout and the mask of its slots with j >= 0"""
    i = np.arange(n)[:, None]
    j = i - hb + np.arange(hb + 1)[None, :]
    return i, j, j >= 0


def band_scale(H, s):
    """k_band_scale: (Hs, hs_diag), Hs_ij = (H_ij * s_i) * s_j on the slots with j >= 0; the others hold 0.0 here (the device
    leaves them unspecified)"""
    n, w = H.shape
    i, j, ok = _offsets(n, w - 1)
    Hs = np.zeros((n, w))
    Hs[ok] = (H[ok] * s[np.broadcast_to(i, ok.shape)[ok]]) * s[j[ok]]
    return Hs, Hs[:, w - 1].copy()


def band_shift(Hs, v):
    """k_band_shift: A = Hs + diag(v * v)"""
    A = np.array(Hs, dtype=np.float64, copy=True)
    A[:, -1] = Hs[:, -1] + v * v
    return A


def band_symv(Hs, x):
    """k_band_symv: y = Hs x in the kernel's order.  Row i starts from 0.0 and adds, one rounded product and one rounded sum per
    term, the columns max(0, i-hb) .. i from row i, then i+1 .. min(n-1, i+hb) from the rows below.  The sum never becomes -0.0, so
    adding +0.0 in place of a term outside the matrix changes no bit; every row therefore runs the same 2hb+1 terms."""
    n, w = Hs.shape
    hb = w - 1
    rows = np.arange(n)
    y = np.zeros(n)
    for d in range(-hb, hb + 1):                    # column j = i + d, ascending
        j = rows + d
        valid = (j >= 0) & (j < n)
        jc = np.clip(j, 0, n - 1)
        h = Hs[rows, hb + d] if d <= 0 else Hs[jc, hb - d]
        y = y + np.where(valid, np.where(valid, h, 0.0) * x[jc], 0.0)
    return y


def band_to_dense(band):
    """the symmetric dense matrix of a lower band"""
    n, w = band.shape
    hb = w - 1
    A = np.zeros((n, n))
    for i in range(n):
        for j in range(max(0, i - hb), i + 1):
            A[i, j] = A[j, i] = band[i, j - i + hb]
    return A


PREFETCH = 8                                        # kBandPrefetch: K4's ring holds R = hb + 1 + PREFETCH rows


def ring_edge_sizes(hb):
    """the sizes where K4's ring is most fragile: n = hb+1 .. hb+18 (the prologue loads every row up to n = R-1 and the sweep's
    own loads start just above) and n = 2R-1, 2R, 2R+1 (every slot refilled once)"""
    R = hb + 1 + PREFETCH
    return sorted(set(range(hb + 1, hb + 19)) | {2 * R - 1, 2 * R, 2 * R + 1})


def block_band(K, nt, span, rng, zero_frac=0.4):
    """a positive definite band shaped like the batch normal equations: K blocks of nt columns, half bandwidth (span+1) nt - 1,
    nt x nt blocks coupling keyframes up to span apart, of which about zero_frac are whole zero blocks, and the last nt - 6 columns
    of every block row empty (speed-bias columns without a factor) but for the diagonal.  Slots with j < 0 hold NaN."""
    n, hb = K * nt, min((span + 1) * nt - 1, K * nt - 1)
    band = np.zeros((n, hb + 1))
    for ka in range(K):
        for kb in range(max(0, ka - span), ka + 1):
            if ka != kb and rng.uniform() < zero_frac:
                continue
            blk = rng.uniform(-1.0, 1.0, (nt, nt))
            blk[:, 6:] = 0.0; blk[6:, :] = 0.0
            for p in range(nt):
                for q in range(nt):
                    i, j = nt * ka + p, nt * kb + q
                    if j <= i:
                        band[i, j - i + hb] = blk[p, q]
    i = np.arange(n)[:, None]
    j = i - hb + np.arange(hb + 1)[None, :]
    off = (j >= 0) & (j < i)
    rowsum = np.zeros(n)
    np.add.at(rowsum, np.broadcast_to(i, band.shape)[off], np.abs(band[off]))
    np.add.at(rowsum, j[off], np.abs(band[off]))
    band[:, hb] = rowsum + rng.uniform(1e-3, 1.0, n)
    band[j < 0] = np.nan
    return band


def random_spd_band(n, hb, rng, scale_exp=0.0):
    """a diagonally dominant (so positive definite) band, symmetrically scaled by D = diag(10^U(-scale_exp, scale_exp)): with
    scale_exp = 6 its diagonal spans about 1e-12 .. 1e12.  Slots with j < 0 hold NaN, which no path may read."""
    a = rng.uniform(-1.0, 1.0, size=(n, hb + 1))
    i = np.arange(n)[:, None]
    j = i - hb + np.arange(hb + 1)[None, :]
    off = (j >= 0) & (j < i)
    rowsum = np.zeros(n)
    np.add.at(rowsum, np.broadcast_to(i, a.shape)[off], np.abs(a[off]))
    np.add.at(rowsum, j[off], np.abs(a[off]))
    a[:, hb] = rowsum + 1.0 + rng.uniform(0.0, 1.0, size=n)
    dsc = 10.0 ** rng.uniform(-scale_exp, scale_exp, size=n)
    a = a * dsc[:, None] * dsc[np.clip(j, 0, None)]
    a[j < 0] = np.nan
    return a
