"""An extended-precision reference for symmetric positive definite band solves, and bands that are hard to solve.

The band is an (n, hb+1) float64 array in glio_batch_solve's layout: entry (i, j), i-hb <= j <= i, at band[i, j-i+hb]; slots with
j < 0 are never read (the generators below fill them with NaN).
  - refined_solve: LAPACK's banded Cholesky (scipy.linalg.cholesky_banded / cho_solve_banded), then iterative refinement with x
    kept as an unevaluated sum x_hi + x_lo and the residual b - A x formed without rounding error in its products and sums
    (Dekker's two-product and Knuth's two-sum, the 2-term "Dot2" of Ogita, Rump and Oishi).  A residual rounded once per term,
    even in longdouble, would limit the refined x to about kappa * 2^-64 relative: 1e-7 at kappa = 1e12, far from the last bit.
    With the doubled residual each step shrinks the error by about kappa * eps, down to the rounding of x itself.
  - backward_error: the normwise ||b - A x||_inf / (||A||_inf ||x||_inf + ||b||_inf), in longdouble.
  - cond_estimate: kappa_1 = ||A||_1 ||A^-1||_1, the second factor by scipy's onenormest through the banded Cholesky.  A is
    symmetric, so kappa_1 = kappa_inf.
  - factor_band, gauge_band, schur_indefinite_band: positive definite bands that are not diagonally dominant (conditioned from
    1 to 1e12, and singular but for a shift as the batch normal equations without a gauge prior are), and indefinite bands whose
    diagonal blocks are all positive definite.
"""
import numpy as np
import scipy.linalg
import scipy.sparse.linalg

from tests.band_bcr_reference import block_size

EPS = np.finfo(np.float64).eps / 2                  # 2^-53, the unit roundoff
_SPLIT = 134217729.0                                # 2^27 + 1: Veltkamp's splitter for float64
_CHUNK = 1 << 18                                    # residual rows per pass: n of about 4 M stays in memory


def lapack_band(band):
    """the lower band in LAPACK's layout: ab[d, j] = A[j+d, j]"""
    n, w = band.shape
    hb = w - 1
    ab = np.zeros((w, n))
    for d in range(min(w, n)):
        ab[d, :n - d] = band[d:, hb - d]
    return ab


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = _SPLIT * a
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _residual(band, x_hi, x_lo, rhs):
    """b - A (x_hi + x_lo), rounded once at the end: every product a x_hi is exact (two-product), the sums are carried as two-sums,
    and the a x_lo terms (2^-53 of the others) are added in float64"""
    n, w = band.shape
    hb = w - 1
    A = np.nan_to_num(band)
    out = np.empty(n)
    for r0 in range(0, n, _CHUNK):
        rows = np.arange(r0, min(n, r0 + _CHUNK))
        s = rhs[rows].astype(np.float64).copy()
        c = np.zeros(len(rows))
        for d in range(-hb, hb + 1):                # column j = i + d
            j = rows + d
            valid = (j >= 0) & (j < n)
            jc = np.clip(j, 0, n - 1)
            a = np.where(valid, A[rows, hb + d] if d <= 0 else A[jc, hb - d], 0.0)
            p, e = _two_prod(a, x_hi[jc])
            s, t = _two_sum(s, -p)
            c += t - e - a * x_lo[jc]
        out[rows] = s + c
    return out


def refined_solve(band, rhs, max_steps=40):
    """-> (x_ref, converged): A x = b by the banded Cholesky and iterative refinement with a doubled residual, stopping once the
    correction is below 2^-60 of ||x||_inf.  converged is False when the factorisation fails or the corrections do not get there."""
    band = np.asarray(band, np.float64)
    rhs = np.asarray(rhs, np.float64).reshape(len(band))
    try:
        c = scipy.linalg.cholesky_banded(lapack_band(np.nan_to_num(band)), lower=True, check_finite=False)
    except np.linalg.LinAlgError:
        return None, False
    solve = lambda r: scipy.linalg.cho_solve_banded((c, True), r, check_finite=False)
    x_hi = solve(rhs)
    x_lo = np.zeros_like(x_hi)
    if not np.all(np.isfinite(x_hi)):
        return None, False
    last = np.inf
    for _ in range(max_steps):
        dx = solve(_residual(band, x_hi, x_lo, rhs))
        size = np.max(np.abs(dx))
        if not size < last / 2:                     # stagnating (kappa eps near 1) or not finite
            return x_hi, False
        last = size
        x_hi, t = _two_sum(x_hi, dx)
        x_lo = x_lo + t
        x_hi, x_lo = _two_sum(x_hi, x_lo)
        if size <= 2.0 ** -60 * np.max(np.abs(x_hi)):
            return x_hi, True
    return x_hi, False


def backward_error(band, x, rhs):
    """||b - A x||_inf / (||A||_inf ||x||_inf + ||b||_inf) in longdouble, A the symmetric band; rows in chunks"""
    band = np.asarray(band, np.float64)
    n, w = band.shape
    hb = w - 1
    xl = np.asarray(x, np.float64).astype(np.longdouble)
    b = np.asarray(rhs, np.float64).reshape(n)
    rmax = np.longdouble(0)
    amax = np.longdouble(0)
    for r0 in range(0, n, _CHUNK):
        rows = np.arange(r0, min(n, r0 + _CHUNK))
        r = b[rows].astype(np.longdouble)
        rowabs = np.zeros(len(rows), np.longdouble)
        for d in range(-hb, hb + 1):
            j = rows + d
            valid = (j >= 0) & (j < n)
            jc = np.clip(j, 0, n - 1)
            h = np.where(valid, band[rows, hb + d] if d <= 0 else band[jc, hb - d], 0.0)
            h = np.nan_to_num(h).astype(np.longdouble)
            r -= h * xl[jc]
            rowabs += np.abs(h)
        rmax = max(rmax, np.max(np.abs(r)))
        amax = max(amax, np.max(rowabs))
    return float(rmax / (amax * np.max(np.abs(xl)) + np.max(np.abs(b))))


def norm1(band):
    """||A||_1 = ||A||_inf of the symmetric band"""
    n, w = band.shape
    hb = w - 1
    A = np.abs(np.nan_to_num(band))
    s = A.sum(axis=1)                               # the row's own part, columns i-hb .. i
    for d in range(1, min(w, n)):                   # and entry (i+d, i) for the columns right of the diagonal
        s[:n - d] += A[d:, hb - d]
    return float(np.max(s))


def cond_estimate(band):
    """kappa_1(A) = ||A||_1 * onenormest(A^-1), A^-1 applied through the banded Cholesky; inf when that Cholesky fails"""
    band = np.asarray(band, np.float64)
    n = len(band)
    try:
        c = scipy.linalg.cholesky_banded(lapack_band(np.nan_to_num(band)), lower=True, check_finite=False)
    except np.linalg.LinAlgError:
        return np.inf
    solve = lambda r: scipy.linalg.cho_solve_banded((c, True), r, check_finite=False)
    op = scipy.sparse.linalg.LinearOperator((n, n), matvec=solve, rmatvec=solve, matmat=solve, dtype=np.float64)
    inv = scipy.sparse.linalg.onenormest(op) if n > 1 else abs(solve(np.ones(1))[0])
    return norm1(band) * float(inv)


def _nan_outside(band):
    n, w = band.shape
    j = np.arange(n)[:, None] - (w - 1) + np.arange(w)[None, :]
    band[j < 0] = np.nan
    return band


def _gram(Lb):
    """the lower band of L L^T for the lower band L (Lb[i, t] = L[i, i-t]) of half bandwidth hb: entry (i, i-d) is
    sum_t L[i, i-t] L[i-d, i-t], t = d .. hb"""
    n, w = Lb.shape
    hb = w - 1
    A = np.zeros((n, w))
    for d in range(min(w, n)):
        A[d:, hb - d] = np.einsum("ij,ij->i", Lb[d:, d:], Lb[:n - d, :w - d])
    return A


def factor_band(n, hb, rng, grade):
    """A = L L^T with L = (I + N) diag(l): N a random strictly lower band of half bandwidth hb whose rows sum to at most 1/2 in
    magnitude (so I + N and its inverse stay within a factor 3), and l = 10^U(-grade, 0) with one entry 1 and one 10^-grade.  So
    kappa(A) is within a factor 9 of 10^(2 grade) once n >= 2: not a diagonal scaling away from a dominant band, and not dominant."""
    l = 10.0 ** rng.uniform(-grade, 0.0, n)
    if n >= 2:
        a, b = rng.choice(n, 2, replace=False)
        l[a], l[b] = 1.0, 10.0 ** -grade
    Lb = np.zeros((n, hb + 1))                      # Lb[i, t] = L[i, i-t]
    Lb[:, 0] = l
    if hb:
        N = rng.uniform(-1.0, 1.0, (n, hb)) * (0.5 / hb)
        for t in range(1, min(hb, n - 1) + 1):
            Lb[t:, t] = N[t:, t - 1] * l[:n - t]
    return _nan_outside(_gram(Lb))


def gauge_band(n, hb, rng, delta):
    """J^T J + delta I, J the incidence of a weighted graph on n nodes with an edge (i, i-d) for every d <= hb (d = 1 and d = hb
    always, the others with probability 1/2; weights U(0.1, 1)): a Laplacian whose null space is the constant vector, as the batch
    normal equations without a gauge prior are singular along a rigid motion.  Its eigenvalues are delta and delta plus those of
    the Laplacian, so kappa = (lambda_max + delta) / delta, between ||J^T J||_inf / (2 delta) and ||J^T J||_inf / delta + 1."""
    A = np.zeros((n, hb + 1))
    deg = np.zeros(n)
    for d in range(1, min(hb, n - 1) + 1):
        w = rng.uniform(0.1, 1.0, n - d)
        if 1 < d < hb:
            w *= rng.uniform(size=n - d) < 0.5
        A[d:, hb - d] = -w
        deg[d:] += w
        deg[:n - d] += w
    A[:, hb] = deg + delta
    return _nan_outside(A)


SCHUR_WHERE = ("level1", "level2", "last")


def schur_pair(where):
    """the blocks (p, p+1) that schur_indefinite_band couples, and the block and level at which block cyclic reduction meets the
    non-positive pivot.  Level 0 factors the original odd diagonal blocks, which are positive definite here, so a failure can only
    surface when the coupling's even block is eliminated: at level tz(p) for p even, or in the last block left for p = 0.  The
    natural (K4) order fails in block p+1, which for "level1" and "last" is a block that BCR eliminates at level 0."""
    return {"level1": (2, 1), "level2": (4, 2), "last": (0, None)}[where]


def schur_indefinite_band(n, hb, rng, where):
    """a band whose every b x b diagonal block is positive definite but which is indefinite: factor_band(.., grade=0) (kappa <= 9)
    plus one coupling between the last row of block p and the first row of block p+1 three times the geometric mean of their
    diagonals, so that 2 x 2 principal submatrix, and A, have a clearly negative eigenvalue.  p = schur_pair(where)[0]; every
    principal submatrix without both rows is factor_band's, so positive definite.  Needs hb >= 1 and n > (p + 1) b."""
    b = block_size(hb)
    p = schur_pair(where)[0]
    assert hb >= 1 and n > (p + 1) * b, (n, hb, where)
    A = factor_band(n, hb, rng, 0)
    i, j = (p + 1) * b, (p + 1) * b - 1
    A[i, j - i + hb] = 3.0 * np.sqrt(A[i, hb] * A[j, hb])
    return A
