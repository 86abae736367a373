"""The face tests of the grid kNN searches, restated in float32 on the CPU.

k_knn_box (box_face_open, the row skip of scan_rows_batched) and the loop-closure 1-NN (nn_face_open) close a face of the
searched box when the 5th (1st) distance is inside  bs = (face - q) * 0.999 - slack,  with the face computed as
ox + (float)k * cell.  The points were put in their cells by cell_coord, floor((x - ox) * inv_cell), rounded in float too.
The search is exact only if no point that cell_coord puts beyond a face lies nearer to the query than bs.

This file mirrors the host grid layout of grid_build and both float expressions, and measures, face by face, the float
"gap": how much nearer than the computed face a point counted beyond it can lie.  Two findings:
  * the computed face can be several mm off the exact face ox + k * cell (above 2^16 m, more than the old fixed 2 mm
    margin), but the points live on the same float lattice as the face: for grids a few tens of metres wide (the 12 m sparse maps of the device tests included) the gap is 0
    at any offset up to 2^20 m, so the old margin was never short there;
  * the gap grows with the grid's extent: where the grid spans tens of kilometres (|x - ox| large, not only |x|), up to
    a few ulp of the largest coordinate; from 2^15 m on that is more than 2 mm.  GridDesc::slack = max(2 mm, 8 ulp(M))
    covers it.  tests/test_gpu_knn_exactness.py shows the miss on the device and checks the fix.
"""
import numpy as np
import pytest

F32 = np.float32
PTS_PER_CELL = 8.0          # capi.cu: Context::pts_per_cell
OLD_SLACK = 2e-3
SLACK_ULPS = 8              # grid.cu face_slack


def grid_layout(mn, mx, n, cell_hint=0.0, pts_per_cell=PTS_PER_CELL):
    """grid_build's layout (grid.cu): (origin[3], cell, inv_cell, n[3]) from the float bounding box and the point count"""
    mn = np.asarray(mn, F32); mx = np.asarray(mx, F32)
    L = (mx - mn + F32(1e-3)).astype(F32)
    cell = F32(cell_hint)
    if not cell > 0:
        area = 2.0 * (float(L[0]) * float(L[1]) + float(L[1]) * float(L[2]) + float(L[0]) * float(L[2]))
        cell = F32(np.sqrt(pts_per_cell * area / n))
        cell = min(max(cell, F32(0.05)), F32(4.0))
    while float(np.ceil(L[0] / cell + F32(1))) * float(np.ceil(L[1] / cell + F32(1))) * float(np.ceil(L[2] / cell + F32(1))) > 48.0e6:
        cell = F32(cell * F32(1.26))
    o = (mn - F32(0.5) * cell).astype(F32)
    nn = (np.floor((mx - o) / cell) + 2).astype(np.int64)
    return o, F32(cell), F32(F32(1.0) / cell), nn


def face(o, cell, k):
    """the device's face position oa + (float)k * cell, rounded as written (-fmad=false)"""
    return F32(o) + np.asarray(k).astype(F32) * F32(cell)


def cell_coord(v, o, inv):
    return np.floor((np.asarray(v, F32) - F32(o)) * F32(inv)).astype(np.int64)


def face_slack(o, cell, nn):
    o = np.asarray(o, F32)
    M = max(max(abs(float(o[d])), abs(float(face(o[d], cell, nn[d])))) for d in range(3))
    return max(F32(OLD_SLACK), F32(SLACK_ULPS) * np.spacing(F32(M)))


def _ord(x):
    i = np.asarray(x, F32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7fffffff), i)


def _flt(o):
    o = np.asarray(o, np.int64)
    return np.where(o < 0, (-o) | 0x80000000, o).astype(np.uint32).view(F32)


def first_float_in_cell(o, cell, inv, k):
    """the smallest float x with cell_coord(x) >= k, for every k (bisection over the ordered float bits)"""
    k = np.asarray(k, np.int64)
    f = face(o, cell, k)
    a = _ord(f - F32(2) * cell - F32(1)); b = _ord(f + F32(2) * cell + F32(1))
    assert (cell_coord(_flt(a), o, inv) < k).all() and (cell_coord(_flt(b), o, inv) >= k).all()
    while (b - a > 1).any():
        m = (a + b) // 2
        up = cell_coord(_flt(m), o, inv) >= k
        a = np.where(up, a, m); b = np.where(up, m, b)
    return _flt(b)


def face_gaps(o, cell, inv, n):
    """per face k = 1..n-1 of one axis: (up, down) gaps in metres.  up: face - (first float of cell k), how much nearer than
    an upper face at k a point of cell >= k can be; down: (last float of cell k-1) - face, the same for a lower face."""
    k = np.arange(1, n)
    f = face(o, cell, k).astype(np.float64)
    x = first_float_in_cell(o, cell, inv, k)
    return f - x.astype(np.float64), np.nextafter(x, F32(-np.inf)).astype(np.float64) - f


def worst_gap(o, cell, inv, nn):
    return max(max(g.max() for g in face_gaps(o[d], cell, inv, nn[d])) for d in range(3))


# ---- 1. the exact-face rounding (the bound a real-number argument would need) -------------------------------------------
TABLE_MM = {3000: 0.10, 20000: 0.79, 40000: 1.57, 70000: 3.13, 140000: 6.25}


def exact_face_error(off, cell=0.7, faces=400):
    o = F32(F32(off) - F32(0.5) * F32(cell))
    k = np.arange(faces)
    return np.abs(face(o, cell, k).astype(np.float64) - (float(o) + k * float(F32(cell)))).max()


@pytest.mark.parametrize("off", sorted(TABLE_MM))
def test_exact_face_rounding_table(off):
    """cell 0.7 m, origin off - 0.35 m, faces 0..399: the computed face is up to half an ulp off the exact one; the fixed
    2 mm would not cover that from 2^16 m up (which is why a bound on it alone cannot prove the search exact)"""
    e = exact_face_error(off)
    assert round(e * 1e3, 2) == TABLE_MM[off]
    assert (e > OLD_SLACK) == (off >= 2 ** 16)
    assert e <= 0.5 * np.spacing(F32(off + 400 * 0.7))


# ---- 2. small grids at large offsets: the float gap ----------------------------------------------------------------------
OFFSETS = [0.0, 3000.0, 20000.0, 2.0 ** 15 - 8, 40000.0, 2.0 ** 16 + 8, 70000.0, 140000.0, 2.0 ** 18, 2.0 ** 20]
AXES = {"x": (1, 0, 0), "y": (0, 1, 0), "z": (0, 0, 1), "xyz": (1, 1, 1)}


def box_layout(off, axis, sign, n=3000, size=12.0):
    """the layout of a sparse map of n points filling a `size` m box whose low corner is moved by sign * off along axis"""
    mn = np.asarray(AXES[axis], np.float64) * sign * off
    return grid_layout(mn.astype(F32), (mn + size).astype(F32), n)


@pytest.mark.parametrize("off", OFFSETS)
def test_small_grids_have_no_gap_at_any_offset(off):
    worst = []
    for axis in AXES:
        for sign in (1, -1):
            o, cell, inv, nn = box_layout(off, axis, sign)
            assert abs(float(cell) - 1.518) < 0.001 and (nn <= 10).all()
            worst.append(worst_gap(o, cell, inv, nn))
            assert worst[-1] <= face_slack(o, cell, nn)
    # the old constant held too: in a grid this narrow faces and cell bounds agree to within a float step of the
    # unshifted axes, whatever the offset
    assert max(worst) < 1e-6


# ---- 3. wide grids: the gap the slack has to cover -----------------------------------------------------------------------
def wide_layout(x0, extent, cell, depth=2.0):
    """a thin grid along x from x0 to x0 + extent, depth metres deep in y and z, cell edge `cell`"""
    mn = np.array([x0, 0.0, 0.0], F32)
    mx = np.array([x0 + extent, depth, depth], F32)
    return grid_layout(mn, mx, 1000, cell_hint=cell)


@pytest.mark.parametrize("x0,extent,cell,gapped", [(0.0, 40000.0, 0.6, True), (-30000.0, 100000.0, 4.0, True), (-100000.0, 200000.0, 4.0, True), (0.0, 80000.0, 4.0, False), (1000.0, 20000.0, 1.0, False)])
def test_wide_grids_need_more_than_2mm(x0, extent, cell, gapped):
    o, c, inv, nn = wide_layout(x0, extent, cell)
    up, dn = face_gaps(o[0], c, inv, nn[0])
    g = max(up.max(), dn.max())
    M = max(abs(float(o[0])), abs(float(face(o[0], c, nn[0]))))
    assert g <= face_slack(o, c, nn)
    assert (g > OLD_SLACK) == gapped, (g, M)
    if gapped:
        assert M >= 2 ** 15


def test_slack_ulps_cover_the_worst_gap():
    """random layouts (offsets to 2^21 m, extents 10 m .. 200 km, both signs, grids across 0): the largest gap seen is 5
    ulp(M); the slack takes 8"""
    rng = np.random.default_rng(5)
    worst = 0.0
    for _ in range(300):
        ext = 10 ** rng.uniform(1, 5.3)
        x0 = -ext / 2 if rng.random() < 0.3 else rng.choice([-1, 1]) * 10 ** rng.uniform(0, 6.3)
        mn = np.array([x0, 0, 0], F32); mx = np.array([x0 + ext, 20, 20], F32)
        o, c, inv, nn = grid_layout(mn, mx, int(10 ** rng.uniform(3, 6)))
        up, dn = face_gaps(o[0], c, inv, nn[0])
        M = max(abs(float(o[0])), abs(float(face(o[0], c, nn[0]))))
        worst = max(worst, max(up.max(), dn.max()) / float(np.spacing(F32(M))))
    assert 2 < worst <= SLACK_ULPS - 2


def test_slack_is_the_old_2mm_below_2_12():
    for M in (0.0, 100.0, 3000.0, 4095.0):
        o, c, inv, nn = grid_layout(np.array([M - 20, -5, -5], F32), np.array([M - 1, 5, 5], F32), 5000)
        assert face_slack(o, c, nn) == F32(OLD_SLACK)
    o, c, inv, nn = grid_layout(np.array([70000, 0, 0], F32), np.array([70020, 5, 5], F32), 5000)
    assert face_slack(o, c, nn) == F32(8 * 2.0 ** -7)
