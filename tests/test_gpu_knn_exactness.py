"""The device kNN searches against brute force where their face tests are tightest: sparse maps (5th distances comparable to
the cell, faces open often) at world offsets from 20 km to 2^18 m on each axis and both signs, with map points on the
faces and queries stepped one float at a time across whole cells; grids tens of kilometres wide, where a point that
cell_coord counts beyond a face lies nearer than the float face (tests/test_knn_margins.py), with a query built around
each such face; and a tie exactly at a face.  idx5 / sqd5 are compared with oracle.knn5_brute, the rest of the
association with oracle.assoc_scan_to_map / assoc_pair, the loop-closure 1-NN with pyoracle_loop.nn, all bit for bit.
Every fixture first shows, with the CPU grid mirror, that it puts brute-force neighbours where the face test decides."""
import numpy as np
import pytest

from tests.test_knn_margins import AXES, F32, OLD_SLACK, _flt, _ord, cell_coord, face, face_gaps, first_float_in_cell, grid_layout

pytestmark = pytest.mark.gpu

IDENT_T = np.zeros(3)
IDENT_Q = np.array([1.0, 0, 0, 0])
GATE_SQ = 1.5                                    # default_params().kd_max_radius
OFFSETS = [20000.0, 2.0 ** 15 - 8, 40000.0, 2.0 ** 16 + 8, 70000.0, 140000.0, 2.0 ** 18]
BOX = 12.0                                       # the sparse maps: 3000 points, cell 1.52 m, 5th distance ~0.9 m
WIDE_CELL = 0.6                                  # the wide surf grid: 66 669 x 5 x 5 cells over 40 km


@pytest.fixture(scope="module")
def ctx():
    from glio_b200 import api
    c = api.Context(0, keep_debug=1, t_lb=[0.0, 0.0, 0.0])
    yield c
    c.close()


@pytest.fixture(scope="module")
def wide_ctx():
    from glio_b200 import api
    c = api.Context(0, keep_debug=1, t_lb=[0.0, 0.0, 0.0], cell_size=WIDE_CELL)
    yield c
    c.close()


# ---- fixtures ------------------------------------------------------------------------------------------------------------
def offset_fixture(off, axis, sign, n_map=3000, n_rand=50000, n_line=50000, seed=0, size=BOX):
    """a sparse map (a `size` m box) moved by sign * off along `axis`; a third of it on float faces of the mirrored grid (the face
    itself or up to two floats either side); random queries plus lines stepped one float at a time along the moved axis,
    each across more than a cell (at most 2000 steps)"""
    rng = np.random.default_rng(seed + int(off) % 1000 + 7 * (sign + 1) + len(axis))
    shift = np.asarray(AXES[axis], np.float64) * sign * off
    lo = shift.astype(F32); hi = (shift + size).astype(F32)
    o, cell, inv, nn = grid_layout(lo, hi, n_map)
    m = rng.uniform(lo, hi, (n_map, 3)).astype(F32)
    m[0] = lo; m[1] = hi                                          # the bounding box the layout assumed
    ax = int(np.argmax(np.asarray(AXES[axis])))
    on = np.arange(2, n_map // 3)
    k = rng.integers(1, nn[ax] - 1, len(on))
    m[on, ax] = np.clip(_flt(_ord(face(o[ax], cell, k)) + rng.integers(-2, 3, len(on))), lo[ax], hi[ax])
    q = rng.uniform(lo, hi, (n_rand, 3)).astype(F32)
    steps = min(2000, int(1.2 * float(cell) / float(np.spacing(F32(abs(off) + size)))) + 1)
    starts = rng.uniform(lo, hi, (n_line // steps + 1, 3)).astype(F32)
    line = np.repeat(starts, steps, axis=0)
    line[:, ax] = _flt(_ord(line[:, ax]) + np.tile(np.arange(steps), len(starts)))
    return m, np.concatenate([q, line]), (o, cell, inv, nn)


def wide_fixture(kind, x0, extent, depth, cell_hint, b_frac, n_faces, gap_min, seed=3):
    """a thin map along x, from x0 to x0 + extent.  At n_faces faces where the first float of the next cell lies more than
    gap_min below the face: a query in the cell two below (face distance b = b_frac * cell), a point at that first float
    (nearer than the face), and in-box points (k = 5 for surf, 1 for the 1-NN) at a distance between the two, so that the
    old margin closes the face on them; plus lines of queries stepped one float at a time over four cells either side."""
    rng = np.random.default_rng(seed)
    lo = np.array([x0, 0, 0], F32); hi = np.array([x0 + extent, depth, depth], F32)
    o, cell, inv, nn = grid_layout(lo, hi, 1000, cell_hint=cell_hint)
    up, _ = face_gaps(o[0], cell, inv, nn[0])
    cand = np.nonzero(up > gap_min)[0] + 1
    cand = cand[(cand > 4) & (cand < nn[0] - 4)]
    picked = []
    for k in rng.permutation(cand):
        if all(abs(k - j) > 8 for j in picked):
            picked.append(int(k))
        if len(picked) == n_faces:
            break
    pts = [lo, hi]
    qs, lines = [], []
    y0 = z0 = F32(depth / 2)
    for k in picked:
        F = face(o[0], cell, k)
        X = first_float_in_cell(o[0], cell, inv, np.array([k]))[0]
        qx = F32(F - F32(b_frac * float(cell)))
        assert cell_coord(qx, o[0], inv) == k - 2
        b = F32(F - qx)
        bs = F32(F32(b * F32(0.999)) - F32(OLD_SLACK))
        dp = float(X - qx)
        r = 0.5 * (dp + float(bs))                               # nearer than the old bs, farther than the point past the face
        assert dp < r < float(bs)
        pts.append(np.array([X, y0, z0], F32))
        nin = 5 if kind == "surf" else 1
        for i in range(nin):
            xi = F32(qx - F32(0.9 * r))
            a = float(qx - xi)
            rho = np.sqrt(r * r - a * a)
            th = 2 * np.pi * i / 5
            pts.append(np.array([xi, y0 + rho * np.cos(th), z0 + rho * np.sin(th)], F32))
        qs.append(np.array([qx, y0, z0], F32))
        span = 4 * int(float(cell) / float(np.spacing(qx))) + 1     # four cells either side of the query, one float a step
        xs = _flt(_ord(qx) + np.arange(-span, span))
        lines.append(np.stack([xs, np.full_like(xs, y0), np.full_like(xs, z0)], 1))
    perm = rng.permutation(len(pts) - 2) + 2
    m = np.stack(pts)[np.concatenate([[0, 1], perm])]
    return m, np.stack(qs), np.concatenate(lines), (o, cell, inv, nn)


# ---- the failure band ------------------------------------------------------------------------------------------------------
def band(m, q, idx, layout, kind):
    """the queries whose brute-force top-5 (or 1-NN) holds a point where the face test is tight.  kind "rounding": a point
    in another cell than the query, within the rounding of the float face it lies just past (|face - exact face| > 2 mm,
    the bound the old fixed margin did not cover).  kind "old-margin": a point past a face of the query's 3x3x3 start box
    that is nearer to the query than the old margin's bs: the old face test closes that face before it is scanned."""
    o, cell, inv, nn = layout
    hit = np.zeros(len(q), bool)
    idx = idx.reshape(len(q), -1)
    valid = idx >= 0
    for ax in range(3):
        c = np.clip(cell_coord(q[:, ax], o[ax], inv), 0, nn[ax] - 1)[:, None]
        pa = m[np.where(valid, idx, 0), ax]
        pc = cell_coord(pa, o[ax], inv)
        for up in (True, False):
            if kind == "rounding":
                k = pc if up else pc + 1                         # the face on the query's side of the point's cell
                F = face(o[ax], cell, k).astype(np.float64)
                err = np.abs(F - (float(o[ax]) + k * float(cell)))
                across = (pc > c) if up else (pc < c)
                hit |= (valid & across & (np.abs(pa - F) <= err) & (err > OLD_SLACK)).any(1)
            else:
                k = c + 2 if up else c - 1
                F = face(o[ax], cell, k)
                beyond = valid & ((pc >= k) & (k < nn[ax]) if up else (pc < k) & (k > 0))
                b = (F - q[:, ax][:, None]) if up else (q[:, ax][:, None] - F)
                bs = (b * F32(0.999) - F32(OLD_SLACK)).astype(F32)
                hit |= (beyond & (np.abs(pa - q[:, ax][:, None]) < bs)).any(1)
    return int(hit.sum())


# ---- comparisons ----------------------------------------------------------------------------------------------------------
def check_knn(oracle, m, q, d):
    """idx5 / sqd5 == brute force for every query whose 5th distance passes the gate (beyond it the search is gate-bounded);
    a query brute force flags as a tie is checked by the (distance, index) rule"""
    bi, bd, tie = oracle.knn5_brute(m, q)
    gated = bd[:, 4] < GATE_SQ
    bad = np.nonzero(gated & ~((d["idx5"] == bi).all(1) & (d["sqd5"] == bd).all(1)))[0]
    assert len(bad) == 0, f"{len(bad)} of {int(gated.sum())} gated queries differ from brute force, first {bad[:8]}"
    for i in np.nonzero(gated & (tie != 0))[0][:200]:
        dd = oracle_dist(m, q[i])
        order = np.lexsort((np.arange(len(m)), dd))[:5]
        assert np.array_equal(d["idx5"][i], order)
    return bi, bd, gated


def oracle_dist(m, q):
    d = m - q
    return ((d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def check_assoc(oracle, m, q, d, n=None):
    o = oracle.assoc_scan_to_map(m, q, IDENT_T, IDENT_Q)
    assert np.array_equal(d["pm"], q)
    assert np.array_equal(d["status"], o["status"]), f"status differs at {np.nonzero(d['status'] != o['status'])[0][:10]}"
    ok = o["status"] != oracle.GO_FAIL_RADIUS
    assert np.array_equal(d["idx5"][ok], o["idx5"][ok]) and np.array_equal(d["sqd5"][ok], o["sqd5"][ok])
    assert np.array_equal(d["plane"][ok], o["plane"][ok])
    if n is not None:
        assert n == o["nvalid"]
    return o


def scan_to_map(ctx, oracle, m, q):
    ctx.set_map(m)
    n = ctx.assoc_scan_to_map(0, q, IDENT_T, IDENT_Q)
    d = ctx.get_assoc_debug(0, len(q))
    check_knn(oracle, m, q, d)
    check_assoc(oracle, m, q, d, n)
    return d


def window3(ctx, oracle, m, q):
    parts = np.array_split(q, 3)
    ctx.set_map(m)
    ctx.window_set_scans(parts)
    poses = np.tile(np.r_[IDENT_T, IDENT_Q], (3, 1))
    nm = ctx.window_associate(poses)
    for s, p in enumerate(parts):
        d = ctx.get_assoc_debug(s, len(p))
        check_knn(oracle, m, p, d)
        check_assoc(oracle, m, p, d, nm[s])


def pairs(ctx, oracle, m, q):
    pose = np.r_[IDENT_T, IDENT_Q]
    ctx.batch_clear()
    ctx.batch_set_frame(0, q, pose)
    ctx.batch_set_frame(1, m, pose)
    nm = ctx.batch_associate_pairs([0], [1])
    ro = oracle.assoc_pair(q, IDENT_T, IDENT_Q, m, IDENT_T, IDENT_Q)
    g = ctx.batch_get_matches(0, 1, len(q))
    v = ro["status"] == oracle.GO_VALID
    assert g["n"] == nm[0] == ro["nvalid"]
    assert np.array_equal(g["src"], np.nonzero(v)[0].astype(np.int32))
    assert np.array_equal(g["weight"], ro["weight"][v]) and np.array_equal(g["normal_cent"], ro["normal_cent"][v])
    ctx.batch_clear()


def loop_nn(ctx, m, q):
    from oracle import pyoracle_loop
    r = ctx.icp_align(q, m, correspondences=True, max_iterations=1, max_correspondence_distance=30.0)
    cq, cm, cd = r["corr"]
    bi, bd = pyoracle_loop.nn(m, q)
    keep = bd <= np.float32(900.0)
    assert np.array_equal(cq, np.nonzero(keep)[0].astype(np.int32))
    bad = np.nonzero((cm != bi[keep]) | (cd != bd[keep]))[0]
    assert len(bad) == 0, f"{len(bad)} of {len(cq)} 1-NN differ from brute force, first {cq[bad[:8]]}"


# ---- 1. world offsets --------------------------------------------------------------------------------------------------------
# queries whose brute-force top-5 holds a point within a face's rounding (> 2 mm) of that face, per fixture, from 2^16 m
ROUNDING_BAND_MIN = 200


@pytest.mark.parametrize("sign", [1, -1])
@pytest.mark.parametrize("axis", list(AXES))
@pytest.mark.parametrize("off", OFFSETS)
def test_scan_to_map_at_world_offsets(ctx, oracle, off, axis, sign):
    m, q, lay = offset_fixture(off, axis, sign)
    assert len(q) >= 100000
    d = scan_to_map(ctx, oracle, m, q)
    bi, _, _ = oracle.knn5_brute(m, q)
    if off >= 2 ** 16:
        assert band(m, q, bi, lay, "rounding") >= ROUNDING_BAND_MIN
    assert (d["sqd5"][:, 4] < GATE_SQ).sum() > 20000          # most queries pass the gate: their top-5 is compared


@pytest.mark.parametrize("sign", [1, -1])
@pytest.mark.parametrize("off", OFFSETS)
def test_other_paths_at_world_offsets(ctx, oracle, off, sign):
    m, q, lay = offset_fixture(off, "xyz", sign, n_rand=10000, n_line=10000, seed=1)
    window3(ctx, oracle, m, q)
    pairs(ctx, oracle, m, q)
    loop_nn(ctx, m, q[::4].copy())
    if off >= 2 ** 16:
        bi, _, _ = oracle.knn5_brute(m, q)
        assert band(m, q, bi, lay, "rounding") >= ROUNDING_BAND_MIN // 10


# ---- 2. wide grids: points nearer than the face they are counted beyond -------------------------------------------------------
def test_wide_grid_scan_to_map(wide_ctx, oracle):
    m, qs, lines, lay = wide_fixture("surf", 0.0, 40000.0, 2.0, WIDE_CELL, 1.33, 120, 3e-3)
    q = np.concatenate([qs, lines])
    assert len(q) >= 100000
    bi, _, _ = oracle.knn5_brute(m, q)
    assert band(m, qs, bi[:len(qs)], lay, "old-margin") == len(qs) >= 90          # every face with a gap over 3 mm, 8 cells apart
    assert band(m, q, bi, lay, "old-margin") >= 4000
    scan_to_map(wide_ctx, oracle, m, q)


def test_wide_grid_window_and_pairs(wide_ctx, oracle):
    m, qs, lines, lay = wide_fixture("surf", 0.0, 40000.0, 2.0, WIDE_CELL, 1.33, 60, 3e-3, seed=4)
    q = np.concatenate([qs, lines[::3]])
    bi, _, _ = oracle.knn5_brute(m, q)
    assert band(m, q, bi, lay, "old-margin") >= 60
    window3(wide_ctx, oracle, m, q)
    pairs(wide_ctx, oracle, m, q)


def test_wide_grid_loop_closure_nn(ctx):
    from oracle import pyoracle_loop
    m, qs, lines, lay = wide_fixture("loop", -100000.0, 200000.0, 8.0, 0.0, 1.125, 100, 6e-3, seed=5)
    assert lay[1] == F32(4.0)
    q = np.concatenate([qs, lines[::8]])
    bi, _ = pyoracle_loop.nn(m, qs)
    assert band(m, qs, bi, lay, "old-margin") == len(qs) == 100
    loop_nn(ctx, m, q)


# ---- 3. a tie exactly at a face ---------------------------------------------------------------------------------------------
def tie_fixture(scale):
    """dyadic coordinates (every difference, square and sum exact).  Grid origin -0.25 s, cell 0.5 s; the query at x = 4.625 s
    has its start box's upper x face at 5.25 s.  Six in-box points and one point P on that face all lie at squared distance
    0.453125 s^2; P's index (4) is below the 5th in-box one: the top-5 is {0, 1, 2, 3, 4} and P must be found."""
    s = F32(scale)
    rel = np.array([[-0.625, 0.25, 0], [-0.625, -0.25, 0], [-0.625, 0, 0.25], [-0.625, 0, -0.25], [0.625, 0.25, 0],
                    [-0.25, 0.625, 0], [-0.25, -0.625, 0]], F32)
    q = np.array([4.625, 4.0, 4.0], F32) * s
    pts = q + rel * s
    m = np.concatenate([pts, np.array([[0, 0, 0], [8, 8, 8]], F32) * s]).astype(F32)
    return m, q[None, :]


def test_tie_on_a_face_is_found(ctx, oracle):
    from glio_b200 import api
    m, q = tie_fixture(1.0)
    o, cell, inv, nn = grid_layout(m.min(0), m.max(0), len(m), cell_hint=0.5)
    assert float(o[0]) == -0.25 and float(cell) == 0.5
    assert cell_coord(q[0, 0], o[0], inv) == 9 and float(face(o[0], cell, 11)) == 5.25 == m[4, 0]
    d2 = oracle_dist(m, q[0])
    assert (d2[:7] == F32(0.453125)).all() and cell_coord(m[4, 0], o[0], inv) == 11
    c = api.Context(0, keep_debug=1, cell_size=0.5)
    try:
        c.set_map(m)
        c.assoc_scan_to_map(0, q, IDENT_T, IDENT_Q)
        d = c.get_assoc_debug(0, 1)
    finally:
        c.close()
    assert list(d["idx5"][0]) == [0, 1, 2, 3, 4] and (d["sqd5"][0] == F32(0.453125)).all()
    bi, bd, tie = oracle.knn5_brute(m, q)
    assert tie[0] and np.array_equal(bi[0], d["idx5"][0])
    # the 1-NN: the same geometry at cell 4 (the loop grid's cell for a cloud this sparse), P the only point at the tie
    m8, q8 = tie_fixture(8.0)
    o, cell, inv, nn = grid_layout(m8.min(0), m8.max(0), 3)
    assert float(cell) == 4.0 and float(face(o[0], cell, 11)) == m8[4, 0]
    tgt = m8[[4, 5, 7, 8]]                                     # P first: it wins the (distance, index) tie with the in-box point
    src = np.concatenate([q8, tgt[2:]])
    r = ctx.icp_align(src, tgt, correspondences=True, max_iterations=1, max_correspondence_distance=30.0)
    cq, cm, cd = r["corr"]
    assert cm[list(cq).index(0)] == 0 and cd[list(cq).index(0)] == F32(0.453125 * 64)
