"""Edge cases of the device front end against the CPU oracle, bit for bit: the feature extraction of features.cu (curvature
ties, points inside 0.5 m, every sector-sort size class, the sector and ring caps, the per-ring voxel filter's pass-through
and voxel faces, strided and device-resident input, and the ring spacing the concurrent rings need), the local map's voxel
filter of grid.cu (one voxel population per branch of k_vox_sort, each form of the exclusive scan, PCL's pass-through and the
2^28-voxel refusal), and the K0 grid + kNN on a map spread over kilometres and at large world offsets.  Every case also checks
that what it targets really happens in its input.  The fixtures and the Python transliteration of the selection live in
tests/test_frontend_edges.py, which checks them on the CPU."""
import numpy as np
import pytest

from tests.test_frontend_edges import (F32, SCAN_BOXES, layout, line, near_fill, near_sweep, ring_points, scan_box_points,
                                       select_features, textured, tie_sweep)

pytestmark = pytest.mark.gpu

IDENT_T = np.zeros(3)
IDENT_Q = np.array([1.0, 0, 0, 0])
FEATURE_KEYS = ("curvature", "label", "sharp", "less_sharp", "flat", "less_flat", "less_flat_ds")


@pytest.fixture(scope="module")
def ctx():
    from glio_b200 import api
    c = api.Context(0, keep_debug=1)
    yield c
    c.close()


def features_case(ctx, oracle, cloud, ss, se, buf=None, intensity_offset=None, **kw):
    """the device's extract_features (on buf, default the packed cloud) == the oracle's stable order, every output"""
    o = oracle.extract_features(cloud, ss, se, stable=True, **kw)
    d = ctx.extract_features(cloud if buf is None else buf, ss, se, intensity_offset=intensity_offset, **kw)
    for k in FEATURE_KEYS:
        assert d[k].shape == o[k].shape and np.array_equal(d[k], o[k]), k
    return d, o


def ring_counts(idx, ss, se):
    return np.array([((idx >= a) & (idx < b)).sum() for a, b in zip(ss, se)])


# ---- A. feature extraction ---------------------------------------------------------------------------------------------------
def test_curvature_ties(ctx, oracle):
    cloud, ss, se = tie_sweep()
    d, _ = features_case(ctx, oracle, cloud, ss, se)
    a = select_features(cloud, ss, se)
    b = select_features(cloud, ss, se, ties="reverse")
    for k in ("sharp", "less_sharp", "flat"):                # the tie order decides the picks
        assert not np.array_equal(np.sort(a[k]), np.sort(b[k])), k
    assert np.array_equal(d["sharp"], a["sharp"]) and np.array_equal(d["flat"], a["flat"])


def test_points_inside_half_a_metre(ctx, oracle):
    cloud, ss, se = near_sweep()
    d, _ = features_case(ctx, oracle, cloud, ss, se)
    near = select_features(cloud, ss, se)["near"]
    assert (select_features(cloud, ss, se, near_filter=False)["label"][near] == -1).any()    # would have been flat
    assert (d["label"][near] == 2).any() and not (d["label"][near] == -1).any()
    x = cloud[:, :3]
    r2 = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2]
    assert np.isin(np.nonzero(r2 == F32(0.25))[0], d["less_flat"]).any()


SECTOR_LENGTHS = [1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 1024, 1365]


def test_sector_sizes_of_every_sort_width(ctx, oracle):
    """end - start = 6 L: every sector holds L points, so the sector sort runs at each power-of-two width up to 2048"""
    rng = np.random.default_rng(21)
    cloud, ss, se = layout([textured(6 * L + 11, rng, r, 6.0 + r) for r, L in enumerate(SECTOR_LENGTHS)])
    assert list((se - ss) // 6) == SECTOR_LENGTHS
    d, _ = features_case(ctx, oracle, cloud, ss, se)
    assert (ring_counts(d["sharp"], ss, se)[1:] > 0).all()


def test_short_and_uneven_rings_and_ds_rate(ctx, oracle):
    rng = np.random.default_rng(22)
    spans = [5, 6, 7, 11, 13, 60, 6, 7, 11, 13]               # end - start: 5 is skipped, the others split unevenly
    cloud, ss, se = layout([textured(s + 11, rng, r, 6.0 + r) for r, s in enumerate(spans)])
    assert list(se - ss) == spans
    d, _ = features_case(ctx, oracle, cloud, ss, se)
    assert ring_counts(d["less_flat"], ss, se)[0] == 0 and (d["label"][ss[0]:se[0]] == 0).all()
    d3, _ = features_case(ctx, oracle, cloud, ss, se, ds_rate=3)
    skipped = np.concatenate([np.arange(ss[r], se[r]) for r in range(len(ss)) if r % 3 != 0])
    assert (d3["label"][skipped] == 0).all() and not np.isin(d3["less_flat"], skipped).any()


def less_flat_ring(F, R, rng, ring, spread=None):
    """a ring of R + 11 points inside 0.5 m except the first F points of its range: F far points on a 1/16 m raster (or
    uniform in the box `spread`); with edge_thres out of reach none of them is an edge, so exactly F are less flat"""
    xyz = near_fill(R + 11, rng)
    k = np.arange(F)
    if spread is None:
        far = np.stack([10 + (k % 64) / 16 + rng.random(F) * 0.01, 5 + (k // 64) / 16, rng.random(F) * 0.01], 1)
    else:
        far = rng.uniform(spread[0], spread[1], (F, 3))
    xyz[5:5 + F] = far
    return ring_points(xyz, ring)


NO_EDGES = dict(edge_thres=1e9)


def test_sector_cap(ctx, oracle):
    from glio_b200 import api
    rng = np.random.default_rng(23)
    cloud, ss, se = layout([less_flat_ring(6000, 6 * 4096, rng, 0)])
    d, _ = features_case(ctx, oracle, cloud, ss, se)
    assert len(d["less_flat"]) > 4096 and len(d["sharp"]) == 12
    cloud, ss, se = layout([less_flat_ring(6000, 6 * 4096 + 1, rng, 0)])       # the last sector holds 4097 points
    with pytest.raises(api.GlioError, match="more than 4096"):
        ctx.extract_features(cloud, ss, se)
    features_case(ctx, oracle, *tie_sweep())


def test_ring_cap(ctx, oracle):
    from glio_b200 import api
    rng = np.random.default_rng(24)
    cloud, ss, se = layout([less_flat_ring(8192, 6 * 2048, rng, 0), less_flat_ring(300, 600, rng, 1)])
    d, _ = features_case(ctx, oracle, cloud, ss, se, **NO_EDGES)
    assert list(ring_counts(d["less_flat"], ss, se)) == [8192, 300]
    cloud, ss, se = layout([less_flat_ring(300, 600, rng, 0), less_flat_ring(8193, 6 * 2048, rng, 1)])
    with pytest.raises(api.GlioError, match="more than 8192"):
        ctx.extract_features(cloud, ss, se, **NO_EDGES)
    features_case(ctx, oracle, *tie_sweep())


def test_ring_voxel_filter_sizes(ctx, oracle):
    """less-flat counts around the voxel sort's widths; the raster puts ~40 points in a voxel"""
    rng = np.random.default_rng(25)
    Fs = [256, 257, 4096, 4097, 8192]
    cloud, ss, se = layout([less_flat_ring(F, 6 * ((F + 300) // 6), rng, r) for r, F in enumerate(Fs)])
    d, o = features_case(ctx, oracle, cloud, ss, se, **NO_EDGES)
    assert list(ring_counts(d["less_flat"], ss, se)) == Fs
    assert (o["ring_ds_count"] > 0).all() and (o["ring_ds_count"] * 8 < np.array(Fs)).all()


def test_ring_voxel_filter_pass_through(ctx, oracle):
    """ds_v 0.01 over a 100 m box: dx*dy*dz > INT32_MAX, PCL passes the ring's less-flat points through unchanged; the
    compact ring next to it is still filtered"""
    rng = np.random.default_rng(26)
    cloud, ss, se = layout([less_flat_ring(3000, 3600, rng, 0, spread=(-50.0, 50.0)), less_flat_ring(3000, 3600, rng, 1, spread=(3.0, 3.1))])
    d, o = features_case(ctx, oracle, cloud, ss, se, ds_v=0.01, **NO_EDGES)
    lf0 = d["less_flat"][d["less_flat"] < se[0]]
    assert o["ring_ds_count"][0] == len(lf0) == 3000 and 0 < o["ring_ds_count"][1] < 3000
    assert np.array_equal(d["less_flat_ds"][:3000], cloud[lf0])


def test_ring_voxel_filter_points_on_voxel_faces(ctx, oracle):
    """coordinates k * 0.4f (both signs) and the floats either side of them"""
    rng = np.random.default_rng(27)
    faces = np.arange(-6, 7, dtype=F32) * F32(0.4)
    vals = np.concatenate([faces, np.nextafter(faces, F32(-np.inf)), np.nextafter(faces, F32(np.inf))])
    F = 4000
    xyz = near_fill(6 * 800 + 11, rng)
    xyz[5:5 + F] = rng.choice(vals, (F, 3))
    cloud, ss, se = layout([ring_points(xyz, 0)])
    d, o = features_case(ctx, oracle, cloud, ss, se, **NO_EDGES)
    x = cloud[d["less_flat"], :3]
    assert np.isin(x, faces).all(axis=1).sum() > 50 and o["ring_ds_count"][0] < len(x)


def test_strided_and_device_resident_input(ctx, oracle):
    import torch
    cloud, ss, se = tie_sweep()
    buf = np.full((len(cloud), 6), np.nan, F32)
    buf[:, :3] = cloud[:, :3]
    buf[:, 5] = cloud[:, 3]
    d6, _ = features_case(ctx, oracle, cloud, ss, se, buf=buf, intensity_offset=5)
    h, _ = features_case(ctx, oracle, cloud, ss, se)
    dev = torch.from_numpy(cloud).cuda()
    g = ctx.extract_features(dev, ss, se)
    torch.cuda.synchronize()
    for k in FEATURE_KEYS:
        assert np.array_equal(g[k], h[k]) and np.array_equal(d6[k], h[k]), k


def spaced_rings(gap, n=400, end0=200):
    """two rings on one straight line at 1/16 m spacing (each step 0.0039 m^2, inside the 0.05 m^2 suppression radius), with
    1/8 m spikes (curvature 1.5625, sharp) at the last point of ring 0's range and the first of ring 1's: ring 0's suppression
    chain reaches the 5 points past its end"""
    p = line(n, 10.0, 5.0)
    st1 = end0 + gap
    p[[end0 - 1, st1], 2] = 0.125
    cloud = np.concatenate([ring_points(p[:end0 + 3], 0), ring_points(p[end0 + 3:], 1)])
    return cloud, np.array([5, st1], np.int32), np.array([end0, n - 6], np.int32)


@pytest.mark.parametrize("gap", [5, 11])
def test_ring_spacing_accepted(ctx, oracle, gap):
    cloud, ss, se = spaced_rings(gap)
    d, _ = features_case(ctx, oracle, cloud, ss, se)
    assert d["label"][se[0] - 1] == 2 and d["label"][ss[1]] == 2


@pytest.mark.parametrize("gap", [4, 1, 0, -30])
def test_ring_spacing_refused(ctx, oracle, gap):
    """rings closer than 5 points (or overlapping) would race on the device; the reference processes them in sequence"""
    from glio_b200 import api
    cloud, ss, se = spaced_rings(gap)
    if gap == 4:                                             # in sequence, ring 0's suppression reaches ring 1's spike
        assert oracle.extract_features(cloud, ss, se)["label"][ss[1]] != 2
    with pytest.raises(api.GlioError, match=r"rings 0 \[5, 200\] and 1 \[%d, 394\]" % ss[1]):
        ctx.extract_features(cloud, ss, se)
    with pytest.raises(api.GlioError, match=r"rings 1 \[5, 200\] and 0 "):   # listed in the other order: same refusal
        ctx.extract_features(cloud, ss[::-1].copy(), se[::-1].copy())
    features_case(ctx, oracle, *tie_sweep())


def test_ring_spacing_counts_only_processed_rings(ctx, oracle):
    """a ring skipped by ds_rate or too short to process may overlap the others"""
    cloud, ss, se = spaced_rings(11)
    ss3 = np.array([ss[0], ss[0] + 50, ss[1]], np.int32)
    se3 = np.array([se[0], se[0] + 20, se[1]], np.int32)
    features_case(ctx, oracle, cloud, ss3, se3, ds_rate=2)
    se3[1] = ss3[1] + 5
    features_case(ctx, oracle, cloud, ss3, se3)


# ---- B. local-map voxel filter ---------------------------------------------------------------------------------------------
POPULATIONS = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000, 5000]
SORT_CLASSES = [(2, 32), (33, 64), (65, 128), (129, 256), (257, 1 << 30)]    # k_vox_sort's warp widths and the rank fallback


def voxel_population_cloud(seed=31, leaf=0.4):
    """one voxel per population, about 1000 m out (a float sum of its points depends on their order), points interleaved"""
    rng = np.random.default_rng(seed)
    pts, vox = [], []
    for v, n in enumerate(POPULATIONS):
        c = (np.array([2500 + 3 * v, -1250 + v, 40]) + 0.5) * leaf
        pts.append(c + rng.uniform(-0.35 * leaf, 0.35 * leaf, (n, 3)))
        vox.append(np.full(n, v))
    perm = rng.permutation(sum(POPULATIONS))
    return np.concatenate(pts).astype(F32)[perm], np.concatenate(vox)[perm]


def seq_sum(x):
    return np.cumsum(x, axis=0, dtype=F32)[-1]


def test_voxel_populations_of_every_sort_branch(ctx, oracle):
    x, v = voxel_population_cloud()
    for lo, hi in SORT_CLASSES:                              # the within-voxel order changes the float sum in every class
        assert any(not np.array_equal(seq_sum(x[v == k]), seq_sum(x[v == k][::-1]))
                   for k, n in enumerate(POPULATIONS) if lo <= n <= hi), (lo, hi)
    world = [oracle.transform_points(part, IDENT_T, IDENT_Q) for part in np.array_split(x, 3)]
    ref, vid = oracle.voxel_filter(np.concatenate(world), 0.4, stable=True)
    assert len(ref) == len(POPULATIONS)
    got = []
    ctx.localmap_clear()
    for part in np.array_split(x, 3):
        ctx.localmap_push(part, IDENT_T, IDENT_Q)
    for _ in range(2):
        assert ctx.localmap_build(0.4) == len(ref)
        got.append(ctx.get_map())
        assert np.array_equal(got[-1], ref)
    rev = np.stack([seq_sum(x[v == k][::-1]) / F32(n) for k, n in enumerate(POPULATIONS)])
    assert not np.array_equal(rev, got[0])                  # a reversed order would have been caught
    ctx.localmap_clear()


def scan_launches(ctx):
    p = ctx.lib_profile_read()
    return p.get("k_scan_block", (0, 0))[1], p.get("k_scan_add", (0, 0))[1]


# launches of the voxel filter's two exclusive scans of nvox + 1 items: one block / two launches / recursive
SCAN_FORMS = {(4095, 1): (2, 0), (4096, 1): (2, 2), (4095, 4097): (2, 2), (4096, 4096): (4, 4)}


@pytest.mark.parametrize("nx,ny", SCAN_BOXES)
def test_voxel_filter_scan_forms(ctx, oracle, nx, ny):
    x = scan_box_points(nx, ny)
    ref, vid = oracle.voxel_filter(x, 1.0, stable=True)
    ctx.localmap_clear()
    ctx.localmap_push(x, IDENT_T, IDENT_Q)
    ctx.lib_profile(True)
    try:
        n = ctx.localmap_build(1.0)
        built = scan_launches(ctx)
        got = ctx.get_map()
        ctx.lib_profile(True)                                # a fresh record: the K0 grid build that localmap_build ends with
        ctx.set_map(got)
        grid = scan_launches(ctx)
    finally:
        ctx.lib_profile(False)
    assert (built[0] - grid[0], built[1] - grid[1]) == SCAN_FORMS[(nx, ny)]
    assert n == len(ref) and np.array_equal(got, ref)
    ctx.localmap_clear()


def test_voxel_filter_pass_through(ctx, oracle):
    rng = np.random.default_rng(33)
    x = rng.uniform(-60, 60, (5000, 3)).astype(F32)
    assert oracle.voxel_filter(x, 0.01) is None               # 12000^3 voxels > INT32_MAX: PCL passes the input through
    ctx.localmap_clear()
    ctx.localmap_push(x[:2000], IDENT_T, IDENT_Q)
    ctx.localmap_push(x[2000:], IDENT_T, IDENT_Q)
    assert ctx.localmap_build(0.01) == len(x)
    assert np.array_equal(ctx.get_map(), x)
    ctx.localmap_clear()


def test_voxel_filter_refuses_more_than_2_28_voxels(ctx, oracle):
    from glio_b200 import api
    rng = np.random.default_rng(34)
    x = rng.uniform(-20, 20, (20000, 3)).astype(F32)
    far = np.array([[3900.5, 3900.5, 0.5]], F32)             # 3921 x 3921 x 41 voxels at leaf 1: > 2^28, < 2^31
    ctx.localmap_clear()
    ctx.localmap_push(far, IDENT_T, IDENT_Q)
    ctx.localmap_push(x, IDENT_T, IDENT_Q)
    with pytest.raises(api.GlioError, match=r"2\^28 voxels"):
        ctx.localmap_build(1.0)
    ctx.localmap_pop_front()
    ref, _ = oracle.voxel_filter(x, 0.4, stable=True)
    assert ctx.localmap_build(0.4) == len(ref) and np.array_equal(ctx.get_map(), ref)
    ctx.localmap_clear()


# ---- C. grid build and kNN -------------------------------------------------------------------------------------------------
def run_case(ctx, oracle, map_xyz, scan_xyz, t=IDENT_T, q=IDENT_Q, slot=0):
    map_xyz = np.ascontiguousarray(map_xyz, np.float32); scan_xyz = np.ascontiguousarray(scan_xyz, np.float32)
    ctx.set_map(map_xyz)
    n = ctx.assoc_scan_to_map(slot, scan_xyz, t, q)
    o = oracle.assoc_scan_to_map(map_xyz, scan_xyz, t, q)
    Q = len(scan_xyz)
    d = ctx.get_assoc_debug(slot, Q)
    assert np.array_equal(d["pm"], o["pm"])
    assert np.array_equal(d["status"], o["status"]), f"status differs at {np.nonzero(d['status'] != o['status'])[0][:10]}"
    ok = o["status"] != oracle.GO_FAIL_RADIUS
    assert np.array_equal(d["idx5"][ok], o["idx5"][ok]), "kNN indices differ"
    assert np.array_equal(d["sqd5"][ok], o["sqd5"][ok]), "kNN distances differ"
    assert np.array_equal(d["plane"][ok], o["plane"][ok])
    assert n == o["nvalid"]
    m = ctx.get_matches(slot, Q)
    v = o["status"] == oracle.GO_VALID
    assert np.array_equal(m["src"], np.nonzero(v)[0].astype(np.int32))
    assert np.array_equal(m["nsd"], o["nsd"][v]) and np.array_equal(m["weight"], o["weight"][v])
    return o


def wall(rng, n, noise=0.01):
    """points on the plane x = 5 (a wall), 6 m x 3 m"""
    p = np.empty((n, 3), np.float32)
    p[:, 0] = 5.0 + rng.normal(0, noise, n); p[:, 1] = rng.uniform(-3, 3, n); p[:, 2] = rng.uniform(0, 3, n)
    return p


def test_spread_map_takes_the_recursive_scan(ctx, oracle):
    """a wall plus a few points kilometres away: the cell size grows until the grid fits 48 M cells, whose scan is recursive"""
    rng = np.random.default_rng(41)
    outliers = np.array([[3000, 0, 0], [0, -2500, 0], [0, 0, 2800], [-1500, 1800, -900], [2200, 2400, 1000]], np.float32)
    m = np.concatenate([wall(rng, 20000), outliers])
    ctx.lib_profile(True)
    try:
        ctx.set_map(m)
        launches = scan_launches(ctx)
    finally:
        ctx.lib_profile(False)
    assert launches == (2, 2)
    o = run_case(ctx, oracle, m, np.concatenate([wall(rng, 2000, noise=0.03), outliers + np.float32(0.5)]))
    assert (o["status"] == oracle.GO_VALID).sum() > 1000


@pytest.mark.parametrize("off", [(3000.0, -1250.5, 40.0), (20000.0, -15000.0, 300.0)])
def test_large_world_offsets(ctx, oracle, off):
    rng = np.random.default_rng(42)
    off = np.array(off, np.float32)
    o = run_case(ctx, oracle, wall(rng, 15000) + off, wall(rng, 2000, noise=0.04) + off)
    assert (o["status"] == oracle.GO_VALID).sum() > 500
