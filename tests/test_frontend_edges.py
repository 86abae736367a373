"""Edge-case fixtures of the front end's feature extraction (Preprocessing.cpp:529-655) and of the local map's voxel filter,
checked on the CPU: the oracle's stable feature selection against a short Python transliteration of Preprocessing.cpp:549-650
on sweeps with exact curvature ties and points inside 0.5 m, and the oracle's voxel filter against a numpy formulation on the
voxel boxes whose scans take each form of the device's exclusive scan.  tests/test_gpu_frontend_edges.py runs the device on the
same fixtures against the oracle bit for bit, so there "matches the oracle" also means "matches the reference" on these edges."""
import numpy as np
import pytest

F32 = np.float32


# ---- sweep construction ----------------------------------------------------------------------------------------------------
def layout(rings):
    """Concatenate per-ring (m, 4) x,y,z,intensity arrays the way the reference builds laserCloud (Preprocessing.cpp:522-526):
    scan_start = size before the ring + 5, scan_end = size after it - 6."""
    ss, se, size = [], [], 0
    for r in rings:
        ss.append(size + 5)
        size += len(r)
        se.append(size - 6)
    return np.ascontiguousarray(np.concatenate(rings), F32), np.array(ss, np.int32), np.array(se, np.int32)


def ring_points(xyz, ring):
    """x,y,z plus the reference's intensity, ring + 0.1 relTime"""
    m = len(xyz)
    out = np.empty((m, 4), F32)
    out[:, :3] = xyz
    out[:, 3] = F32(ring) + F32(0.1) * (np.arange(m, dtype=F32) / F32(max(m - 1, 1)))
    return out


def line(m, x0, y, z=0.0, step=1 / 16):
    """a straight run with dyadic coordinates: every sum of the curvature is exact, so its interior curvature is exactly 0"""
    k = np.arange(m, dtype=np.float64)
    return np.stack([x0 + k * step, np.full(m, y), np.full(m, z)], 1)


def zigzag(m, x0, y, z=0.0, step=1 / 16, a=1 / 8):
    """a period-2 zig-zag of amplitude a: 10 neighbours - 10 p = -12 (+-a) in z, so every interior curvature is 144 a^2 (2.25)"""
    p = line(m, x0, y, z, step)
    p[:, 2] += np.where(np.arange(m) % 2 == 0, a, -a)
    return p


def near_fill(m, rng, r=0.45):
    """points inside 0.5 m of the sensor (the reference drops them from the flat and less-flat sets)"""
    d = rng.normal(size=(m, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * (r * rng.random((m, 1)) ** (1 / 3))


def textured(m, rng, ring, y0):
    """a ring of dyadic pieces: runs (curvature 0), zig-zags (2.25), steps and 1/256-quantised jitter: many exact ties"""
    k = np.arange(m)
    p = line(m, -m / 32, y0)
    pos = 0
    while pos < m:
        L = int(rng.integers(6, 41))
        s = slice(pos, min(m, pos + L))
        t = int(rng.integers(0, 4))
        if t == 1:
            p[s, 2] += np.where(k[s] % 2 == 0, 0.125, -0.125)
        elif t == 2:
            p[s, 1] += 0.25
        elif t == 3:
            p[s, 1:] += rng.integers(-32, 33, (len(k[s]), 2)) / 256
        pos += L
    return ring_points(p, ring)


def tie_sweep():
    """ring 0: a straight run (curvature exactly 0 throughout: the flat picks are a choice among ties); ring 1: a zig-zag
    (exactly 2.25 throughout, no suppression since a step is 0.066 m^2: the sharp and less-sharp picks are a choice among
    ties); ring 2: runs and zig-zags alternating every 40 points"""
    m = 6 * 120 + 11
    mixed = line(m, -30.0, 7.0)
    k = np.arange(m)
    mixed[:, 2] += np.where((k // 40) % 2 == 1, np.where(k % 2 == 0, 0.125, -0.125), 0.0)
    return layout([ring_points(line(m, 10.0, 5.0), 0), ring_points(zigzag(m, 20.0, -5.0), 1), ring_points(mixed, 2)])


def near_points_on_the_boundary(rng):
    """points with |p|^2 exactly 0.25 in float and their neighbouring floats, each in the middle of a short run"""
    pts = [[0.5, 0, 0], [0, 0.5, 0], [0, 0, -0.5], [-0.5, 0, 0], [0.3, 0.4, 0], [0.4, -0.3, 0], [0, -0.3, 0.4]]
    d = rng.normal(size=(12, 3))
    pts += list(0.5 * d / np.linalg.norm(d, axis=1, keepdims=True))
    out = []
    for p in np.array(pts, F32):
        for q in (p, np.nextafter(p, F32(0)), np.nextafter(p, F32(2) * p)):
            out.append(q)
    return np.array(out, F32)


def near_sweep(seed=5):
    """ring 0: a far run, a near run (2/256 .. 81/256 m: exactly flat, so flat but for the 0.5 m filter), a far run; ring 1:
    a zig-zag entirely inside 0.5 m (every point sharp material); ring 2: points on the |p|^2 = 0.25 boundary"""
    rng = np.random.default_rng(seed)
    r0 = np.concatenate([line(80, 10.0, 5.0), line(80, 2 / 256, 0.0, step=1 / 256), line(91, -40.0, 5.0)])
    r1 = zigzag(6 * 8 + 11, 1 / 64, 0.0, step=1 / 128)
    b = near_points_on_the_boundary(rng)
    runs = [line(11, 0.0, 0.0, step=1 / 512) + q.astype(np.float64) - np.array([5 / 512, 0, 0]) for q in b]
    for run, q in zip(runs, b):
        run[5] = q                                              # the boundary point itself, bit for bit
    r2 = np.concatenate([line(5, 10.0, 5.0)] + runs + [line(6, 12.0, 5.0)])
    return layout([ring_points(r0, 0), ring_points(r1, 1), ring_points(r2, 2)])


# ---- Preprocessing.cpp:549-650 in Python ---------------------------------------------------------------------------------------
def curvature(xyz):
    """float32, the reference's left-to-right sum (:529-534)"""
    x = np.ascontiguousarray(xyz[:, :3], F32)
    n = len(x)
    acc = x[0:n - 10].copy()
    for k in range(1, 5):
        acc = acc + x[k:n - 10 + k]
    acc = acc - F32(10) * x[5:n - 5]
    for k in range(6, 11):
        acc = acc + x[k:n - 10 + k]
    c = np.zeros(n, F32)
    c[5:n - 5] = (acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1]) + acc[:, 2] * acc[:, 2]
    return c


def select_features(cloud, ss, se, ds_rate=1, edge_thres=1.0, surf_thres=0.1, ties="index", near_filter=True):
    """Sort every sector by (curvature, index) (ties="reverse": by (curvature, -index)), pick <= 2 sharp + 8 less-sharp from the
    top and <= 4 flat from the bottom with the +-5 neighbour suppression, then the less-flat points; floats compared in double
    as the reference's promotions do."""
    x = np.ascontiguousarray(cloud[:, :3], F32)
    n = len(x)
    curv = curvature(x)
    c64 = curv.astype(np.float64)
    r2 = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2]
    near = (r2.astype(np.float64) < 0.25) if near_filter else np.zeros(n, bool)
    d = x[1:] - x[:-1]
    close = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float64) <= 0.05   # close[i]: i -> i + 1
    picked = np.zeros(n, bool)
    label = np.zeros(n, np.int8)
    sharp, less_sharp, flat, less_flat = [], [], [], []

    def suppress(ind):
        for l in range(1, 6):
            if not close[ind + l - 1]:
                break
            picked[ind + l] = True
        for l in range(1, 6):
            if not close[ind - l]:
                break
            picked[ind - l] = True

    for r in range(len(ss)):
        if se[r] - ss[r] < 6 or r % ds_rate != 0:
            continue
        for j in range(6):
            sp = ss[r] + (se[r] - ss[r]) * j // 6
            ep = ss[r] + (se[r] - ss[r]) * (j + 1) // 6 - 1
            idx = np.arange(sp, ep + 1)
            order = idx[np.lexsort((idx if ties == "index" else -idx, curv[sp:ep + 1]))]
            largest = 0
            for ind in order[::-1]:
                if not picked[ind] and c64[ind] > edge_thres:
                    largest += 1
                    if largest <= 2:
                        label[ind] = 2; sharp.append(ind); less_sharp.append(ind)
                    elif largest <= 10:
                        label[ind] = 1; less_sharp.append(ind)
                    else:
                        break
                    picked[ind] = True
                    suppress(ind)
            smallest = 0
            for ind in order:
                if near[ind]:
                    continue
                if not picked[ind] and c64[ind] < surf_thres:
                    label[ind] = -1; flat.append(ind)
                    smallest += 1
                    if smallest >= 4:
                        break
                    picked[ind] = True
                    suppress(ind)
            less_flat += [k for k in range(sp, ep + 1) if not near[k] and label[k] <= 0]
    a = lambda v: np.array(v, np.int32)
    return dict(curvature=curv, label=label, sharp=a(sharp), less_sharp=a(less_sharp), flat=a(flat), less_flat=a(less_flat), near=near)


def assert_same_selection(o, p):
    assert np.array_equal(o["curvature"], p["curvature"])
    for k in ("label", "sharp", "less_sharp", "flat", "less_flat"):
        assert np.array_equal(o[k], p[k]), k


def test_oracle_selection_with_ties_matches_the_transliteration(oracle):
    cloud, ss, se = tie_sweep()
    o = oracle.extract_features(cloud, ss, se, stable=True)
    p = select_features(cloud, ss, se)
    assert_same_selection(o, p)
    # not vacuous: the tie order decides which sharp, less-sharp and flat points are taken
    q = select_features(cloud, ss, se, ties="reverse")
    for k in ("sharp", "less_sharp", "flat"):
        assert not np.array_equal(np.sort(p[k]), np.sort(q[k])), k
    in1 = p["sharp"][(p["sharp"] >= ss[1]) & (p["sharp"] < se[1])]
    in0 = p["flat"][(p["flat"] >= ss[0]) & (p["flat"] < se[0])]
    assert len(in1) == 12 and (p["curvature"][in1] == F32(2.25)).all() and len(in0) == 24 and (p["curvature"][in0] == 0).all()


def test_oracle_near_filter_matches_the_transliteration(oracle):
    cloud, ss, se = near_sweep()
    o = oracle.extract_features(cloud, ss, se, stable=True)
    p = select_features(cloud, ss, se)
    assert_same_selection(o, p)
    near = p["near"]
    # the filter decides: near points would be flat without it, and the sharp picks ignore it
    q = select_features(cloud, ss, se, near_filter=False)
    assert (q["label"][near] == -1).any() and not (p["label"][near] == -1).any()
    assert (p["label"][near] == 2).sum() >= 2 and not near[p["less_flat"]].any()
    # |p|^2 == 0.25 in float is kept, the float below it is dropped
    x = cloud[:, :3]
    r2 = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2]
    inside = np.zeros(len(cloud), bool)
    inside[ss[2]:se[2]] = True
    assert (inside & (r2 == F32(0.25))).sum() >= 5 and (inside & near & (r2 > F32(0.2499))).sum() >= 5
    assert np.isin(np.nonzero(inside & (r2 == F32(0.25)))[0], o["less_flat"]).any()


# ---- voxel boxes of the scan regimes ---------------------------------------------------------------------------------------
# leaf 1.0, points within 0.25 of voxel centres; the scan over the voxel table has nvox + 1 entries:
# 4096 (one block), 4097 (two launches), 2^24 (two launches, 4096 blocks), 2^24 + 1 (recursive)
SCAN_BOXES = [(4095, 1), (4096, 1), (4095, 4097), (4096, 4096)]


def scan_box_points(nx, ny, seed=0, nfill=300_000):
    """1-3 points in each of min(nx*ny, nfill) voxels of an nx x ny x 1 box at leaf 1.0, the two corner voxels always filled"""
    rng = np.random.default_rng(seed + nx + ny)
    nv = nx * ny
    vox = np.arange(nv) if nv <= nfill else np.unique(np.concatenate([[0, nv - 1], rng.choice(nv, nfill, replace=False)]))
    reps = rng.integers(1, 4, len(vox))
    v = np.repeat(vox, reps)
    c = np.stack([v % nx + 0.5, v // nx + 0.5, np.full(len(v), 0.5)], 1)
    p = (c + rng.uniform(-0.25, 0.25, c.shape)).astype(F32)
    return p[rng.permutation(len(p))]


def np_voxel(x, leaf):
    inv = F32(1) / F32(leaf)
    mb = np.floor(x.min(0) * inv).astype(np.int64)
    div = np.floor(x.max(0) * inv).astype(np.int64) - mb + 1
    ijk = (np.floor(x * inv) - mb.astype(F32)).astype(np.int64)
    vid = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    u, inv_i, cnt = np.unique(vid, return_inverse=True, return_counts=True)
    mean = np.zeros((len(u), 3))
    np.add.at(mean, inv_i, x.astype(np.float64))
    return u, mean / cnt[:, None], div


@pytest.mark.parametrize("nx,ny", SCAN_BOXES)
def test_oracle_voxel_filter_at_the_scan_boxes(oracle, nx, ny):
    x = scan_box_points(nx, ny)
    u, mean, div = np_voxel(x, 1.0)
    assert list(div) == [nx, ny, 1]
    got, vid = oracle.voxel_filter(x, 1.0, stable=True)
    assert np.array_equal(vid, u)
    assert np.abs(got - mean).max() <= 4e-7 * max(nx, ny)            # <= 3 points per voxel: a few ulp of the coordinate
