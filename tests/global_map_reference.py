"""References of the sort-based VoxelGrid (glio_voxel_filter) and of save_pcd's global map (glio_loop_global_map,
GLIO/src/Estimator.cpp:5324-5349), shared by tests/test_global_map.py (CPU) and tests/test_gpu_global_map.py.

- global_map(): the oracle's global map, built on the oracle primitives only: pyoracle.transform_points twice (transformCloud by
  Tbl, then by the keyframe pose) and the stable pyoracle.voxel_filter (ds_filter_global_map).
- np_transform() / np_voxel_filter() / np_global_map(): an independent numpy formulation of the same arithmetic: Eigen's
  quaternion rotation in float64 in Eigen's operation order, rounded to float; PCL's applyFilter with float32 bounds, int32 voxel
  indices wrapped to 32 bits and sorted unsigned with argsort(kind="stable"), sequential float32 sums divided by the float count.
- The box fixtures of the key-width, pass-through and wrap cases.
"""
import numpy as np

F32 = np.float32
INT32_MAX = 2**31 - 1


# ---- numpy formulation -----------------------------------------------------------------------------------------------------
def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def np_transform(xyz, t, q):
    """float(q * double(p) + t): Eigen 3.3 _transformVector (uv = u x v; uv += uv; v + w uv + u x uv) in float64, no FMA"""
    v = np.asarray(xyz, F32).reshape(-1, 3).astype(np.float64)
    q = np.asarray(q, np.float64); t = np.asarray(t, np.float64)
    u = np.broadcast_to(q[1:], v.shape)
    uv = _cross(u, v)
    uv = uv + uv
    c = _cross(u, uv)
    o = (v + q[0] * uv) + c
    return (o + t).astype(F32)


def np_voxel_keys(x, leaf):
    """(keys uint32, filtered): PCL's applyFilter voxel index of every point; filtered False = PCL's pass-through"""
    x = np.asarray(x, F32).reshape(-1, 3)
    inv = F32(1) / F32(leaf)
    mn = x.min(0); mx = x.max(0)
    d = [int(F32(F32(mx[k] - mn[k]) * inv)) + 1 for k in range(3)]
    if d[0] * d[1] * d[2] > INT32_MAX:
        return None, False
    min_b = np.floor(mn * inv).astype(np.int64)
    div = np.floor(mx * inv).astype(np.int64) - min_b + 1
    ijk = (np.floor(x * inv) - min_b.astype(F32)).astype(np.int64)
    mul = [1, int(div[0]), int((div[0] * div[1]) & 0xffffffff)]
    key = (ijk[:, 0] + ijk[:, 1] * mul[1] + ijk[:, 2] * mul[2]) & 0xffffffff
    return key.astype(np.uint32), True


def seq_segment_sums(v, starts, lens):
    """float32 sums of v[starts[s] : starts[s] + lens[s]], each left to right"""
    acc = np.zeros((len(starts), v.shape[1]), F32)
    for k in range(int(lens.max()) if len(lens) else 0):
        a = lens > k
        acc[a] = acc[a] + v[starts[a] + k]
    return acc


def np_voxel_filter(x, leaf):
    """(points, filtered): the stable VoxelGrid of x (pass-through: x itself, filtered False)"""
    x = np.asarray(x, F32).reshape(-1, 3)
    if len(x) == 0:
        return x.copy(), True
    key, ok = np_voxel_keys(x, leaf)
    if not ok:
        return x.copy(), False
    order = np.argsort(key, kind="stable")
    ks = key[order]
    heads = np.concatenate([[True], ks[1:] != ks[:-1]])
    starts = np.nonzero(heads)[0]
    lens = np.diff(np.concatenate([starts, [len(ks)]]))
    s = seq_segment_sums(x[order], starts, lens)
    return (s / lens.astype(F32)[:, None]).astype(F32), True


def np_global_map(clouds, poses, q_bl, t_bl, interval, leaf):
    """(points, filtered, n_raw) of save_pcd's block in the numpy formulation"""
    parts = [np_transform(np_transform(clouds[i], t_bl, q_bl), poses[i][:3], poses[i][3:]) for i in range(0, len(clouds), interval)]
    cat = np.concatenate(parts) if parts else np.zeros((0, 3), F32)
    pts, f = np_voxel_filter(cat, leaf)
    return pts, f, len(cat)


# ---- the oracle's global map -------------------------------------------------------------------------------------------------
def concatenation(po, L, interval):
    """transformCloud(transformCloud(surf_frames[i], &Tbl), &pose_info_keyframe[i]) for i = 0, interval, ..., concatenated"""
    parts = []
    for i in range(0, len(L.clouds), interval):
        c = L.clouds[i]
        if len(c) == 0:
            continue
        p = L.poses[i]
        parts.append(po.transform_points(po.transform_points(c, np.array(L.t_bl), np.array(L.q_bl)), p[:3], p[3:]))
    return np.concatenate(parts) if parts else np.zeros((0, 3), F32)


def global_map(po, L, interval=3, leaf=0.2):
    """(points, filtered, n_raw) of the oracle's store L (pyoracle_loop.LoopOracle): the stable VoxelGrid of the concatenation"""
    cat = concatenation(po, L, interval)
    if len(cat) == 0:
        return cat, True, 0
    f = po.voxel_filter(cat, leaf, stable=True)
    return (cat.copy(), False, len(cat)) if f is None else (f[0], True, len(cat))


# ---- box fixtures ------------------------------------------------------------------------------------------------------------
def box_cloud(lo, hi, n, seed):
    """n points: the two corners lo, hi (they fix the bounds) and n - 2 uniform points between them, shuffled"""
    rng = np.random.default_rng(seed)
    lo = np.asarray(lo, np.float64); hi = np.asarray(hi, np.float64)
    p = np.concatenate([[lo, hi], lo + rng.uniform(0, 1, (n - 2, 3)) * (hi - lo)]).astype(F32)
    return p[rng.permutation(n)]


# leaf 1: (corner lo, corner hi) of boxes whose voxel keys need exactly `bits` bits (the radix sort takes ceil(bits / 8) passes)
KEY_BIT_BOXES = {
    1: ((0.25, 0.25, 0.25), (1.5, 0.75, 0.75)),                 # div (2, 1, 1): keys 0..1
    8: ((0.25, 0.25, 0.25), (128.5, 0.75, 0.75)),               # 129 voxels
    9: ((0.25, 0.25, 0.25), (256.5, 0.75, 0.75)),               # 257
    16: ((0.25, 0.25, 0.25), (32768.5, 0.75, 0.75)),            # 2^15 + 1
    17: ((0.25, 0.25, 0.25), (65536.5, 0.75, 0.75)),            # 2^16 + 1
    24: ((0.25, 0.25, 0.25), (2896.5, 2896.5, 0.75)),           # 2897^2 = 8392609 > 2^23
    25: ((0.25, 0.25, 0.25), (4096.5, 4096.5, 0.75)),           # 4097^2 = 16785409 > 2^24
    32: ((0.9, 0.9, 0.25), (46340.1, 46340.1, 0.75)),           # dx = dy = 46340 (passes), div = 46341: 2147488281 > 2^31
}

# leaf 1: the closest products to INT32_MAX (prime) on either side
BELOW_INT32_MAX = ((0.0, 0.0, 0.0), (2316.5, 1660.5, 557.5))    # 2317 * 1661 * 558 = 2147483646: filtered
ABOVE_INT32_MAX = ((0.0, 0.0, 0.0), (2047.5, 1023.5, 1023.5))   # 2048 * 1024 * 1024 = 2^31: passed through
# div product past 2^32 while dx * dy * dz = 2^30 + 1 passes: keys wrap, voxels 2^30 apart along z share a key
WRAP_BOX = ((0.9, 0.9, 0.5), (1.1, 1.1, 1073741824.0))
# div product 1291^3 between INT32_MAX and 2^32: the int32 key goes negative, the unsigned order puts it last
NEGATIVE_KEY_BOX = ((0.9, 0.9, 0.9), (1290.1, 1290.1, 1290.1))


def wrap_cloud(n=4000, seed=5):
    """WRAP_BOX with points clustered at both ends of z, so that wrapped keys really merge voxels"""
    rng = np.random.default_rng(seed)
    lo, hi = WRAP_BOX
    a = np.stack([rng.uniform(0.9, 1.1, n), rng.uniform(0.9, 1.1, n), rng.uniform(0.5, 3.0, n)], 1)
    b = np.stack([rng.uniform(0.9, 1.1, n), rng.uniform(0.9, 1.1, n), 1073741824.0 - rng.uniform(0, 2000.0, n)], 1)
    p = np.concatenate([[lo, hi], a, b]).astype(F32)
    return p[rng.permutation(len(p))]
