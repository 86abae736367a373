"""The sort-based VoxelGrid (glio_voxel_filter, Context.voxel_filter) and save_pcd's global map (glio_loop_global_map,
LoopClosure.global_map) on the device against the CPU oracle's stable order, bit for bit: leaves, strides, host and device memory,
point counts around the warp and tile sizes up to 2 million, negative coordinates and points on voxel faces, voxels of 1 to 5000
points 1000 m out, agreement with the dense filter of glio_localmap_build wherever that one applies, boxes past 2^28 voxels, at
both sides of PCL's INT32_MAX leaf-size check and with wrapped keys, the number of radix passes per key width, argument errors,
the loop drive's keyframe store, and that neither entry point disturbs the context, its odometries or its loop objects.  The
oracle's global map and the box fixtures live in tests/global_map_reference.py, which tests/test_global_map.py checks on the CPU
against an independent numpy formulation."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth
from tests.global_map_reference import (ABOVE_INT32_MAX, BELOW_INT32_MAX, F32, KEY_BIT_BOXES, NEGATIVE_KEY_BOX, box_cloud, concatenation,
                                        global_map, wrap_cloud)

pytestmark = pytest.mark.gpu

IDENT_T = np.zeros(3)
IDENT_Q = np.array([1.0, 0, 0, 0])
EXTRINSIC = dict(q_lb=synth.quat_from_rpy(0.01, -0.015, 0.02), t_lb=(0.1, -0.05, 0.28))
ERR_ARG = -3


@pytest.fixture(scope="module")
def ctx():
    from glio_b200 import api
    c = api.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pl():
    from oracle import pyoracle_loop
    pyoracle_loop.build()
    return pyoracle_loop


def scene_cloud(n, leaf, seed):
    """negative and positive coordinates, with a quarter of the points exactly on voxel faces (multiples of the leaf)"""
    rng = np.random.default_rng(seed)
    x = np.concatenate([rng.uniform(-60, 60, (n, 2)), rng.uniform(-5, 15, (n, 1))], 1)
    face = rng.random((n, 3)) < 0.25
    x = np.where(face, np.round(x / leaf) * leaf, x).astype(F32)
    return x


def strided(x, stride, seed=0):
    """x in columns 0..2 of an (n, stride) array; the other lanes hold noise, NaN among it (never read)"""
    if stride == 3:
        return np.ascontiguousarray(x)
    rng = np.random.default_rng(seed)
    a = rng.normal(size=(len(x), stride)).astype(F32)
    a[:, 3:][rng.random((len(x), stride - 3)) < 0.1] = np.nan
    a[:, :3] = x
    return a


def oracle_filter(oracle, x, leaf):
    r = oracle.voxel_filter(np.ascontiguousarray(x[:, :3]), leaf, stable=True)
    return (np.ascontiguousarray(x[:, :3]), False) if r is None else (r[0], True)


def check(ctx, oracle, x, leaf, buf=None, out="host", filtered=True):
    """ctx.voxel_filter(buf or x) == the oracle's stable VoxelGrid of x, bit for bit"""
    got, f = ctx.voxel_filter(x if buf is None else buf, leaf, out=out)
    if out == "device":
        assert got.is_cuda
        got = got.cpu().numpy()
    ref, g = oracle_filter(oracle, x, leaf)
    assert f == g == filtered
    assert got.shape == ref.shape and np.array_equal(got, ref)
    return ref


def launches(ctx, name):
    return ctx.lib_profile_read().get(name, (0, 0))[1]


# ---- inputs ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 100_000, 2_000_000])
def test_point_counts(ctx, oracle, n):
    import torch
    leaf = {1: 0.9, 31: 0.4, 32: 0.2, 33: 0.9, 1000: 0.4, 100_000: 0.2, 2_000_000: 0.2}[n]
    x = scene_cloud(n, leaf, seed=n)
    check(ctx, oracle, x, leaf)
    check(ctx, oracle, x, leaf, buf=torch.from_numpy(x).cuda(), out="device")


@pytest.mark.parametrize("stride", [3, 4, 8])
@pytest.mark.parametrize("in_mem,out", [("host", "host"), ("host", "device"), ("device", "host"), ("device", "device")])
def test_strides_and_memory(ctx, oracle, stride, in_mem, out):
    import torch
    x = scene_cloud(20000, 0.4, seed=stride)
    a = strided(x, stride, seed=stride)
    buf = a if in_mem == "host" else torch.from_numpy(a).cuda()
    check(ctx, oracle, x, 0.4, buf=buf, out=out)


@pytest.mark.parametrize("leaf", [0.9, 0.4, 0.2])
def test_leaves_with_faces_and_negative_coordinates(ctx, oracle, leaf):
    x = scene_cloud(50000, leaf, seed=int(100 * leaf))
    on_face = np.isclose(x / F32(leaf), np.round(x / F32(leaf)), rtol=0, atol=1e-3)
    assert on_face.any(axis=1).mean() > 0.3 and (x < 0).any(axis=0).all()
    ref = check(ctx, oracle, x, leaf)
    assert len(ref) < len(x)


POPULATIONS = [1, 2, 31, 32, 33, 255, 256, 257, 1000, 2048, 2049, 5000]


def test_voxel_populations_1000_m_out(ctx, oracle):
    """one voxel per population, interleaved, about 1000 m out, where the order of a voxel's points changes its float sum"""
    rng = np.random.default_rng(31)
    leaf = 0.4
    pts = [(np.array([2500 + 3 * v, -2500 + v, 40]) + 0.5) * leaf + rng.uniform(-0.35 * leaf, 0.35 * leaf, (n, 3)) for v, n in enumerate(POPULATIONS)]
    x = np.concatenate(pts).astype(F32)[rng.permutation(sum(POPULATIONS))]
    ref = check(ctx, oracle, x, leaf)
    assert len(ref) == len(POPULATIONS)
    lit = oracle.voxel_filter(x, leaf, stable=False)[0]
    assert not np.array_equal(lit, ref)                       # std::sort's order gives other bits: an unstable sort would be caught
    for n in (1, 5000):                                         # a voxel alone in its cloud: no key bit, no radix pass
        x1 = (np.array([1000.3, -1000.3, 40.3]) + rng.uniform(-0.1, 0.1, (n, 3))).astype(F32)
        check(ctx, oracle, x1, leaf)


# ---- agreement with the dense filter ----------------------------------------------------------------------------------------
def dense(ctx, x, leaf):
    ctx.localmap_clear()
    ctx.localmap_push(x, IDENT_T, IDENT_Q)
    ctx.localmap_build(leaf)
    m = ctx.get_map()
    ctx.localmap_clear()
    return m


def test_agrees_with_the_dense_filter(ctx, oracle):
    from tests.test_frontend_edges import SCAN_BOXES, scan_box_points
    cases = [(scene_cloud(60000, leaf, seed=7), leaf) for leaf in (0.9, 0.4, 0.2)]
    cases += [(box_cloud(*KEY_BIT_BOXES[b], 6000, seed=b), 1.0) for b in (8, 9, 16, 17, 24, 25)]
    cases += [(scan_box_points(nx, ny), 1.0) for nx, ny in SCAN_BOXES]
    for x, leaf in cases:
        got, f = ctx.voxel_filter(x, leaf)
        assert f and np.array_equal(got, dense(ctx, x, leaf))


# ---- large boxes -------------------------------------------------------------------------------------------------------------
def test_box_the_dense_filter_refuses(ctx, oracle):
    from glio_b200 import api
    rng = np.random.default_rng(34)
    x = np.concatenate([[[3900.5, 3900.5, 0.5]], rng.uniform(-20, 20, (20000, 3))]).astype(F32)
    with pytest.raises(api.GlioError, match=r"2\^28 voxels"):
        dense(ctx, x, 1.0)
    ctx.localmap_clear()
    check(ctx, oracle, x, 1.0)


def test_int32_max_and_wrapped_keys(ctx, oracle):
    check(ctx, oracle, box_cloud(*BELOW_INT32_MAX, 3000, seed=2), 1.0, filtered=True)
    x = box_cloud(*ABOVE_INT32_MAX, 3000, seed=3)
    got = check(ctx, oracle, x, 1.0, filtered=False)
    assert np.array_equal(got, x)                               # the input, in input order
    check(ctx, oracle, wrap_cloud(), 1.0)
    check(ctx, oracle, box_cloud(*NEGATIVE_KEY_BOX, 5000, seed=4), 1.0)


@pytest.mark.parametrize("bits", sorted(KEY_BIT_BOXES))
def test_radix_passes_follow_the_key_width(ctx, oracle, bits):
    x = box_cloud(*KEY_BIT_BOXES[bits], 5000, seed=bits)
    ctx.lib_profile(True)
    try:
        check(ctx, oracle, x, 1.0)
        n_hist, n_scatter = launches(ctx, "k_vs_hist"), launches(ctx, "k_vs_scatter")
        n_key, n_cent = launches(ctx, "k_vs_key"), launches(ctx, "k_vs_centroid")
    finally:
        ctx.lib_profile(False)
    assert n_hist == n_scatter == (bits + 7) // 8 and n_key == n_cent == 1


# ---- argument errors ---------------------------------------------------------------------------------------------------------
def raw(ctx, p, n, stride, in_mem, leaf, cap, out, out_mem, n_out=True):
    m = C.c_int64(-7); f = C.c_int32(-7)
    rc = ctx._lib.glio_voxel_filter(ctx._h, p, C.c_int64(n), C.c_int(stride), C.c_int(in_mem), C.c_float(leaf), C.c_int64(cap), out,
                                    C.c_int(out_mem), C.byref(m) if n_out else None, C.byref(f))
    return rc, m.value, f.value


def test_argument_errors_leave_the_context_usable(ctx, oracle):
    import torch
    from glio_b200 import api
    H, D = api.HOST, api.DEVICE
    x = scene_cloud(1000, 0.4, seed=9)
    ref, _ = oracle_filter(oracle, x, 0.4)
    hp = x.ctypes.data_as(C.c_void_p)
    out = np.zeros((1000, 3), F32)
    op = out.ctypes.data_as(C.c_void_p)
    dx = torch.from_numpy(x).cuda()
    t8 = torch.zeros(64, dtype=torch.uint8, device="cuda")
    dout = torch.zeros((1000, 3), dtype=torch.float32, device="cuda")
    dp, dop = C.c_void_p(dx.data_ptr()), C.c_void_p(dout.data_ptr())
    n0 = ctx.launch_count
    bad = [
        (hp, 1000, 2, H, 0.4, 1000, op, H), (hp, 1000, 65, H, 0.4, 1000, op, H),      # stride
        (hp, 1000, 3, H, 0.0, 1000, op, H), (hp, 1000, 3, H, -0.4, 1000, op, H),      # leaf <= 0
        (hp, 1000, 3, H, float("nan"), 1000, op, H), (hp, 1000, 3, H, float("inf"), 1000, op, H),
        (None, 1000, 3, H, 0.4, 1000, op, H), (hp, 1000, 3, H, 0.4, 1000, None, H),   # null cloud, null output
        (hp, -1, 3, H, 0.4, 1000, op, H), (hp, 1000, 3, H, 0.4, -1, op, H),           # sizes
        (hp, 1000, 3, 7, 0.4, 1000, op, H), (hp, 1000, 3, H, 0.4, 1000, op, 7),       # mem
        (hp, 1000, 3, D, 0.4, 1000, op, H), (hp, 1000, 3, H, 0.4, 1000, op, D),       # host memory claimed as device memory
        (C.c_void_p(t8.data_ptr() + 2), 4, 3, D, 0.4, 1000, op, H),                   # misaligned device cloud
        (hp, 1000, 3, H, 0.4, 10, C.c_void_p(t8.data_ptr() + 2), D),                  # misaligned device output
    ]
    for b in bad:
        assert raw(ctx, *b)[0] == ERR_ARG, b
    assert raw(ctx, hp, 1000, 3, H, 0.4, 1000, op, H, n_out=False)[0] == ERR_ARG
    assert ctx.launch_count == n0                               # refused before anything ran
    for v in (np.nan, np.inf, -np.inf):                         # non-finite coordinates, host and device, one point or all of them
        for rows in ([17], slice(None)):
            y = x.copy(); y[rows, 1] = v
            assert raw(ctx, y.ctypes.data_as(C.c_void_p), 1000, 3, H, 0.4, 1000, op, H)[0] == ERR_ARG
            dy = torch.from_numpy(y).cuda()
            assert raw(ctx, C.c_void_p(dy.data_ptr()), 1000, 3, D, 0.4, 1000, dop, D)[0] == ERR_ARG
    y = x.copy(); y[5, 0] = np.nan
    assert raw(ctx, y.ctypes.data_as(C.c_void_p), 1000, 3, H, 1e-4, 1000, op, H)[0] == ERR_ARG    # in PCL's pass-through too
    # capacity too small: the true count comes back, nothing is written past the capacity (here: nothing at all)
    for mem, o, ptr in ((H, out, op), (D, dout, dop)):
        o[:] = 7.0
        rc, m, f = raw(ctx, hp, 1000, 3, H, 0.4, len(ref) - 1, ptr, mem)
        assert rc == ERR_ARG and m == len(ref)
        got = o.cpu().numpy() if mem == D else o
        assert (got == 7.0).all()
    n0 = ctx.launch_count
    assert raw(ctx, None, 0, 3, H, 0.4, 0, None, H) == (0, 0, 1)                  # an empty cloud launches nothing
    assert ctx.launch_count == n0
    e, f = ctx.voxel_filter(np.zeros((0, 3), F32), 0.4)
    assert e.shape == (0, 3) and f
    check(ctx, oracle, x, 0.4)                                  # still usable


# ---- global map ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def drive():
    return synth.loop_drive()                                    # 240 keyframes x 2500 points


def fill(loop, L, D, ks=None):
    for k in (range(D["K"]) if ks is None else ks):
        loop.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
        L.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])


def check_map(ctx, oracle, loop, L, interval, leaf, out="host"):
    got, f, n_raw = loop.global_map(interval, leaf, out=out)
    if out == "device":
        got = got.cpu().numpy()
    ref, g, r = global_map(oracle, L, interval, leaf)
    assert (f, n_raw) == (g, r)
    assert got.shape == ref.shape and np.array_equal(got, ref)
    return got


def test_global_map_of_the_loop_drive(ctx, oracle, pl, drive):
    from glio_b200 import api
    loop = api.LoopClosure(ctx); L = pl.LoopOracle()
    try:
        fill(loop, L, drive)
        for stage in range(2):                                   # as inserted, then after correctPoses
            for interval, leaf in ((1, 0.2), (3, 0.2), (1, 0.4), (3, 0.4)):
                got = check_map(ctx, oracle, loop, L, interval, leaf, out="device" if interval == 3 and leaf == 0.4 else "host")
                assert np.array_equal(loop.global_map(interval, leaf)[0], got)            # repeated calls: the same bits
            new = np.array(L.poses); new[:, 0] += 0.05; new[:, 1] -= 0.02; new[:, 3:] = [synth.quat_mul(synth.quat_from_rpy(0, 0, 0.001), q) for q in new[:, 3:]]
            loop.set_poses(0, new); L.set_poses(0, new)
    finally:
        loop.close()


def test_global_map_edge_stores(ctx, oracle, pl):
    from glio_b200 import api
    D = synth.loop_drive(K=12, n_points=800, dt=1.0, seed=synth.SEED0 + 43)
    loop = api.LoopClosure(ctx, **EXTRINSIC); L = pl.LoopOracle(**EXTRINSIC)
    try:
        n0 = ctx.launch_count
        got, f, n_raw = loop.global_map(3, 0.2)                  # an empty store
        assert got.shape == (0, 3) and f and n_raw == 0 and ctx.launch_count == n0
        empty = np.zeros((0, 3), F32)
        for k in range(D["K"]):                                  # every third keyframe cloud empty
            c = empty if k % 3 == 1 else D["clouds"][k]
            loop.add_keyframe(c, D["poses"][k], D["times"][k]); L.add_keyframe(c, D["poses"][k], D["times"][k])
        for interval in (1, 2, 3, D["K"], D["K"] + 5):           # interval >= size: keyframe 0 alone
            check_map(ctx, oracle, loop, L, interval, 0.2)
        # a far keyframe stretches the box past 2^28 voxels (sort range), a farther one past INT32_MAX (PCL's pass-through)
        for far, filtered in ((np.array([8000.0, 0.0, 0.0]), True), (np.array([2.0e6, 1.0e6, 0.0]), False)):
            pose = D["poses"][0].copy(); pose[:3] += far
            loop.add_keyframe(D["clouds"][0], pose, D["times"][-1] + 1); L.add_keyframe(D["clouds"][0], pose, D["times"][-1] + 1)
            got = check_map(ctx, oracle, loop, L, 1, 0.2)
            ref, g, _ = global_map(oracle, L, 1, 0.2)
            cat = concatenation(oracle, L, 1)
            box = np.prod([int(F32(cat[:, k].max() - cat[:, k].min()) * F32(5)) + 1 for k in range(3)], dtype=np.float64)
            assert g == filtered and box > 2**28 and (box <= 2**31 - 1) == filtered
            if not filtered:
                assert np.array_equal(got, concatenation(oracle, L, 1))
        # the two transforms round twice: the device's concatenation (passed through at a tiny leaf) differs from one combined pose
        cat, f, n_raw = loop.global_map(1, 1e-4)
        assert not f and np.array_equal(cat, concatenation(oracle, L, 1))
        one = np.concatenate([oracle.transform_points(c, *map(np.array, pl.world_of_cloud(p, L.q_bl, L.t_bl)))
                              for c, p in zip(L.clouds, L.poses) if len(c)])
        assert one.shape == cat.shape and not np.array_equal(one, cat)
        with pytest.raises(api.GlioError):
            loop.global_map(0, 0.2)
        with pytest.raises(api.GlioError):
            loop.global_map(3, 0.0)
        check_map(ctx, oracle, loop, L, 3, 0.4)
    finally:
        loop.close()


# ---- non-interference ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sweeps():
    """surf features and full clouds of four sweeps of the device front end"""
    from glio_b200 import api
    R = synth.raw_drive(4)
    c = api.Context(0)
    st = api.ImuState()
    surf, full = [], []
    try:
        for k in range(4):
            q = api.imu_sweep_rotation(st, R["stamps"], R["gyro"], R["t_scan_next"][k])
            cloud, ss, se = c.prepare_scan(R["sweeps"][k], 32, q_imu=q)
            surf.append(c.extract_features(cloud, ss, se, 1, 1.0, 0.1, 0.4)["less_flat_ds"].copy()); full.append(cloud.copy())
    finally:
        c.close()
    return surf, full


def _window_results(c, P):
    from glio_b200 import api
    c.set_map(P["map_xyz"])
    c.window_set_scans(P["scans"])
    nm = c.window_associate(P["poses_init"])
    m = c.get_matches(0, len(P["scans"][0]))
    r = c.window_solve(P["poses_init"], None, None, api.default_solver_options())
    return nm, m, r


def _odom_key(r):
    return (r["pose"].tobytes(), r["rel_pose"].tobytes(), r["keyframe"], r["n_map"], r["n_scan"], [x["pose"].tobytes() for x in r["rounds"]])


def _loop_key(r):
    i = r["icp"]
    return (r["detected"], r["closest_his_idx"], r["accepted"], r["n_latest_ds"], r["n_his_ds"], i["final"].tobytes(), i["fitness"],
            None if r["pose_from"] is None else r["pose_from"].tobytes())


def test_the_filters_leave_the_context_alone(sweeps):
    import torch
    from glio_b200 import api
    surf, full = sweeps
    P = synth.window_problem(W=3, Q=2000, M=40000, seed=synth.SEED0 + 21)
    D = synth.loop_drive(K=70, n_points=800, dt=1.0, seed=synth.SEED0 + 35)
    c = api.Context(0); fresh = api.Context(0)
    try:
        a = _window_results(c, P)
        objs = []
        for ctx in (c, fresh):
            odo = api.Odometry(ctx, max_solver_time_s=1e9)
            loop = api.LoopClosure(ctx)
            for k in range(70):
                loop.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
            r0 = [odo.step(surf[k], full[k]) for k in range(2)]
            ctx.localmap_clear()
            for k in range(3):
                ctx.localmap_push(D["clouds"][k], D["poses"][k][:3], D["poses"][k][3:])
            ctx.localmap_build(0.4)
            objs.append((odo, loop, r0, ctx.get_map()))
        # the exports, on c only
        for k in range(3):
            c.voxel_filter(full[k], 0.9); c.voxel_filter(torch.from_numpy(full[k]).cuda(), 0.2, out="device")
        objs[0][1].global_map(3, 0.2); objs[0][1].global_map(1, 0.4, out="device")
        with pytest.raises(api.GlioError):
            c.voxel_filter(np.full((10, 3), np.nan, F32), 0.4)
        (o1, l1, r1, m1), (o2, l2, r2, m2) = objs
        assert np.array_equal(c.get_map(), m1) and np.array_equal(m1, m2)
        assert [_odom_key(x) for x in r1] == [_odom_key(x) for x in r2]
        assert [_odom_key(o1.step(surf[k], full[k])) for k in (2, 3)] == [_odom_key(o2.step(surf[k], full[k])) for k in (2, 3)]
        sel = D["poses"][65][:3].astype(np.float32)
        g1, g2 = l1.step(sel, D["times"][65]), l2.step(sel, D["times"][65])
        assert g1["detected"] and _loop_key(g1) == _loop_key(g2)
        b = _window_results(c, P)
        d = _window_results(fresh, P)
        for x in (b, d):
            assert np.array_equal(a[0], x[0])
            assert all(np.array_equal(a[1][k], x[1][k]) for k in ("cp", "nsd", "weight"))
            assert np.array_equal(a[2]["poses"], x[2]["poses"]) and len(a[2]["steps"]) == len(x[2]["steps"])
            assert all(np.array_equal(s, t) for s, t in zip(a[2]["steps"], x[2]["steps"]))
    finally:
        c.close(); fresh.close()


# ---- hand-off --------------------------------------------------------------------------------------------------------------------
def test_keyframe_cloud_filtered_on_the_device_hands_off(oracle, pl, sweeps):
    """downSampleCloud's surf_last_ds on the device: the odometry's keyframe surf cloud -> voxel_filter(0.9) -> the window slot and the
    loop store, with no host copy in between"""
    import torch
    from glio_b200 import api
    surf, full = sweeps
    c = api.Context(0)
    try:
        odo = api.Odometry(c, deskew=1, max_solver_time_s=1e9)
        odo.step(surf[0], torch.from_numpy(full[0]).cuda(), out="device")
        g = odo.step(surf[1], torch.from_numpy(full[1]).cuda(), out="device")
        assert g["keyframe"] and g["surf"].is_cuda
        ds, f = c.voxel_filter(g["surf"], 0.9, out="device")
        assert f and ds.is_cuda and ds.shape[1] == 3
        ref, _ = oracle_filter(oracle, g["surf"].cpu().numpy(), 0.9)
        assert np.array_equal(ds.cpu().numpy(), ref)
        c.window_set_scan(0, ds)
        loop = api.LoopClosure(c); L = pl.LoopOracle()
        loop.add_keyframe(ds, g["pose"], 1.0); L.add_keyframe(ref, g["pose"], 1.0)
        map_xyz = np.ascontiguousarray(full[1][:, :3])
        c.set_map(map_xyz)
        pose = np.array([0, 0, 0, 1.0, 0, 0, 0])
        nm = c.window_associate(pose[None])
        t2, q2 = c.lidar_pose(pose)
        o = oracle.assoc_scan_to_map(map_xyz, ref, t2, q2)
        v = o["status"] == oracle.GO_VALID
        m = c.get_matches(0, len(ref))
        assert nm[0] == o["nvalid"] > 0
        assert np.array_equal(m["src"], np.nonzero(v)[0].astype(np.int32))
        assert np.array_equal(m["nsd"], o["nsd"][v]) and np.array_equal(m["weight"], o["weight"][v])
        check_map(c, oracle, loop, L, 1, 0.2)                    # the store took the filtered cloud
    finally:
        c.close()
