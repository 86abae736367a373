"""Loop-closure registration on the device (glio_icp_align, glio_loop_*) against the sequential oracle (oracle/loop/go_loop.cpp,
oracle/pyoracle_loop.py), bit for bit: every iteration's correspondence count, MSE and transformation, the last correspondence
list, final, iterations, convergence state, aligned cloud and fitness; in the loop step the detection indices, both filtered
clouds, the acceptance and the two poses."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth

pytestmark = pytest.mark.gpu

STRIDE8 = 8


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


def _moved(pts, yaw, t, pitch=0.0):
    q = synth.quat_from_rpy(0.0, pitch, yaw)
    return (np.asarray(pts, np.float64) @ synth.quat_to_R(q).T + np.asarray(t)).astype(np.float32)


def _check(ctx, pl, src, tgt, **opt):
    """device == oracle, every output; returns the oracle's result"""
    g = ctx.icp_align(src, tgt, iter_log=True, correspondences=True, **opt)
    s3 = np.asarray(src)[:, :3] if isinstance(src, np.ndarray) else src.cpu().numpy()[:, :3]
    t3 = np.asarray(tgt)[:, :3] if isinstance(tgt, np.ndarray) else tgt.cpu().numpy()[:, :3]
    o = pl.icp(s3, t3, **opt)
    assert (g["converged"], g["state"], g["iterations"], g["n_corr"]) == (o["converged"], o["state"], o["iterations"], o["n_corr"])
    assert len(g["log"]) == len(o["log"]) == o["iterations"]
    for k, (a, b) in enumerate(zip(g["log"], o["log"])):
        assert a[1] == b[1], f"iteration {k}: correspondence count"
        assert a[2] == b[2], f"iteration {k}: mse {a[2]!r} != {b[2]!r}"
        assert np.array_equal(a[0], b[0]), f"iteration {k}: transformation"
    for a, b in zip(g["corr"], o["corr"]):
        assert np.array_equal(a, b), "last correspondence list"
    assert np.array_equal(g["final"], o["final"])
    assert np.array_equal(g["aligned"], o["aligned"])
    assert g["fitness"] == o["fitness"]
    assert g["n_source"] == len(s3) and g["n_target"] == len(t3)
    return o


def _loop_clouds(pl, K=80, n_points=1500, seed=synth.SEED0 + 31):
    D = synth.loop_drive(K=K, n_points=n_points, dt=1.0, seed=seed)
    L = pl.LoopOracle()
    for k in range(K):
        L.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
    j = K - 5
    r = L.step(D["poses"][j][:3].astype(np.float32), D["times"][j])
    assert r["detected"]
    return r["latest"], r["his"]


# ---- registration, bit for bit -------------------------------------------------------------------------------------
def test_icp_smallest_clouds(ctx, pl):
    rng = np.random.default_rng(1)
    tgt = rng.uniform(-1.0, 1.0, (5, 3)).astype(np.float32)
    src = _moved(tgt[:3], 0.05, [0.02, -0.01, 0.03])
    _check(ctx, pl, src, tgt)


@pytest.mark.parametrize("n_src,n_tgt,seed", [(50, 80, 2), (2000, 5000, 3), (20000, 60000, 4)])
def test_icp_random_rigid_motion(ctx, pl, n_src, n_tgt, seed):
    rng = np.random.default_rng(seed)
    sc = synth.Scene(-50.0, 50.0, rng)
    tgt = sc.sample(n_tgt, rng, -40.0, 40.0).astype(np.float32)
    src = _moved(sc.sample(n_src, rng, -30.0, 30.0), 0.03, [0.8, -0.4, 0.1], pitch=0.01)
    o = _check(ctx, pl, src, tgt)
    assert o["converged"]


def test_icp_realistic_loop_clouds(ctx, pl):
    lat, his = _loop_clouds(pl)
    o = _check(ctx, pl, lat, his)
    assert o["converged"] and o["iterations"] > 5


def test_icp_target_beyond_100k_points_stride8_and_device(ctx, pl):
    import torch
    rng = np.random.default_rng(6)
    sc = synth.Scene(-80.0, 80.0, rng)
    tgt = sc.sample(130_000, rng, -70.0, 70.0).astype(np.float32)
    src = _moved(sc.sample(25_000, rng, -50.0, 50.0), -0.02, [0.5, 0.2, -0.05])
    s8 = np.zeros((len(src), STRIDE8), np.float32); s8[:, :3] = src; s8[:, 4] = 7.0
    o = _check(ctx, pl, s8, torch.from_numpy(tgt).cuda())
    assert o["converged"] and o["fitness"] < 0.05


# ---- edge cases ------------------------------------------------------------------------------------------------------
def test_every_source_point_beyond_the_gate(ctx, pl):
    rng = np.random.default_rng(7)
    tgt = rng.uniform(-5.0, 5.0, (400, 3)).astype(np.float32)
    src = (tgt[:100] + np.array([100.0, 0.0, 0.0], np.float32)).astype(np.float32)
    o = _check(ctx, pl, src, tgt)
    assert not o["converged"] and o["state"] == pl.NO_CORRESPONDENCES and o["iterations"] == 0


def test_identical_clouds_converge_on_the_transform_test_after_one_iteration(ctx, pl):
    rng = np.random.default_rng(8)
    tgt = rng.uniform(-5.0, 5.0, (1000, 3)).astype(np.float32)
    o = _check(ctx, pl, tgt.copy(), tgt)
    assert o["converged"] and o["state"] == pl.TRANSFORM and o["iterations"] == 1


def test_a_run_that_hits_100_iterations(ctx, pl):
    rng = np.random.default_rng(5)
    sc = synth.Scene(-60.0, 60.0, rng)
    tgt = sc.sample(20000, rng, -40.0, 40.0).astype(np.float32)
    src = _moved(sc.sample(6000, rng, -30.0, 30.0), 0.0, [16.0, 0.3, 0.0])    # along the street: slow convergence
    o = _check(ctx, pl, src, tgt)
    assert o["converged"] and o["state"] == pl.ITERATIONS and o["iterations"] == 100


def test_duplicated_target_points_ties_by_index(ctx, pl):
    rng = np.random.default_rng(9)
    base = rng.uniform(-3.0, 3.0, (300, 3)).astype(np.float32)
    tgt = np.concatenate([base, base, base[::-1]])
    src = _moved(base[:200], 0.02, [0.05, 0.0, 0.0])
    o = _check(ctx, pl, src, tgt)
    assert o["iterations"] >= 1
    assert (o["corr"][1] < 300).all(), "a tie must go to the lowest index"


def test_one_point_target(ctx, pl):
    rng = np.random.default_rng(10)
    tgt = np.array([[1.0, 2.0, 3.0]], np.float32)
    src = (rng.uniform(-1.0, 1.0, (10, 3)) + [1.0, 2.0, 3.0]).astype(np.float32)
    _check(ctx, pl, src, tgt)


def test_source_outside_the_target_bounding_box(ctx, pl):
    rng = np.random.default_rng(11)
    tgt = rng.uniform(0.0, 4.0, (3000, 3)).astype(np.float32)
    src = (rng.uniform(0.0, 4.0, (500, 3)) + [15.0, -12.0, 6.0]).astype(np.float32)
    _check(ctx, pl, src, tgt)


def test_fewer_than_three_correspondences(ctx, pl):
    tgt = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    src = np.array([[0.1, 0, 0], [0, 0.1, 0], [50, 50, 50]], np.float32)
    o = _check(ctx, pl, src, tgt)
    assert o["state"] == pl.NO_CORRESPONDENCES and o["n_corr"] == 2


# ---- the loop step -----------------------------------------------------------------------------------------------
def _drive(loop, oracle, D, ks, sww=5, check_clouds=True):
    """add keyframes ks one by one and step after each, as the Estimator does with the keyframe that just left the window"""
    n_acc = 0
    for k in ks:
        loop.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
        oracle.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
        if len(oracle.clouds) < sww:
            continue
        j = len(oracle.clouds) - sww
        sel = D["poses"][j][:3].astype(np.float32)
        g = loop.step(sel, D["times"][j])
        o = oracle.step(sel, D["times"][j])
        assert (g["detected"], g["closest_his_idx"]) == (o["detected"], o["closest_his_idx"]) and g["n_candidates"] == o["n_candidates"]
        assert g["time_last_loop"] == o["time_last_loop"]
        if not o["detected"]:
            assert g["icp"] is None
            continue
        assert g["latest_frame_idx"] == o["latest_frame_idx"]
        assert (g["n_latest"], g["n_his"], g["n_latest_ds"], g["n_his_ds"]) == (o["n_latest"], o["n_his"], len(o["latest"]), len(o["his"]))
        if check_clouds:
            a, b = loop.clouds()
            assert np.array_equal(a, o["latest"]) and np.array_equal(b, o["his"])
        gi, oi = g["icp"], o["icp"]
        assert (gi["converged"], gi["state"], gi["iterations"], gi["n_corr"]) == (oi["converged"], oi["state"], oi["iterations"], oi["n_corr"])
        assert np.array_equal(gi["final"], oi["final"]) and gi["fitness"] == oi["fitness"]
        assert g["accepted"] == o["accepted"]
        if o["accepted"]:
            n_acc += 1
            assert np.array_equal(g["pose_from"], o["pose_from"]) and np.array_equal(g["pose_to"], o["pose_to"])
            assert g["noise_score"] == o["noise_score"]
    return n_acc


def test_loop_step_matches_the_oracle_along_a_closed_drive(ctx, pl):
    from glio_b200 import api
    D = synth.loop_drive(K=80, n_points=1500, dt=1.0, seed=synth.SEED0 + 32)
    loop = api.LoopClosure(ctx)
    oracle = pl.LoopOracle()
    try:
        n_acc = _drive(loop, oracle, D, range(70))
        assert n_acc > 5, "the drive is supposed to close its loop"
        # correctPoses: the store takes new poses, the next registrations use them
        new = D["poses"][:70].copy(); new[:, 0] += 0.05; new[:, 1] -= 0.02
        loop.set_poses(0, new); oracle.set_poses(0, new)
        for k in range(70):
            D["poses"][k] = new[k]
        _drive(loop, oracle, D, range(70, 80))
        assert len(loop) == 80
    finally:
        loop.close()


def test_loop_step_with_device_keyframes_and_other_options(ctx, pl):
    import torch
    from glio_b200 import api
    D = synth.loop_drive(K=60, n_points=1200, dt=1.0, seed=synth.SEED0 + 33, drift_t=0.02)
    opt = dict(lc_search_radius=7.0, lc_map_width=10, lc_icp_thres=0.3, slide_window_width=3, q_lb=synth.quat_from_rpy(0.01, 0.0, 0.02),
               t_lb=(0.1, -0.05, 0.28))
    loop = api.LoopClosure(ctx, **opt)
    oracle = pl.LoopOracle(**opt)
    try:
        dev = dict(D)
        dev["clouds"] = [torch.from_numpy(np.concatenate([c, np.ones((len(c), 1), np.float32)], 1)).cuda() for c in D["clouds"]]
        n = 0
        for k in range(60):
            loop.add_keyframe(dev["clouds"][k], D["poses"][k], D["times"][k])
            oracle.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
            if len(oracle.clouds) < 3:
                continue
            j = len(oracle.clouds) - 3
            sel = D["poses"][j][:3].astype(np.float32)
            g = loop.step(sel, D["times"][j]); o = oracle.step(sel, D["times"][j])
            assert (g["detected"], g["closest_his_idx"], g["accepted"]) == (o["detected"], o["closest_his_idx"], o["accepted"])
            if o["detected"]:
                n += 1
                a, b = loop.clouds()
                assert np.array_equal(a, o["latest"]) and np.array_equal(b, o["his"])
                assert np.array_equal(g["icp"]["final"], o["icp"]["final"]) and g["icp"]["fitness"] == o["icp"]["fitness"]
            if o["accepted"]:
                assert np.array_equal(g["pose_from"], o["pose_from"]) and np.array_equal(g["pose_to"], o["pose_to"])
        assert n > 0
    finally:
        loop.close()


def test_no_candidate_and_too_recent_candidate_launch_nothing(ctx, pl):
    from glio_b200 import api
    D = synth.loop_drive(K=80, n_points=500, dt=1.0, seed=synth.SEED0 + 34)
    loop = api.LoopClosure(ctx)
    try:
        n0 = ctx.launch_count
        r = loop.step(np.zeros(3, np.float32), 0.0)                       # no keyframe at all
        assert not r["detected"] and r["closest_his_idx"] == -1 and ctx.launch_count == n0
        for k in range(30):
            loop.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
        n0 = ctx.launch_count
        r = loop.step(D["poses"][25][:3].astype(np.float32), D["times"][25])   # every neighbour is less than 30 s away
        assert not r["detected"] and r["closest_his_idx"] == -1 and r["n_candidates"] > 0 and ctx.launch_count == n0
        r = loop.step(np.array([1e4, 0, 0], np.float32), D["times"][25])        # nothing within the radius
        assert not r["detected"] and r["n_candidates"] == 0 and ctx.launch_count == n0
        # a candidate that passes the time test but comes less than 0.2 s after the last loop
        for k in range(30, 80):
            loop.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
        j = 75
        r = loop.step(D["poses"][j][:3].astype(np.float32), D["times"][j])
        assert r["detected"] and r["accepted"], r
        assert r["time_last_loop"] == D["times"][j]
        n0 = ctx.launch_count
        r2 = loop.step(D["poses"][j][:3].astype(np.float32), D["times"][j] + 0.1)
        assert r2["closest_his_idx"] >= 0 and not r2["detected"] and ctx.launch_count == n0
    finally:
        loop.close()


def test_host_synchronisations_per_registration(ctx, pl):
    rng = np.random.default_rng(12)
    tgt = rng.uniform(-5.0, 5.0, (1000, 3)).astype(np.float32)
    g = ctx.icp_align(tgt.copy(), tgt)
    assert g["iterations"] == 1 and g["host_syncs"] == 3       # grid bounds, one batch, the result


# ---- argument errors ------------------------------------------------------------------------------------------------
def test_argument_errors_leave_the_context_usable(ctx, pl):
    import torch
    from glio_b200 import api
    L = ctx._lib
    a = np.zeros((10, 3), np.float32)
    res = api.IcpResult()
    ptr = a.ctypes.data_as(C.c_void_p)
    bad = [
        (ptr, 10, 2, api.HOST, ptr, 10, 3, api.HOST),                 # stride
        (ptr, 10, 3, api.DEVICE, ptr, 10, 3, api.HOST),               # a host pointer claimed as device memory
        (ptr, -1, 3, api.HOST, ptr, 10, 3, api.HOST),                 # size
        (None, 10, 3, api.HOST, ptr, 10, 3, api.HOST),                # null
        (ptr, 10, 3, 7, ptr, 10, 3, api.HOST),                        # mem
    ]
    t8 = torch.zeros(64, dtype=torch.uint8, device="cuda")
    bad.append((C.c_void_p(t8.data_ptr() + 2), 4, 3, api.DEVICE, ptr, 10, 3, api.HOST))   # misaligned device pointer
    n0 = ctx.launch_count
    for b in bad:
        rc = L.glio_icp_align(ctx._h, b[0], C.c_int64(b[1]), C.c_int(b[2]), C.c_int(b[3]), b[4], C.c_int64(b[5]), C.c_int(b[6]), C.c_int(b[7]),
                              None, None, C.byref(res), None, C.c_int(0), None, None, None, C.c_int64(0))
        assert rc == -3, b
    opt = api.default_icp_options(max_iterations=0)
    assert L.glio_icp_align(ctx._h, ptr, C.c_int64(10), C.c_int(3), C.c_int(0), ptr, C.c_int64(10), C.c_int(3), C.c_int(0), C.byref(opt), None,
                            C.byref(res), None, C.c_int(0), None, None, None, C.c_int64(0)) == -3
    assert ctx.launch_count == n0
    loop = api.LoopClosure(ctx)
    try:
        with pytest.raises(api.GlioError):
            loop.add_keyframe(np.zeros((5, 2), np.float32), np.array([0, 0, 0, 1.0, 0, 0, 0]), 0.0)
        with pytest.raises(api.GlioError):
            loop.add_keyframe(a, np.array([0, 0, np.nan, 1.0, 0, 0, 0]), 0.0)
        loop.add_keyframe(a, np.array([0, 0, 0, 1.0, 0, 0, 0]), 0.0)
        with pytest.raises(api.GlioError):
            loop.set_poses(0, np.zeros((2, 7)))                        # keyframe 1 does not exist
        with pytest.raises(api.GlioError):
            loop.step(np.array([np.nan, 0, 0], np.float32), 1.0)
        rc = L.glio_loop_add_keyframe(loop._h, ptr, C.c_int64(10), C.c_int(3), C.c_int(api.DEVICE),
                                      np.array([0, 0, 0, 1.0, 0, 0, 0]).ctypes.data_as(C.c_void_p), C.c_double(0.0), None)
        assert rc == -3
        assert len(loop) == 1
    finally:
        loop.close()
    with pytest.raises(api.GlioError):
        api.LoopClosure(ctx, slide_window_width=0)
    assert ctx.launch_count == n0
    rng = np.random.default_rng(13)
    tgt = rng.uniform(-5.0, 5.0, (500, 3)).astype(np.float32)
    _check(ctx, pl, _moved(tgt[:300], 0.02, [0.1, 0.0, 0.0]), tgt)


# ---- non-interference ---------------------------------------------------------------------------------------------
def _window_results(c, P):
    from glio_b200 import api
    c.set_map(P["map_xyz"])
    c.window_set_scans(P["scans"])
    nm = c.window_associate(P["poses_init"])
    m = c.get_matches(0, len(P["scans"][0]))
    r = c.window_solve(P["poses_init"], None, None, api.default_solver_options())
    return nm, m, r


def test_loop_closure_leaves_the_context_alone(pl):
    from glio_b200 import api
    P = synth.window_problem(W=3, Q=2000, M=40000, seed=synth.SEED0 + 21)
    D = synth.loop_drive(K=70, n_points=800, dt=1.0, seed=synth.SEED0 + 35)
    c = api.Context(0)
    fresh = api.Context(0)
    try:
        a = _window_results(c, P)
        loop = api.LoopClosure(c)
        for k in range(70):
            loop.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
        r = loop.step(D["poses"][65][:3].astype(np.float32), D["times"][65])
        assert r["detected"]
        rng = np.random.default_rng(14)
        tgt = rng.uniform(-5.0, 5.0, (500, 3)).astype(np.float32)
        c.icp_align(tgt[:100].copy(), tgt)
        b = _window_results(c, P)
        d = _window_results(fresh, P)
        for x in (b, d):
            assert np.array_equal(a[0], x[0])
            assert all(np.array_equal(a[1][k], x[1][k]) for k in ("cp", "nsd", "weight"))
            assert np.array_equal(a[2]["poses"], x[2]["poses"]) and len(a[2]["steps"]) == len(x[2]["steps"])
            assert all(np.array_equal(s, t) for s, t in zip(a[2]["steps"], x[2]["steps"]))
    finally:
        c.close(); fresh.close()     # the loop object is freed with its context
