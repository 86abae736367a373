"""The front end's LidarOdometry node on the device (glio_odom_*) against the CPU oracle's literal restatement
(oracle/pyoracle_odom.py), on a seeded 40-sweep drive that goes through the device chain prepare_scan(out="device") ->
extract_features -> Odometry.step with the full cloud device-resident.

Parity runs set max_solver_time_s to 1e9: the shipped 0.015 s limit is wall clock, which no two runs reproduce; the limit's own
path is tested on its own (max_solver_time_s = 0)."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth

pytestmark = pytest.mark.gpu

K = 40
NO_LIMIT = 1e9


@pytest.fixture(scope="module")
def inputs():
    """Per sweep: the device chain's surf features (host, as extract_features returns them) and full cloud (host copy)."""
    import torch
    from glio_b200 import api
    D = synth.raw_drive(K)
    ctx = api.Context(0)
    st = api.ImuState()
    surf, full = [], []
    try:
        for k in range(K):
            q = api.imu_sweep_rotation(st, D["stamps"], D["gyro"], D["t_scan_next"][k])
            cloud, ss, se = ctx.prepare_scan(D["sweeps"][k], 32, q_imu=q, out="device")
            f = ctx.extract_features(cloud, ss, se, 1, 1.0, 0.1, 0.4)
            surf.append(f["less_flat_ds"].copy()); full.append(cloud.cpu().numpy().copy())
        torch.cuda.synchronize()
    finally:
        ctx.close()
    return D, surf, full


def _rot_err(qa, qb):
    qa = np.asarray(qa) / np.linalg.norm(qa); qb = np.asarray(qb) / np.linalg.norm(qb)
    d = synth.quat_mul(synth.quat_conj(qa), qb)
    return 2 * np.arcsin(min(1.0, np.linalg.norm(d[1:])))


def _run_device(odo, surf, full, out="host"):
    import torch
    reps = []
    for s, f in zip(surf, full):
        reps.append(odo.step(s, torch.from_numpy(f).cuda(), out=out))
    return reps


@pytest.mark.parametrize("deskew,scan_match_cnt", [(0, 1), (1, 1), (0, 2), (1, 2)])
def test_forced_replay_matches_oracle(oracle, inputs, deskew, scan_match_cnt):
    import torch
    from glio_b200 import api
    from oracle import pyoracle_odom as od
    D, surf, full = inputs
    ctx = api.Context(0)
    try:
        odo = api.Odometry(ctx, deskew=deskew, scan_match_cnt=scan_match_cnt, max_solver_time_s=NO_LIMIT)
        o = od.OdometryOracle(max_num_iter=12, scan_match_cnt=scan_match_cnt, deskew=deskew)
        n_kf = 0
        for k in range(K):
            g = odo.step(surf[k], torch.from_numpy(full[k]).cuda())
            gmap, gscan = odo.clouds()
            r = o.step(surf[k], full[k], forced=[rd["pose"] for rd in g["rounds"]] if g["rounds"] else None)
            assert g["initialised"] == r["initialised"] and g["keyframe"] == r["keyframe"] and g["skipped"] == r["skipped"], k
            assert g["n_map"] == r["n_map"] and g["n_scan"] == r["n_scan"], k
            if k > 0:
                assert np.array_equal(gmap, r["map"]) and np.array_equal(gscan, r["scan"]), k
            assert len(g["rounds"]) == len(r["rounds"]) == (0 if k == 0 else (8 if k == 1 else scan_match_cnt))
            for gr, rr in zip(g["rounds"], r["rounds"]):
                assert gr["n_match"] == rr["n_match"] > 300, k
                # the solve of the round, from identical matches: the oracle's own result before the forced pose replaced it
                assert gr["iterations"] == rr["iterations"] and gr["successful"] == rr["successful"] and gr["termination"] == rr["termination"], k
                assert np.max(np.abs(gr["pose"][:3] - rr["solved_pose"][:3])) <= 1e-6, k
                assert _rot_err(gr["pose"][3:], rr["solved_pose"][3:]) <= 1e-8, k
            assert np.array_equal(g["rel_pose"], r["rel_pose"]) and np.array_equal(g["pose"], r["pose"]), k
            if r["surf"] is None:
                assert g["surf"] is None and g["full"] is None
            else:
                n_kf += 1
                assert np.array_equal(g["surf"], r["surf"]) and np.array_equal(g["full"], r["full"]), k
        assert n_kf >= 8
    finally:
        ctx.close()


def test_free_running_matches_oracle(oracle, inputs):
    from glio_b200 import api
    from oracle import pyoracle_odom as od
    D, surf, full = inputs
    ctx = api.Context(0)
    try:
        odo = api.Odometry(ctx, max_solver_time_s=NO_LIMIT)
        o = od.OdometryOracle()
        for k, g in enumerate(_run_device(odo, surf, full)):
            r = o.step(surf[k], full[k])
            assert g["keyframe"] == r["keyframe"], k
            assert [x["n_match"] for x in g["rounds"]] == [x["n_match"] for x in r["rounds"]], k
            assert np.max(np.abs(g["pose"][:3] - r["pose"][:3])) <= 1e-6 and _rot_err(g["pose"][3:], r["pose"][3:]) <= 1e-8, k
    finally:
        ctx.close()


def test_edge_cases(oracle, inputs):
    import torch
    from glio_b200 import api
    D, surf, full = inputs
    ctx = api.Context(0)
    try:
        # a first sweep only: clouds passed through, identity pose, no rounds
        odo = api.Odometry(ctx)
        g = odo.step(surf[0], full[0])
        assert g["initialised"] and not g["keyframe"] and not g["rounds"]
        assert np.array_equal(g["surf"], surf[0]) and np.array_equal(g["full"], full[0])
        assert np.array_equal(g["pose"], [0, 0, 0, 1, 0, 0, 0]) and np.array_equal(g["rel_pose"], [0, 0, 0, 1, 0, 0, 0])
        # a surf cloud too small for the map: skipped, kf carried over (initially true), the prediction stands
        g = odo.step(surf[1][:5], None)
        assert g["skipped"] and g["keyframe"] and not g["rounds"] and 0 < g["n_map"] < 10
        # an empty scan: every round has no match and keeps the pose; not an argument error
        odo.reset()
        odo.step(surf[0]); odo.step(surf[1])
        g = odo.step(np.zeros((0, 4), np.float32))
        assert g["n_scan"] == 0 and [x["n_match"] for x in g["rounds"]] == [0] and g["rounds"][0]["iterations"] == 0
        assert g["summary"].termination == 0 and b"No non-constant parameter blocks" in g["summary"].message
        odo.close()
        # max_solver_time_s = 0: iteration 0 only, NO_CONVERGENCE, the pose unchanged
        odo = api.Odometry(ctx, max_solver_time_s=0.0)
        odo.step(surf[0])
        g = odo.step(surf[1])
        assert all(x["iterations"] == 1 and x["termination"] == 1 for x in g["rounds"])
        assert np.array_equal(g["pose"], [0, 0, 0, 1, 0, 0, 0]) and b"Maximum solver time" in g["summary"].message
        odo.close()
        # reset() then the same sequence: bit-identical reports; host and device outputs identical
        odo = api.Odometry(ctx, deskew=1, max_solver_time_s=NO_LIMIT)
        a = _run_device(odo, surf[:8], full[:8])
        odo.reset()
        b = _run_device(odo, surf[:8], full[:8], out="device")
        for x, y in zip(a, b):
            assert np.array_equal(x["pose"], y["pose"]) and np.array_equal(x["rel_pose"], y["rel_pose"]) and x["keyframe"] == y["keyframe"]
            assert [r["n_match"] for r in x["rounds"]] == [r["n_match"] for r in y["rounds"]]
            assert (x["surf"] is None) == (y["surf"] is None)
            if x["surf"] is not None:
                assert isinstance(y["surf"], torch.Tensor) and y["surf"].is_cuda
                assert np.array_equal(x["surf"], y["surf"].cpu().numpy()) and np.array_equal(x["full"], y["full"].cpu().numpy())
        odo.close()
    finally:
        ctx.close()


def test_argument_errors_rejected_before_anything_runs(inputs):
    import torch
    from glio_b200 import api
    D, surf, full = inputs
    ctx = api.Context(0)
    L = ctx._lib
    try:
        odo = api.Odometry(ctx)
        odo.step(surf[0])
        rep = api.OdomReport()
        s = np.ascontiguousarray(surf[1]); dsurf = torch.from_numpy(s).cuda()
        n = C.c_int64(len(s))
        before = ctx.launch_count
        bad = [
            # null surf with points
            (None, n, api.HOST, None, C.c_int64(0), api.HOST, None, None, api.HOST),
            # a device surf that is host memory (not memory of the context's GPU)
            (s.ctypes.data_as(C.c_void_p), n, api.DEVICE, None, C.c_int64(0), api.HOST, None, None, api.HOST),
            # a misaligned device surf (4 bytes past a float4 boundary)
            (C.c_void_p(dsurf.data_ptr() + 4), C.c_int64(len(s) - 1), api.DEVICE, None, C.c_int64(0), api.HOST, None, None, api.HOST),
            # a misaligned device output
            (s.ctypes.data_as(C.c_void_p), n, api.HOST, None, C.c_int64(0), api.HOST, C.c_void_p(dsurf.data_ptr() + 4), None, api.DEVICE),
            # a negative count, a bad mem flag
            (s.ctypes.data_as(C.c_void_p), C.c_int64(-1), api.HOST, None, C.c_int64(0), api.HOST, None, None, api.HOST),
            (s.ctypes.data_as(C.c_void_p), n, 7, None, C.c_int64(0), api.HOST, None, None, api.HOST),
        ]
        for args in bad:
            assert L.glio_odom_step(odo._h, *[a if not isinstance(a, int) else C.c_int(a) for a in args], C.byref(rep)) == -3
        assert ctx.launch_count == before
        # nothing changed: the next sweep is the second one (8 rounds)
        g = odo.step(surf[1])
        assert len(g["rounds"]) == 8
        # a NULL odometry handle
        assert L.glio_odom_step(None, None, C.c_int64(0), C.c_int(0), None, C.c_int64(0), C.c_int(0), None, None, C.c_int(0), C.byref(rep)) == -3
        assert L.glio_odom_reset(None) == -3
        bad_opt = api.default_odom_options(scan_match_cnt=9)
        h = C.c_void_p()
        assert L.glio_odom_create(ctx._h, C.byref(bad_opt), C.byref(h)) == -3
    finally:
        ctx.close()


def _window_results(ctx, P):
    from glio_b200 import api
    ctx.set_map(P["map_xyz"])
    ctx.window_set_scans(P["scans"])
    nm = ctx.window_associate(P["poses_init"])
    m = ctx.get_matches(0, len(P["scans"][0]))
    r = ctx.window_solve(P["poses_init"], None, None, api.default_solver_options())
    return nm, m, r


def test_odometry_leaves_the_context_alone(inputs):
    from glio_b200 import api
    D, surf, full = inputs
    P = synth.window_problem(W=3, Q=2000, M=40000, seed=synth.SEED0 + 21)
    ctx = api.Context(0)
    fresh = api.Context(0)
    try:
        a = _window_results(ctx, P)
        odo = api.Odometry(ctx, max_solver_time_s=NO_LIMIT)
        _run_device(odo, surf[:6], full[:6])
        b = _window_results(ctx, P)
        c = _window_results(fresh, P)
        for x in (b, c):
            assert np.array_equal(a[0], x[0])
            assert all(np.array_equal(a[1][k], x[1][k]) for k in ("cp", "nsd", "weight"))
            assert np.array_equal(a[2]["poses"], x[2]["poses"]) and len(a[2]["steps"]) == len(x[2]["steps"])
            assert all(np.array_equal(s, t) for s, t in zip(a[2]["steps"], x[2]["steps"]))
    finally:
        ctx.close(); fresh.close()


def test_keyframe_cloud_hands_off_to_the_window(inputs):
    import torch
    from glio_b200 import api
    D, surf, full = inputs
    ctx = api.Context(0)
    try:
        odo = api.Odometry(ctx, deskew=1, max_solver_time_s=NO_LIMIT)
        odo.step(surf[0], torch.from_numpy(full[0]).cuda(), out="device")
        g = odo.step(surf[1], torch.from_numpy(full[1]).cuda(), out="device")
        assert g["keyframe"] and g["surf"].is_cuda and g["surf"].shape[1] == 4
        ctx.window_set_scan(0, g["surf"])                         # stride-4 GLIO_DEVICE cloud
        ctx.localmap_push(g["surf"], g["pose"][:3], g["pose"][3:])
        assert ctx.localmap_size()[1] == len(g["surf"])
        ctx.set_map(surf[1][:, :3].copy())
        nm = ctx.window_associate(np.array([[0, 0, 0, 1.0, 0, 0, 0]]))
        assert nm[0] > 0
    finally:
        ctx.close()
