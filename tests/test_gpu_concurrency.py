"""Distinct contexts at the same time, the way an Estimator deploys the library: the window solve, the batch solve, the front
end and loop closure each on its own glio_ctx and its own thread, on one GPU and on two.  Every output of every workload must
equal what the same workload gives alone on a fresh context, bit for bit; a thread's refused calls must leave its own message in
glio_last_error; and a call on a context of another GPU must leave the caller's current device where it was.

The workloads are small versions of what the single-context suites already check against their oracles (test_gpu_window_imu_factors,
test_gpu_device_solve, test_gpu_odometry, test_gpu_loop_closure, test_gpu_global_map), so "equal to the serial run" carries those
checks over to concurrent use.  ctypes releases the GIL around every foreign call, so the C calls of different threads overlap;
each workload records the wall-clock intervals of its calls and the tests assert that those of different workloads overlap."""
import ctypes as C
import threading
import time
from concurrent.futures import ThreadPoolExecutor, wait

import numpy as np
import pytest

from glio_b200 import synth
from tests import test_gpu_imu_factors as ti

pytestmark = pytest.mark.gpu

TIMEOUT_S = 900
W = 5                      # window slots
WINDOWS = 3                # windows solved, each followed by its marginalisation and a slide
K_BATCH = 40
SWEEPS = 10
K_LOOP = 30
SUMMARY_FIELDS = ("termination", "num_iterations", "num_successful_steps", "num_unsuccessful_steps", "num_evaluations",
                  "num_jacobian_evaluations", "num_linear_solves", "num_valid_steps", "initial_cost", "final_cost")   # no timings


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _device_count():
    import torch
    return torch.cuda.device_count()


class Clock:
    """the wall-clock intervals of one workload's calls"""

    def __init__(self):
        self.iv = []

    def __call__(self, fn, *a, **kw):
        t0 = time.monotonic()
        try:
            return fn(*a, **kw)
        finally:
            self.iv.append((t0, time.monotonic()))


def _summary(s):
    return np.array([getattr(s, f) for f in SUMMARY_FIELDS], np.float64)


def _iterations(its):
    return np.array([[float(it[k]) for k in sorted(it)] for it in its], np.float64).reshape(len(its), -1)


def _sel(keep):
    """a selection list, or a marker for 'every match active'"""
    return np.array([-1], np.int32) if keep is None else keep


# ---------------------------------------------------------------------------------------------------------------------------
# inputs (numpy only, generated once)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def inputs(api):
    win = synth.window_imu_problem(W=W + WINDOWS - 1, Q=1500, M=30000, seed=71)
    win_edges = synth.window_edge_problem(W=W + WINDOWS - 1, Q=800, M=30000, seed=72)

    bat = synth.imu_problem(K=K_BATCH)
    cur, oth = (np.asarray(v) for v in bat["pairs"])
    keep = np.abs(cur - oth) <= 6              # the device band solve takes half bandwidths up to 160 (104 at a reach of 6)
    bat["pairs"] = (cur[keep].astype(np.int32), oth[keep].astype(np.int32))
    rng = np.random.default_rng(91)
    scene = synth.Scene(-60.0, K_BATCH + 60.0, rng)
    bat["scans"] = [synth.scan_in_body_frame(scene, bat["poses_true"][k], 2500, np.random.default_rng([91, k]), 20.0)
                    for k in range(K_BATCH)]
    dd = synth.dd_psr_problem(K=K_BATCH, seed=synth.SEED0 + 18)            # imu_problem's trajectory

    drive = synth.raw_drive(SWEEPS)
    loop = synth.loop_drive(K=K_LOOP, n_points=1000, dt=2.0, seed=synth.SEED0 + 32)
    return dict(win=win, win_edges=win_edges, bat=bat, dd=dd, drive=drive, loop=loop)


# ---------------------------------------------------------------------------------------------------------------------------
# workloads: each takes a fresh context on `device` and returns a dict of numpy outputs
# ---------------------------------------------------------------------------------------------------------------------------
def wl_window(api, device, inp, clk):
    """three windows of W = 5: association (planes and edges), seeded selection of both, the solve with the IMU chain and a prior,
    the asynchronous marginalisation, and the slide"""
    P, E = inp["win"], inp["win_edges"]
    f_all = api.imu_factor_records(**P["imu"])
    out = {}
    c = clk(api.Context, device)
    try:
        clk(c.set_map, P["map_xyz"]); clk(c.set_edge_map, E["map_xyz"])
        c.window_use_imu_factors(True); c.window_use_edges(True)
        clk(c.window_set_scans, P["scans"][:W])
        for k in range(W):
            clk(c.window_set_edge_scan, k, E["scans"][k])
        hf = ti._host_factor_set(api, P)                # the first window's prior on KF0 fixes the gauge
        poses = P["poses_init"][:W].copy(); sb = P["sb_init"][:W].copy()
        for s in range(WINDOWS):
            out[f"{s}/n_match"] = clk(c.window_associate, poses)
            out[f"{s}/n_edge"] = clk(c.window_associate_edges, poses)
            ids = np.arange(s, s + W)
            out[f"{s}/n_sel"] = clk(c.select_random, ids, nonce=s, feature_res_num=60)
            out[f"{s}/n_sel_edge"] = clk(c.select_random_edges, ids, nonce=s, feature_res_num=30)
            for k in range(W):
                m = clk(c.get_matches, k, 1500)
                for key in ("cp", "nsd", "weight", "src"):
                    out[f"{s}/{k}/match_{key}"] = m[key]
                e = clk(c.get_edges, k)
                for key in ("cp", "pa", "pb", "s", "src"):
                    out[f"{s}/{k}/edge_{key}"] = e[key]
                out[f"{s}/{k}/sel"] = _sel(clk(c.get_selection, k))
                out[f"{s}/{k}/sel_edge"] = _sel(clk(c.get_edge_selection, k))
            f = f_all[s:s + W - 1].copy(); f["i"] -= s; f["j"] -= s
            clk(c.window_set_imu_factors, f)
            r = clk(c.window_solve, poses, sb, hf, band=max(29, hf.marg_half_bandwidth()))
            out[f"{s}/poses"] = r["poses"]; out[f"{s}/speed_bias"] = r["speed_bias"]; out[f"{s}/steps"] = r["steps"]
            out[f"{s}/summary"] = _summary(r["summary"]); out[f"{s}/iterations"] = _iterations(r["iterations"])
            job = clk(c.window_marginalize_async, r["poses"], r["speed_bias"], hf)
            prior = clk(job.wait)
            for key, v in prior.arrays().items():
                out[f"{s}/prior_{key}"] = np.asarray(v)
            hf = api.HostFactorSet(); hf.set_marg_prior(prior)
            clk(c.window_slide, W)
            if s + 1 < WINDOWS:
                clk(c.window_set_scan, W - 1, P["scans"][s + W]); clk(c.window_set_edge_scan, W - 1, E["scans"][s + W])
                poses = np.concatenate([r["poses"][1:], P["poses_init"][s + W:s + W + 1]])
                sb = np.concatenate([r["speed_bias"][1:], P["sb_init"][s + W:s + W + 1]])
    finally:
        c.close()
    return out


def wl_batch(api, device, inp, clk):
    """K = 40: frames and pair association, then pose, DD pseudorange and IMU factors, and the batch solve on the host solver and
    on the device solver (K4)"""
    P, D = inp["bat"], inp["dd"]
    cur, oth = P["pairs"]
    out = {}
    c = clk(api.Context, device)
    try:
        for k in range(K_BATCH):
            clk(c.batch_set_frame, k, P["scans"][k], P["poses_init"][k])
        out["n_match"] = clk(c.batch_associate_pairs, cur, oth)
        for i in range(0, len(cur), 5):
            m = clk(c.batch_get_matches, int(cur[i]), int(oth[i]), 2500)
            for key in ("cp", "weight", "normal_cent", "src"):
                out[f"{i}/{key}"] = m[key]
        clk(c.batch_set_pose_factors, api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
        clk(c.batch_set_dd_psr_factors, api.dd_psr_factor_records(**D["dd"]), api.dd_psr_sat_records(**D["dd_sats"]), D["R"], D["anchor"])
        c.batch_use_dd_psr_factors(True)
        clk(c.batch_set_imu_factors, api.imu_factor_records(**P["imu"])); c.batch_use_imu_factors(True)
        hf = ti._host_factor_set(api, P)
        for name, on in (("host", False), ("device", True)):
            c.batch_use_device_solver(on)
            r = clk(c.batch_solve, P["poses_init"], P["sb_init"], hf, api.batch_solver_options(max_num_iterations=8))
            out[f"{name}/poses"] = r["poses"]; out[f"{name}/speed_bias"] = r["speed_bias"]; out[f"{name}/steps"] = r["steps"]
            out[f"{name}/summary"] = _summary(r["summary"]); out[f"{name}/iterations"] = _iterations(r["iterations"])
    finally:
        c.close()
    return out


def wl_front_end(api, device, inp, clk):
    """ten sweeps of prepare_scan -> extract_features -> odometry step (no wall-clock solver limit: it would make results depend on
    the load)"""
    D = inp["drive"]
    out = {}
    c = clk(api.Context, device)
    odo = None
    try:
        odo = clk(api.Odometry, c, max_solver_time_s=1e9)
        st = api.ImuState()
        for k in range(SWEEPS):
            q = api.imu_sweep_rotation(st, D["stamps"], D["gyro"], D["t_scan_next"][k])
            cloud, ss, se = clk(c.prepare_scan, D["sweeps"][k], 32, q_imu=q)
            f = clk(c.extract_features, cloud, ss, se, 1, 1.0, 0.1, 0.4)
            out[f"{k}/cloud"] = cloud; out[f"{k}/scan_start"] = ss; out[f"{k}/scan_end"] = se
            for key, v in f.items():
                out[f"{k}/{key}"] = v
            g = clk(odo.step, f["less_flat_ds"], cloud)
            out[f"{k}/pose"] = g["pose"]; out[f"{k}/rel_pose"] = g["rel_pose"]
            out[f"{k}/state"] = np.array([g["initialised"], g["keyframe"], g["skipped"], g["n_map"], g["n_scan"]], np.int64)
            out[f"{k}/summary"] = _summary(g["summary"])
            out[f"{k}/rounds"] = np.array([[rd["n_match"], rd["iterations"], rd["successful"], rd["termination"]] for rd in g["rounds"]],
                                          np.int64).reshape(-1, 4)
            out[f"{k}/round_poses"] = np.array([rd["pose"] for rd in g["rounds"]]).reshape(-1, 7)
            for key in ("surf", "full"):
                out[f"{k}/{key}_out"] = np.zeros((0, 4), np.float32) if g[key] is None else g[key]
    finally:
        if odo is not None:
            odo.close()
        c.close()
    return out


def wl_loop(api, device, inp, clk):
    """a loop object along a closed drive of 30 keyframes: keyframes and a loop step after each, then the global map and a VoxelGrid"""
    D = inp["loop"]
    sww = 5
    out = {}
    c = clk(api.Context, device)
    L = None
    try:
        L = clk(api.LoopClosure, c)
        for k in range(K_LOOP):
            clk(L.add_keyframe, D["clouds"][k], D["poses"][k], D["times"][k])
            if k + 1 < sww:
                continue
            j = k + 1 - sww
            g = clk(L.step, D["poses"][j][:3].astype(np.float32), D["times"][j])
            out[f"{k}/report"] = np.array([g["detected"], g["closest_his_idx"], g["latest_frame_idx"], g["accepted"], g["n_latest"],
                                           g["n_latest_ds"], g["n_his"], g["n_his_ds"], g["n_candidates"]], np.int64)
            out[f"{k}/time_last_loop"] = np.array([g["time_last_loop"]])
            if g["icp"] is not None:
                i = g["icp"]
                out[f"{k}/icp"] = np.array([i["converged"], i["state"], i["iterations"], i["n_source"], i["n_target"], i["n_corr"]], np.int64)
                out[f"{k}/icp_final"] = i["final"]; out[f"{k}/icp_fitness"] = np.array([i["fitness"]])
                a, b = clk(L.clouds)
                out[f"{k}/latest"] = a; out[f"{k}/his"] = b
            if g["accepted"]:
                out[f"{k}/pose_from"] = g["pose_from"]; out[f"{k}/pose_to"] = g["pose_to"]; out[f"{k}/noise"] = np.array([g["noise_score"]])
        pts, filtered, n_raw = clk(L.global_map, 3, 0.2)
        out["global_map"] = pts; out["global_map_info"] = np.array([filtered, n_raw], np.int64)
        vox, filtered = clk(c.voxel_filter, np.concatenate(D["clouds"][:10]), 0.4)
        out["voxel"] = vox; out["voxel_filtered"] = np.array([filtered])
    finally:
        if L is not None:
            L.close()
        c.close()
    return out


def _null_ctx_refusals(api):
    """refusals on no context (glio_last_error(NULL) reads them): a device index past the last GPU, and a null IMU state"""
    L = api.lib()
    n = _device_count()
    h = C.c_void_p()
    q = np.zeros(4)
    return [(lambda: L.glio_create(C.c_int(n), None, C.byref(h)), b"device index out of range"),
            (lambda: L.glio_imu_sweep_rotation(None, None, None, C.c_int64(0), C.c_double(0.0), api._ptr(q)),
             b"glio_imu_sweep_rotation: bad arguments")]


def wl_errors(api, device, inp, clk, rounds=1000, flip=False):
    """refused calls that the host decides before any launch, on the thread's own context and on none; after each, the message read
    back must be that call's own"""
    L = api.lib()
    P = inp["win"]
    c = clk(api.Context, device)
    try:
        c.window_set_imu_factors(api.imu_factor_records(**P["imu"]))        # factors up to slot W + WINDOWS - 2
        dummy_poses = np.zeros((3, 7)); dummy_sb = np.zeros((3, 9)); cost = np.zeros(1)
        own = [
            (lambda: L.glio_batch_declare_pairs(c._h, None, None, C.c_int64(3)), b"glio_batch_declare_pairs: null pair arrays"),
            (lambda: L.glio_batch_set_pose_factors(c._h, None, C.c_int64(-1)), b"glio_batch_set_pose_factors: null factor array"),
            (lambda: L.glio_eval_window_imu_factors(c._h, C.c_int(3), api._ptr(dummy_poses), api._ptr(dummy_sb), C.c_int(0), None, None,
                                                    None, api._ptr(cost)),
             b"glio_eval_window_imu_factors: an IMU factor references a slot outside [0, W)"),
            (lambda: L.glio_window_marginalize(c._h, C.c_int(1), None, None, None, None, C.c_double(1e-8), C.byref(C.c_void_p())),
             b"glio_window_marginalize: need W >= 2, poses and speed_bias"),
        ]
        none = _null_ctx_refusals(api)
        if flip:
            own, none = own[::-1], none[::-1]
        n = 0
        for r in range(rounds):
            for call, msg in own:
                rc = clk(call)
                got = L.glio_last_error(c._h)
                assert rc == -3 and got == msg, (rc, got, msg)
                n += 1
            for call, msg in none:
                rc = clk(call)
                got = L.glio_last_error(None)
                assert rc == -3 and got == msg, (rc, got, msg)
                n += 1
    finally:
        c.close()
    return dict(n_refused=np.array([n]))


WORKLOADS = {"window": wl_window, "batch": wl_batch, "front_end": wl_front_end, "loop": wl_loop}


# ---------------------------------------------------------------------------------------------------------------------------
# running and comparing
# ---------------------------------------------------------------------------------------------------------------------------
def _run_serial(api, inp, device, names=tuple(WORKLOADS)):
    return {n: WORKLOADS[n](api, device, inp, Clock()) for n in names}


def _run_threads(api, inp, jobs, stagger=0.0):
    """jobs: (label, workload name, device, kwargs), one thread each, started in list order `stagger` seconds apart.  Returns
    {label: outputs}, {label: intervals}."""
    clocks = {label: Clock() for label, *_ in jobs}
    before = set(threading.enumerate())

    def one(i, label, name, device, kw):
        time.sleep(i * stagger)
        fn = wl_errors if name == "errors" else WORKLOADS[name]
        return fn(api, device, inp, clocks[label], **kw)

    ex = ThreadPoolExecutor(max_workers=len(jobs), thread_name_prefix="glio-concurrency")
    try:
        futs = {label: ex.submit(one, i, label, name, device, kw) for i, (label, name, device, kw) in enumerate(jobs)}
        done, pending = wait(list(futs.values()), timeout=TIMEOUT_S)
        assert not pending, f"{len(pending)} workload(s) still running after {TIMEOUT_S} s"
        out = {label: f.result() for label, f in futs.items()}
    finally:
        ex.shutdown(wait=True)
    assert set(threading.enumerate()) <= before, "a worker thread outlived its test"
    return out, {label: c.iv for label, c in clocks.items()}


def _assert_jobs_equal_baseline(jobs, out, baseline):
    for label, name, device, _ in jobs:
        if name in WORKLOADS:
            _assert_same(out[label], baseline[name], f"{label} on device {device}")


def _assert_same(got, ref, what):
    assert sorted(got) == sorted(ref), f"{what}: different outputs"
    for k in ref:
        a, b = np.ascontiguousarray(got[k]), np.ascontiguousarray(ref[k])
        assert a.dtype == b.dtype and a.shape == b.shape, f"{what} {k}: {a.dtype}{a.shape} != {b.dtype}{b.shape}"
        assert a.tobytes() == b.tobytes(), f"{what} {k}: not bit-identical to the serial run"


def _assert_overlap(intervals, labels):
    """every listed workload has a call that overlaps a call of another workload in time"""
    for a in labels:
        others = [iv for b, ivs in intervals.items() if b != a for iv in ivs]
        assert any(s0 < e1 and s1 < e0 for s0, e0 in intervals[a] for s1, e1 in others), f"{a} ran alone: nothing overlapped it"


@pytest.fixture(scope="module")
def baseline(api, inputs):
    return _run_serial(api, inputs, 0)


# ---------------------------------------------------------------------------------------------------------------------------
# one GPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_serial_baseline_is_reproducible_and_does_work(api, inputs, baseline):
    """each workload alone, twice on fresh contexts: bit-identical, and each does the work it is meant to"""
    again = _run_serial(api, inputs, 0)
    for n in WORKLOADS:
        _assert_same(again[n], baseline[n], n)
    b = baseline
    for s in range(WINDOWS):
        assert b["window"][f"{s}/n_match"].min() > 100 and b["window"][f"{s}/n_edge"].sum() > 0
        assert b["window"][f"{s}/n_sel"].min() > 0 and b["window"][f"{s}/n_sel_edge"].sum() > 0
        assert b["window"][f"{s}/summary"][1] >= 1 and b["window"][f"{s}/prior_lin_jac"].any()
    assert b["batch"]["n_match"].sum() > 1000
    for name in ("host", "device"):
        assert b["batch"][f"{name}/summary"][1] >= 1
    assert b["front_end"]["0/state"][0] == 1 and sum(len(b["front_end"][f"{k}/rounds"]) for k in range(SWEEPS)) >= SWEEPS - 1
    assert any(k.endswith("/icp") for k in b["loop"]), "the drive is supposed to reach a loop candidate"
    assert len(b["loop"]["global_map"]) > 0 and len(b["loop"]["voxel"]) > 0


def _concurrent_jobs(order):
    jobs = [("window", "window", 0, {}), ("batch", "batch", 0, {}), ("front_end", "front_end", 0, {}), ("loop", "loop", 0, {}),
            ("window2", "window", 0, {}), ("batch2", "batch", 0, {})]
    return [jobs[i] for i in order]


@pytest.mark.parametrize("order,stagger", [((0, 1, 2, 3, 4, 5), 0.0), ((5, 3, 1, 4, 2, 0), 0.05)])
def test_concurrent_contexts_on_one_gpu_equal_the_serial_runs(api, inputs, baseline, order, stagger):
    """every workload on its own context and thread at once, two of them twice: every output equals the serial run bit for bit"""
    jobs = _concurrent_jobs(order)
    out, iv = _run_threads(api, inputs, jobs, stagger)
    _assert_jobs_equal_baseline(jobs, out, baseline)
    _assert_overlap(iv, list(out))


def test_refusals_alongside_work_keep_their_own_messages(api, inputs, baseline):
    """two threads of refused calls (in opposite orders, so their messages differ at every moment) next to the four workloads: each
    reads its own message back after every call, and the workloads still equal the serial runs"""
    jobs = _concurrent_jobs(range(4)) + [("errors", "errors", 0, {}), ("errors_flipped", "errors", 0, dict(flip=True))]
    out, iv = _run_threads(api, inputs, jobs)
    _assert_jobs_equal_baseline(jobs, out, baseline)
    assert out["errors"]["n_refused"][0] == out["errors_flipped"]["n_refused"][0] == 1000 * 6
    _assert_overlap(iv, list(out))


def test_refused_create_reports_on_the_calling_thread(api):
    """glio_create on a device past the last one: refused, the message is the calling thread's, the Python error carries it"""
    for call, msg in _null_ctx_refusals(api):
        assert call() == -3 and api.lib().glio_last_error(None) == msg
    with pytest.raises(api.GlioError, match="device index out of range"):
        api.Context(_device_count())


# ---------------------------------------------------------------------------------------------------------------------------
# two GPUs
# ---------------------------------------------------------------------------------------------------------------------------
two_gpus = pytest.mark.skipif("__import__('torch').cuda.device_count() < 2", reason="needs two GPUs")


@two_gpus
def test_second_gpu_equals_the_first(api, inputs, baseline):
    """every workload on device 1 after device 0 has run it in this process (so a setting made once per process, not once per
    device, would be missing on device 1): bit for bit device 0's outputs"""
    assert baseline is not None                                  # device 0 first
    second = _run_serial(api, inputs, 1)
    for n in WORKLOADS:
        _assert_same(second[n], baseline[n], f"{n} on device 1")


@two_gpus
def test_two_gpus_at_once(api, inputs, baseline):
    jobs = [(f"{n}@{d}", n, d, {}) for n in WORKLOADS for d in (0, 1)]
    out, iv = _run_threads(api, inputs, jobs)
    _assert_jobs_equal_baseline(jobs, out, baseline)
    _assert_overlap(iv, list(out))


@two_gpus
@pytest.mark.parametrize("torch_dev,ctx_dev", [(0, 1), (1, 0)])
def test_calls_leave_the_current_device_alone(api, inputs, torch_dev, ctx_dev):
    """entry points on a context of the other GPU, a refused one included, return with the caller's current device unchanged"""
    import torch
    P, D = inputs["win"], inputs["drive"]

    def here():
        assert torch.cuda.current_device() == torch_dev
        assert torch.empty(1, device="cuda").device.index == torch_dev

    with torch.cuda.device(torch_dev):
        c = api.Context(ctx_dev); here()
        try:
            c.set_map(P["map_xyz"]); here()
            c.window_set_scans(P["scans"][:W]); here()
            c.window_associate(P["poses_init"][:W]); here()
            assert api.lib().glio_batch_declare_pairs(c._h, None, None, C.c_int64(3)) == -3; here()
            cloud, ss, se = c.prepare_scan(D["sweeps"][0], 32); here()
            c.extract_features(cloud, ss, se, 1, 1.0, 0.1, 0.4); here()
            o = api.Odometry(c); here()
            o.close(); here()
            lp = api.LoopClosure(c); here()
            lp.close(); here()
            o = api.Odometry(c); lp = api.LoopClosure(c)           # left attached: glio_destroy frees them
        finally:
            c.close()
        here()
