"""Ceres-API shim route for the batch refinement's pose factors (K2p: LidarPoseFactorBatchRelativeAutoDiff, delta_q_factor_auto),
driven by tests/cpp/shim_pose_routes_test.cpp: problems built with optimizeBatchWithLandMark's call sequence give the same iterates
host-only and device-routed and through glio_batch_solve, blocks K2p cannot evaluate exactly stay on the host, and problems without
pose blocks launch no K2p kernel."""
import ctypes as C
import struct

import numpy as np
import pytest

from glio_b200 import synth
from tests import eval_reference as er
from tests import pose_factor_reference as pr
from tests import shim_common as sc

REL, DQ, LOOKALIKE = 0, 1, 2                      # the driver's pose record kinds (2: LidarPoseFactorAutoDiff, no trait)
YAW, ANCHOR = 0.3, np.array([12.0, -7.0, 3.0])    # the constant yaw offset and anchor of the level-0 problems
PAIR_DTYPE = np.dtype([("kind", "<i4"), ("i", "<i4"), ("j", "<i4"), ("alt", "<i4"), ("dq", "<f8", (4,)), ("dp", "<f8", (3,)),
                       ("loss", "<f8")])
BIN_DTYPE = np.dtype([("kc", "<i4"), ("ko", "<i4"), ("cp", "<f8", (3,)), ("nc", "<f8", (6,)), ("score", "<f8")])
DD_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("s1", "<f8", (3,)), ("s2", "<f8", (3,)), ("rho_i", "<f8"), ("rho_j", "<f8"),
                     ("w", "<f8")])


def pose_records(i, j, kind, dq, dp=None, alt=None, loss=-1.0):
    n = len(i)
    r = np.zeros(n, PAIR_DTYPE)
    r["i"], r["j"], r["kind"] = i, j, kind
    r["dq"] = np.asarray(dq, np.float64).reshape(n, 4)
    if dp is not None:
        r["dp"] = np.asarray(dp, np.float64).reshape(n, 3)
    r["alt"] = -1 if alt is None else alt
    r["loss"] = loss
    return r


def write_problem(path, poses, pose, sb=None, n_rcv=0, epoch=0, t_param=None, q_const=None, q_ident=None, alt_t=None, binary=None,
                  priors=(), betweens=(), dds=None, max_iter=10, time_limit=1e9):
    poses = np.asarray(poses, np.float64).reshape(-1, 7); K = len(poses)
    z = lambda a: np.asarray(a if a is not None else np.zeros(K), np.int32).tobytes()
    alt_t = np.zeros((0, 3)) if alt_t is None else np.asarray(alt_t, np.float64).reshape(-1, 3)
    binary = np.zeros(0, BIN_DTYPE) if binary is None else binary
    dds = np.zeros(0, DD_DTYPE) if dds is None else dds
    with open(path, "wb") as f:
        f.write(struct.pack("<iii", K, n_rcv, epoch))
        f.write(poses.tobytes()); f.write(np.ascontiguousarray(sb if sb is not None else np.zeros((K, 9)), np.float64).tobytes())
        f.write(struct.pack("<d", YAW)); f.write(ANCHOR.tobytes())
        f.write(z(t_param)); f.write(z(q_const)); f.write(z(q_ident))
        f.write(struct.pack("<i", len(pose))); f.write(np.ascontiguousarray(pose, PAIR_DTYPE).tobytes())
        f.write(struct.pack("<i", len(alt_t))); f.write(alt_t.tobytes())
        f.write(struct.pack("<i", len(binary))); f.write(np.ascontiguousarray(binary, BIN_DTYPE).tobytes())
        f.write(struct.pack("<i", len(priors)))
        for (k, t0, q0, sb0, sw) in priors:
            f.write(struct.pack("<i", k)); f.write(np.asarray(t0, np.float64).tobytes()); f.write(np.asarray(q0, np.float64).tobytes())
            f.write(np.asarray(sb0 if sb0 is not None else np.zeros(9), np.float64).tobytes()); f.write(np.asarray(sw, np.float64).tobytes())
        f.write(struct.pack("<i", len(betweens)))
        for (i, j, dp, dq, dv, dt, sw) in betweens:
            f.write(struct.pack("<ii", i, j)); f.write(np.asarray(dp, np.float64).tobytes()); f.write(np.asarray(dq, np.float64).tobytes())
            f.write(np.asarray(dv, np.float64).tobytes()); f.write(struct.pack("<d", dt)); f.write(np.asarray(sw, np.float64).tobytes())
        f.write(struct.pack("<i", len(dds))); f.write(np.ascontiguousarray(dds, DD_DTYPE).tobytes())
        f.write(struct.pack("<id", max_iter, time_limit))


# ---------------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------------
def _rz(yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def dd_records(T, seed, per_pair=None, w=2.0, noise=0.3):
    """pseudorange-like stand-ins between consecutive keyframes (dd_psr_factor_20's blocks t_i, t_j, yaw, anchor): range
    differences to two satellites 20 km away, measured at the true positions plus noise; at least 12 per keyframe pair on short
    trajectories.  The positions are over-determined and the noise pulls against the pose factors, so the optimum keeps a cost
    with pose-factor residuals in it"""
    rng = np.random.default_rng(seed)
    K = len(T)
    per_pair = per_pair or max(3, 12 // max(K - 1, 1))
    rec = np.zeros(max(K - 1, 1) * per_pair, DD_DTYPE)
    n = 0
    for k in range(max(K - 1, 1)):
        j = k + 1 if K > 1 else k
        for _ in range(per_pair):
            s = rng.normal(size=(2, 3)); s[:, 2] = np.abs(s[:, 2]) + 0.5
            s = 2.0e4 * s / np.linalg.norm(s, axis=1)[:, None]
            a, b = ANCHOR + _rz(YAW) @ s[0], ANCHOR + _rz(YAW) @ s[1]
            rd = lambda t: np.linalg.norm(t - a) - np.linalg.norm(t - b)
            rec[n] = (k, j, s[0], s[1], rd(T[k, :3]) + rng.normal(0, noise), rd(T[j, :3]) + rng.normal(0, noise), w)
            n += 1
    return rec


def pose_list(P):
    return pose_records(P["i"], P["j"], np.where(P["kind"] == 1, DQ, REL), P["dq"], P["dp"])


def curved_pose_graph(K, seed, search_range=6):
    """synth.pose_graph_problem's level-0 construction (synth.attitude_factors, synth.relative_pose_factors) on a trajectory that
    also curves in y and z.  Without IMU factors the roll about a straight path's direction of travel is barely observable, and a
    near-null direction of the normal equations carries rounding-level differences between evaluation orders into the iterates."""
    rng = np.random.default_rng(seed)
    truth = synth.trajectory(K, rng)
    k = np.arange(K)
    truth[:, 1] += 2.0 * np.sin(0.9 * k); truth[:, 2] += 1.5 * np.cos(0.6 * k)
    kf = synth.perturb(truth, rng, sig_t=0.01, sig_r_deg=0.05)
    init = synth.perturb(truth, rng, sig_t=0.03, sig_r_deg=0.2)
    ai, aj, adq = synth.attitude_factors(kf, search_range)
    ri, rj, rdq, rdp = synth.relative_pose_factors(kf, search_range)
    return dict(K=K, poses_true=truth, kf=kf, poses_init=init, i=np.concatenate([ai, ri]), j=np.concatenate([aj, rj]),
                kind=np.concatenate([np.ones(len(ai), np.int32), np.zeros(len(ri), np.int32)]),
                dq=np.concatenate([adq, rdq]), dp=np.concatenate([np.zeros((len(ai), 3)), rdp]))


def level0(K, seed=synth.SEED0 + 16):
    """the shipped sms_fusion_level 0 problem: attitude then relative factors, speed-bias / receiver-clock blocks added and
    unused, constant yaw and anchor, pseudorange stand-ins"""
    P = curved_pose_graph(K, seed)
    return dict(P=P, poses=P["poses_init"], pose=pose_list(P), kw=dict(n_rcv=4, epoch=8, dds=dd_records(P["poses_true"], seed)))


def imu_chain(T, sb):
    rng = np.random.default_rng(7)
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)])
    priors = [(0, T[0, :3], T[0, 3:], np.zeros(9), sw * 3)]
    betweens = []
    for i in range(len(T) - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        betweens.append((i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw))
    return priors, betweens


def binary_records(P, n=20, seed=3, batch_score=2.5):
    rng = np.random.default_rng(seed)
    cur, oth = P["pairs"]
    out = []
    for a, b in zip(cur, oth):
        m = er.make_pair(rng, P["poses_true"][a], P["poses_true"][b], n, noise=0.02)
        r = np.zeros(n, BIN_DTYPE)
        r["kc"], r["ko"], r["cp"], r["nc"] = a, b, m["cp"].astype(np.float64), m["nc"]
        r["score"] = batch_score * m["weight"].astype(np.float64)
        out.append(r)
    return np.concatenate(out) if out else np.zeros(0, BIN_DTYPE)


def level1(K, seed=synth.SEED0 + 16, attitude=True):
    """sms_fusion_level 1: attitude factors, BinaryLidarPlaneNormFactor blocks of the batch pairs, an IMU-like host chain"""
    P = synth.pose_graph_problem(K=K, seed=seed, level=1)
    sb = np.zeros((K, 9))
    priors, betweens = imu_chain(P["poses_true"], sb)
    pose = pose_list(P) if attitude else np.zeros(0, PAIR_DTYPE)
    return dict(P=P, poses=P["poses_init"], pose=pose, kw=dict(sb=sb, binary=binary_records(P), priors=priors, betweens=betweens))


def write_case(path, c, **kw):
    args = dict(c["kw"]); args.update(kw)
    write_problem(path, c["poses"], c["pose"], **args)


def routable(pose, K, t_param=None, q_const=None, q_ident=None, binary=None):
    """the shim's routing rule, restated: every block active, q quaternion-parameterized, t plain, no loss, a trait, and each q of a
    single (t, q) keyframe pairing"""
    t_param = np.zeros(K, bool) if t_param is None else np.asarray(t_param, bool)
    q_bad = (np.zeros(K, bool) if q_const is None else np.asarray(q_const, bool)) | (np.zeros(K, bool) if q_ident is None else np.asarray(q_ident, bool))
    cand = []
    for r in pose:
        ok = r["kind"] in (REL, DQ) and r["loss"] < 0 and not q_bad[r["i"]] and not q_bad[r["j"]]
        if r["kind"] == REL:
            ok = ok and not t_param[r["j"]] and (r["alt"] >= 0 or not t_param[r["i"]])
        cand.append(ok)
    ts_of_q = {}
    for r, ok in zip(pose, cand):
        if ok and r["kind"] == REL:
            ts_of_q.setdefault(int(r["i"]), set()).add(("alt", int(r["alt"])) if r["alt"] >= 0 else ("t", int(r["i"])))
            ts_of_q.setdefault(int(r["j"]), set()).add(("t", int(r["j"])))
    if binary is not None:
        for r in binary:
            for k in (int(r["kc"]), int(r["ko"])):
                ts_of_q.setdefault(k, set()).add(("t", k))
    return sum(1 for r, ok in zip(pose, cand) if ok and r["i"] != r["j"] and len(ts_of_q.get(int(r["i"]), ())) <= 1 and len(ts_of_q.get(int(r["j"]), ())) <= 1)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
POSES = {"near": dict(offset=0.0), "3km": dict(offset=3000.0), "20km": dict(offset=20000.0), "q_nonunit": dict(qnorm=[0.5, 2.0, 1.3, 0.8])}


@pytest.mark.parametrize("fx", list(POSES))
def test_host_evaluate_pose_functors(tmp_path, fx):
    """Problem::Evaluate of a pose-only problem (host Jets) against the longdouble reference of both functors: pins the restated
    functors and their block order"""
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    rng = np.random.default_rng(11)
    K = 9
    kw = dict(POSES[fx])
    if "qnorm" in kw:
        kw["qnorm"] = np.resize(kw["qnorm"], K)
    poses = er.make_poses(K, rng, spread=3.0, **kw)
    n = 40
    i = rng.integers(0, K, n); j = (i + rng.integers(1, 4, n) * rng.choice([-1, 1], n)) % K
    dq = rng.normal(size=(n, 4)); dq[:, 0] += 4.0; dq /= np.linalg.norm(dq, axis=1)[:, None]
    kind = rng.choice([REL, DQ], n)
    dp = rng.normal(0, 1.5, (n, 3))
    write_problem(tmp_path / "p.bin", poses, pose_records(i, j, kind, dq, dp))
    r = sc.run_driver(exe, "evaluate", [tmp_path / "p.bin"])[0]
    from glio_b200 import api
    f = api.pose_factor_records(i, j, np.where(kind == REL, api.POSE_RELATIVE, api.POSE_DELTA_Q), dq, np.where((kind == REL)[:, None], dp, 0.0))
    ref = pr.pose_blocks(poses, f)
    er.assert_within(r["eval_cost"], ref["cost"], ref["Mcost"], "cost")
    g = r["gradient"][:15 * K].reshape(K, 15)                     # per keyframe t, q (tangent), speed-bias; then yaw and anchor
    er.assert_within(g[:, :6], ref["g"], ref["Mg"], "gradient")
    assert np.all(g[:, 6:] == 0) and np.all(r["gradient"][15 * K:] == 0)
    assert ref["cost"] > 0


def test_trait_descriptions_are_the_constructor_arguments(tmp_path):
    """both traits return dq / dp bit for bit (values that are not floats, signed zeros, a subnormal, a non-unit dq), the private
    members of LidarPoseFactorBatchRelativeAutoDiff read through the explicit-instantiation idiom; the look-alike has no trait"""
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    rng = np.random.default_rng(4)
    n = 12
    dq = rng.normal(size=(n, 4)) * 0.7; dp = rng.normal(0, 1e3, (n, 3))
    dq[0] = [-0.0, 0.0, 5e-324, 1.0 + 2.0 ** -52]; dp[1] = [-0.0, 1e-300, np.pi * 1e7]
    kind = np.array([REL, DQ] * (n // 2))
    kind[-1] = LOOKALIKE
    write_problem(tmp_path / "d.bin", er.make_poses(2, rng), pose_records(np.zeros(n, int), np.ones(n, int), kind, dq, dp))
    desc = sc.run_driver(exe, "describe", [tmp_path / "d.bin"], desc_ints=2)[0]["desc"]
    assert len(desc) == n
    for k, (ok, fk, v) in enumerate(desc):
        if kind[k] == LOOKALIKE:
            assert ok == 0 and fk == 0
            continue
        assert ok == 1 and fk == (5 if kind[k] == REL else 6)
        got_q, got_p = np.array(v[:4]), np.array(v[4:])
        assert got_q.tobytes() == dq[k].tobytes()
        assert got_p.tobytes() == (dp[k] if kind[k] == REL else np.zeros(3)).tobytes()


def test_host_solve_level0(tmp_path):
    """the level-0 problem solved on the host only (no context): no device block, and the solve removes almost all of the
    attitude factors' initial cost (the initial rotations are 0.2 degrees off, the factors' keyframe poses 0.05 degrees)"""
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    c = level0(30)
    write_case(tmp_path / "h.bin", c)
    r = sc.run_driver(exe, "host", [tmp_path / "h.bin"])[0]
    assert r["device_blocks"] == 0 and r["device_pose"] == 0 and r["pose_launches"] == 0
    assert r["cost"][1] < 1e-3 * r["cost"][0]


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("level,K", [(0, 2), (0, 7), (0, 40), (0, 200), (1, 13), (1, 40), (1, 200)])
def test_device_matches_host(tmp_path, level, K):
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    c = level0(K) if level == 0 else level1(K)
    path = tmp_path / "p.bin"
    write_case(path, c)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    n_pose = len(c["pose"])
    nb = len(c["kw"].get("binary", ()))
    assert n_pose > 0 and host["device_blocks"] == 0
    assert dev["device_pose"] == n_pose and dev["device_blocks"] == n_pose + nb
    assert dev["pose_launches"] >= dev["n_iters"]                 # K2p runs in every evaluation
    sc.assert_same_solve(dev, host, sb=False, iterate_abs=1e-10)


def _dd_band_callback(api, ctx, hf, dds, nt):
    """host factors for glio_batch_solve: hf (may be None) plus the pseudorange stand-ins, each of whose two rows touches one t"""
    L = ctx._lib
    a = ANCHOR[None, :] + dds["s1"] @ _rz(YAW).T; b = ANCHOR[None, :] + dds["s2"] @ _rz(YAW).T

    def cb(user, K, p, s, want_jac, H, hb, g, cost):
        if hf is not None:
            rc = L.glio_hf_evaluate_band(hf._h, K, p, s, want_jac, H, hb, g, cost)
            if rc != 0:
                return rc
        else:
            cost[0] = 0.0
        P = np.ctypeslib.as_array(p, (K * 7,)).reshape(K, 7)
        band = np.ctypeslib.as_array(H, (K * nt * (hb + 1),)).reshape(K * nt, hb + 1) if want_jac else None
        gv = np.ctypeslib.as_array(g, (K * nt,)) if want_jac else None
        ct = 0.0
        for n, d in enumerate(dds):
            for k, rho in ((int(d["i"]), d["rho_i"]), (int(d["j"]), d["rho_j"])):
                t = P[k, :3]
                ua, ub = t - a[n], t - b[n]
                la, lb = np.linalg.norm(ua), np.linalg.norm(ub)
                r = d["w"] * (la - lb - rho)
                ct += 0.5 * r * r
                if want_jac:
                    J = d["w"] * (ua / la - ub / lb)
                    for x in range(3):
                        gv[nt * k + x] += J[x] * r
                        for y in range(x + 1):
                            band[nt * k + x, y - x + hb] += J[x] * J[y]
        cost[0] = cost[0] + ct
        return 0
    return api.HOST_FACTORS_BAND_FN(cb)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [0, 1])
def test_device_matches_glio_batch_solve(tmp_path, level):
    """the device-routed solve against glio_batch_solve with glio_batch_use_pose_factors(1), the same pose list and LiDAR pairs,
    and the host stand-ins passed through the band callback"""
    from glio_b200 import api
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    K = 40
    c = level0(K) if level == 0 else level1(K)
    max_iter = 8
    path = tmp_path / "p.bin"
    write_case(path, c, max_iter=max_iter)
    dev = sc.run_driver(exe, "device", [path])[0]
    P = c["P"]
    ctx = api.Context(0)
    hf = None
    try:
        if level == 1:
            B = c["kw"]["binary"]
            cur, oth = P["pairs"]
            ctx.batch_declare_pairs(cur, oth)
            for a, b in zip(cur, oth):
                m = (B["kc"] == a) & (B["ko"] == b)
                ctx.batch_set_pair_matches(int(a), int(b), B["cp"][m].astype(np.float32), B["nc"][m], (B["score"][m] / 2.5).astype(np.float32))
            hf = api.HostFactorSet()
            for a in c["kw"]["priors"]: hf.add_prior(*a)
            for a in c["kw"]["betweens"]: hf.add_between(*a)
        ctx.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"]))
        ctx.batch_use_pose_factors(True)
        sb = c["kw"].get("sb")
        nt = 15 if sb is not None else 6
        dds = c["kw"].get("dds", np.zeros(0, DD_DTYPE))
        fn = _dd_band_callback(api, ctx, hf, dds, nt)
        pb = np.array(c["poses"], np.float64).copy(); sbv = None if sb is None else np.array(sb, np.float64).copy()
        opt = api.batch_solver_options(max_num_iterations=max_iter)
        summ = api.SolverSummary(); log = (api.Iteration * 64)()
        ctx._chk(ctx._lib.glio_batch_solve(ctx._h, C.c_int(K), api._ptr(pb), api._ptr(sbv), fn, None, C.byref(opt), C.byref(summ), log,
                                           C.c_int(64), None, C.c_int64(0)))
        its = api.iterations_to_dicts(log, min(summ.num_iterations, 64))
    finally:
        ctx.close()
    bs = dict(termination=int(summ.termination), n_iters=summ.num_iterations, cost=(summ.initial_cost, summ.final_cost), poses=pb,
              iters=[(i["iteration"], int(i["step_is_successful"]), i["cost"], i["trust_region_radius"]) for i in its])
    assert dev["device_pose"] == len(c["pose"])
    sc.assert_same_solve(dev, bs, sb=False, iterate_abs=1e-10)


@pytest.mark.gpu
def test_blocks_that_stay_on_the_host(tmp_path):
    """pose blocks K2p cannot evaluate exactly stay on the host: the device count is exactly the routable one and the solve agrees
    with the host-only one"""
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    K = 30
    c = level0(K)
    base = c["pose"]
    rng = np.random.default_rng(8)
    take = base[base["kind"] == REL][:6].copy()
    loss = take[:2].copy(); loss["loss"] = 0.5                                       # a loss
    look = take[2:4].copy(); look["kind"] = LOOKALIKE                                # LidarPoseFactorAutoDiff (0.2 weights, no trait)
    conflict = take[4:5].copy(); conflict["i"] = 20; conflict["j"] = 21; conflict["alt"] = 0   # q_20 paired with t_20 and another t
    pose = np.concatenate([base, loss, look, conflict])
    t_param = np.zeros(K, int); q_const = np.zeros(K, int); q_ident = np.zeros(K, int)
    q_const[5] = 1                                                                   # a constant q
    q_ident[11] = 1                                                                  # a q without QuaternionParameterization
    t_param[16] = 1                                                                  # a t with a local parameterization
    alt_t = c["poses"][20:21, :3] + rng.normal(0, 0.01, 3)
    expect = routable(pose, K, t_param, q_const, q_ident)
    assert 0 < expect < len(pose) - 40
    path = tmp_path / "m.bin"
    write_problem(path, c["poses"], pose, t_param=t_param, q_const=q_const, q_ident=q_ident, alt_t=alt_t, **c["kw"])
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    assert host["device_blocks"] == 0
    assert dev["device_pose"] == dev["device_blocks"] == expect
    sc.assert_same_solve(dev, host, sb=False, iterate_abs=1e-10)
    assert np.array_equal(dev["poses"][5, 3:], c["poses"][5, 3:])                  # the constant q stayed put

    # delta_q-only keyframes: the attitude factors alone, the positions held by the stand-ins and a prior; K2p adds rotation
    # columns only, every t row and column comes from the host blocks
    c1 = level1(K)
    P = c1["P"]
    priors, _ = imu_chain(P["poses_true"], None)
    path = tmp_path / "dq.bin"
    write_problem(path, c1["poses"], c1["pose"], sb=np.zeros((K, 9)), priors=priors, dds=dd_records(P["poses_true"], 5))
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    assert dev["device_pose"] == dev["device_blocks"] == len(c1["pose"]) == routable(c1["pose"], K)
    sc.assert_same_solve(dev, host, sb=False, iterate_abs=1e-10)


@pytest.mark.gpu
def test_pose_pair_counts_around_the_kernel_block(tmp_path):
    """chains with exactly 1, 7, 8, 9, 16 and 17 distinct pose pairs (K2p gives 8 pairs to a block), relative and delta_q factors
    on each pair, solved in turn on one context and on the host"""
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    paths = []
    for n_pairs in (1, 7, 8, 9, 16, 17):
        c = level0(n_pairs + 1, seed=synth.SEED0 + 40 + n_pairs)
        p = c["pose"]
        p = p[np.abs(p["i"] - p["j"]) == 1]                                          # neighbours only: exactly K - 1 pairs
        assert len({(min(a, b), max(a, b)) for a, b in zip(p["i"], p["j"])}) == n_pairs
        path = tmp_path / f"c{n_pairs}.bin"
        write_problem(path, c["poses"], p, **c["kw"])
        paths.append((path, len(p)))
    dev = sc.run_driver(exe, "device", [p for p, _ in paths])
    host = sc.run_driver(exe, "host", [p for p, _ in paths])
    for d, h, (_, n) in zip(dev, host, paths):
        assert d["device_pose"] == n
        sc.assert_same_solve(d, h, sb=False, iterate_abs=1e-10)


@pytest.mark.gpu
def test_solve_sequences_on_one_context(tmp_path):
    """pose problem -> binary-only problem -> pose problem on one context print the same text (%.17g) as fresh contexts, also with
    glio_batch_use_pose_factors(1) set and after a direct caller left another pose list with the switch on; the binary-only
    problem launches no K2p kernel"""
    exe = sc.build_driver(tmp_path, "shim_pose_routes_test")
    paths = [tmp_path / f"s{i}.bin" for i in range(4)]
    write_case(paths[0], level0(40))
    write_case(paths[1], level1(30, attitude=False))
    write_case(paths[2], level1(30))
    write_case(paths[3], level0(25, seed=synth.SEED0 + 17))
    fresh = [sc.run_driver(exe, "device", [p])[0] for p in paths]
    assert [f["pose_launches"] > 0 for f in fresh] == [True, False, True, True]
    assert fresh[1]["device_pose"] == 0 and fresh[1]["device_blocks"] > 0
    for flags in ((), ("--use-pose",), ("--preload-pose", "40")):
        seq = sc.run_driver(exe, "device", paths, *flags)
        assert len(seq) == 4
        for a, b in zip(seq, fresh):
            assert a["text"] == b["text"]
