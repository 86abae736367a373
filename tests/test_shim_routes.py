"""Ceres-API shim routes for LidarEdgeFactor (K2e) and LidarPlaneNormIncreFactor (K2 in a front-end context), driven by
tests/cpp/shim_routes_test.cpp: problems built with the reference's call sequences give the same iterates host-only and
device-routed, blocks the kernels cannot evaluate exactly stay on the host, and plane-only problems launch no edge kernel."""
import struct

import numpy as np
import pytest

from glio_b200 import synth
from tests import eval_reference as er
from tests import shim_common as sc

PLANE, BINARY, EDGE, INCRE = 1, 2, 3, 4          # glio::FactorKind
IDENT_Q, ZERO_T = np.array([1.0, 0.0, 0.0, 0.0]), np.zeros(3)
LIDAR_CONST, HUBER = 7.5, 1.0


def lidar_records(kind, kf, cp, a=None, b=None, d=None, s=None, q_lb=IDENT_Q, t_lb=ZERO_T, loss=-1.0, kf2=None):
    """(n,) records of the driver's LiDAR section; every per-block value may be a scalar or an (n, ...) array."""
    n = len(cp)
    rec = np.zeros(n, dtype=[("kind", "<i4"), ("kf", "<i4"), ("kf2", "<i4"), ("v", "<f8", (19,))])
    rec["kind"] = kind; rec["kf"] = kf; rec["kf2"] = -1 if kf2 is None else kf2
    v = rec["v"]
    v[:, 0:3] = np.asarray(cp, np.float64)
    if a is not None: v[:, 3:6] = np.asarray(a, np.float64)
    if b is not None: v[:, 6:9] = np.asarray(b, np.float64)
    if d is not None: v[:, 9] = np.asarray(d, np.float64)
    if s is not None: v[:, 10] = np.asarray(s, np.float64)
    v[:, 11:15] = np.asarray(q_lb, np.float64); v[:, 15:18] = np.asarray(t_lb, np.float64); v[:, 18] = loss
    return rec


def write_problem(path, poses, lidar, ctx, sb=None, priors=(), betweens=(), ranges=(), t_param=None, q_const=None, strategy=0,
                  max_iter=15, time_limit=1e9):
    """ctx: dict(q_lb, t_lb, lidar_const, huber, unit_score) -- the device context's parameters"""
    poses = np.asarray(poses, np.float64).reshape(-1, 7); W = len(poses)
    lidar = np.concatenate(lidar) if isinstance(lidar, (list, tuple)) else lidar
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", W, 1 if sb is not None else 0))
        f.write(poses.tobytes()); f.write(np.ascontiguousarray(sb if sb is not None else np.zeros((W, 9)), np.float64).tobytes())
        f.write(np.asarray(ctx["q_lb"], np.float64).tobytes()); f.write(np.asarray(ctx["t_lb"], np.float64).tobytes())
        f.write(struct.pack("<ddi", ctx["lidar_const"], ctx["huber"], ctx["unit_score"]))
        f.write(np.asarray(t_param if t_param is not None else np.zeros(W), np.int32).tobytes())
        f.write(np.asarray(q_const if q_const is not None else np.zeros(W), np.int32).tobytes())
        f.write(struct.pack("<i", len(lidar))); f.write(lidar.tobytes())
        f.write(struct.pack("<i", len(priors)))
        for (k, t0, q0, sb0, sw) in priors:
            f.write(struct.pack("<i", k)); f.write(np.asarray(t0, np.float64).tobytes()); f.write(np.asarray(q0, np.float64).tobytes())
            f.write(np.asarray(sb0 if sb0 is not None else np.zeros(9), np.float64).tobytes()); f.write(np.asarray(sw, np.float64).tobytes())
        f.write(struct.pack("<i", len(betweens)))
        for (i, j, dp, dq, dv, dt, sw) in betweens:
            f.write(struct.pack("<ii", i, j)); f.write(np.asarray(dp, np.float64).tobytes()); f.write(np.asarray(dq, np.float64).tobytes())
            f.write(np.asarray(dv, np.float64).tobytes()); f.write(struct.pack("<d", dt)); f.write(np.asarray(sw, np.float64).tobytes())
        f.write(struct.pack("<i", len(ranges)))
        for (k, lever, sat, rho, w_) in ranges:
            f.write(struct.pack("<i", k)); f.write(np.asarray(lever, np.float64).tobytes()); f.write(np.asarray(sat, np.float64).tobytes())
            f.write(struct.pack("<dd", rho, w_))
        f.write(struct.pack("<iid", strategy, max_iter, time_limit))


# ---------------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------------
FRONT_CTX = dict(q_lb=IDENT_Q, t_lb=ZERO_T, lidar_const=1.0, huber=0.1, unit_score=1)


def front_end_problem(oracle):
    """one scan-matching round of the front end (the problem of test_front_end_scan_matcher_settings): the oracle's
    association with the front end's gates, one LidarPlaneNormIncreFactor per match"""
    P = synth.window_problem(W=1, Q=4000, M=60000, seed=synth.SEED0 + 9)
    t2, q2 = synth.lidar_pose_in_world(P["poses_init"][0, :3], P["poses_init"][0, 3:])
    state = np.concatenate([t2, q2])[None, :]
    prm = oracle.default_params(); prm.kd_max_radius = 1.0; prm.surf_dist_thres = 0.06; prm.weight_min = 0.4; prm.lidar_const = 1.0
    o = oracle.assoc_scan_to_map(P["map_xyz"], P["scans"][0], t2, q2, prm=prm)
    v = o["status"] == oracle.GO_VALID
    return state, P["scans"][0][v], o["nsd"][v]


def incre_records(cp, nsd, kf=0, loss=0.1):
    return lidar_records(INCRE, kf, cp, a=nsd[:, :3], d=nsd[:, 3], loss=loss)


def corner_clouds(P, M=40000, Q=800):
    """a corner map and per-keyframe corner scans of the same scene and trajectory as synth.window_problem(seed) (the RNG order
    of window_problem rebuilds both), in the style of synth.window_edge_problem"""
    rng = np.random.default_rng(P["seed"])
    scene = synth.Scene(-60.0, P["W"] + 60.0, rng, n_boxes=30)
    truth = synth.trajectory(P["W"], rng)
    assert np.array_equal(truth, P["poses_true"])
    r2 = np.random.default_rng(P["seed"] + 2000)
    map_xyz = synth.corner_sample(scene, M, r2, -55.0, P["W"] + 55.0, noise=0.02).astype(np.float32)
    scans = []
    for k in range(P["W"]):
        t, q = truth[k, :3], truth[k, 3:]
        pw = synth.corner_sample(scene, Q, r2, t[0] - 50.0, t[0] + 50.0, noise=0.02)
        scans.append((((pw - t) @ synth.quat_to_R(q)) @ synth.quat_to_R(P["q_lb"]).T + P["t_lb"]).astype(np.float32))
    return map_xyz, scans


def window_edges(oracle, P, kfs, n_sel=100, score=4.0):
    """edge correspondences from tests/edge_reference.py's association at the initial poses; score 4 puts part of the
    residuals above the Huber delta"""
    from tests import edge_reference as eref
    map_xyz, scans = corner_clouds(P)
    tree = oracle.KdTree(map_xyz)
    out = {}
    for k in kfs:
        t2, q2 = synth.lidar_pose_in_world(P["poses_init"][k, :3], P["poses_init"][k, 3:], P["q_lb"], P["t_lb"])
        e = eref.associate_edges(oracle, map_xyz, scans[k], t2, q2, tree=tree)
        assert e["n"] >= n_sel
        out[k] = dict(cp=e["cp"][:n_sel], pa=e["pa"][:n_sel], pb=e["pb"][:n_sel], s=np.full(n_sel, score))
    return out


def edge_raw_residuals(pose, e, q_lb, t_lb):
    R = er.edge_residuals(pose, e["cp"], e["pa"], e["pb"], e["s"], q_lb, t_lb, 0.0)
    return np.abs(R["r"].astype(np.float64))


def window_case(oracle):
    """W = 4: keyframe 0 planes and edges, 1 planes only, 2 edges only, 3 both; plus the stand-in host factors"""
    P, kf, cp, nsd, w, sb0, priors, betweens, ranges = sc.make_problem(oracle, synth)
    keep = kf != 2
    kf, cp, nsd, w = kf[keep], cp[keep], nsd[keep], w[keep]
    E = window_edges(oracle, P, (0, 2, 3))
    raw = np.concatenate([edge_raw_residuals(P["poses_init"][k], E[k], P["q_lb"], P["t_lb"]) for k in E])
    assert (raw > HUBER).any() and (raw < HUBER).any()
    ctx = dict(q_lb=P["q_lb"], t_lb=P["t_lb"], lidar_const=LIDAR_CONST, huber=HUBER, unit_score=0)
    planes = [lidar_records(PLANE, k, cp[kf == k], a=nsd[kf == k, :3], d=nsd[kf == k, 3], s=LIDAR_CONST * w[kf == k].astype(np.float64),
                            q_lb=P["q_lb"], t_lb=P["t_lb"], loss=HUBER) for k in range(4)]
    edges = {k: lidar_records(EDGE, k, E[k]["cp"], a=E[k]["pa"], b=E[k]["pb"], s=E[k]["s"], q_lb=P["q_lb"], t_lb=P["t_lb"], loss=HUBER) for k in E}
    return dict(P=P, kf=kf, cp=cp, nsd=nsd, w=w, sb0=sb0, priors=priors, betweens=betweens, ranges=ranges, E=E, ctx=ctx,
                planes=planes, edges=edges)


def window_lidar(c, W=4, with_edges=True):
    """the LiDAR blocks of keyframes 0..W-1, keyframe by keyframe (planes, then edges); with_edges may be a set of keyframes"""
    out = []
    for k in range(W):
        out.append(c["planes"][k])
        if with_edges and k in c["edges"] and (with_edges is True or k in with_edges):
            out.append(c["edges"][k])
    return np.concatenate(out)


def write_window(path, c, W=4, with_edges=True, extra=None, **kw):
    lid = window_lidar(c, W, with_edges)
    if extra is not None:
        lid = np.concatenate([lid, extra])
    write_problem(path, c["P"]["poses_init"][:W], lid, c["ctx"], sb=c["sb0"][:W],
                  priors=[p for p in c["priors"] if p[0] < W], betweens=[b for b in c["betweens"] if b[1] < W],
                  ranges=[r for r in c["ranges"] if r[0] < W], **kw)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_host_evaluate_edge_and_incre_functors(tmp_path):
    """Problem::Evaluate of edge-only and Incre-only problems against the extended-precision reference: pins the functors"""
    exe = sc.build_driver(tmp_path, "shim_routes_test")
    rng = np.random.default_rng(5)
    poses = er.make_poses(2, rng)
    q_lb, t_lb = er.Q_LB_NONUNIT, er.T_LB
    ctx = dict(q_lb=q_lb, t_lb=t_lb, lidar_const=LIDAR_CONST, huber=0.3, unit_score=0)
    E = [er.make_edges(rng, poses[k], 300, q_lb, t_lb) for k in range(2)]
    lid = np.concatenate([lidar_records(EDGE, k, E[k]["cp"], a=E[k]["pa"], b=E[k]["pb"], s=E[k]["s"], q_lb=q_lb, t_lb=t_lb, loss=0.3) for k in range(2)])
    write_problem(tmp_path / "e.bin", poses, lid, ctx)
    r = sc.run_driver(exe, "evaluate", [tmp_path / "e.bin"])[0]
    ref = er.unary_blocks(poses, E, q_lb, t_lb, LIDAR_CONST, 0.3, fn="edge")
    er.assert_within(r["eval_cost"], ref["cost"].sum(), ref["Mcost"].sum(), "edge cost")
    er.assert_within(r["gradient"], ref["g"].ravel(), ref["Mg"].ravel(), "edge gradient")      # blocks t, q per keyframe
    assert (ref["cost"] > 0).all()

    # Incre: (q, t) blocks, identity extrinsic, no score; residual n.(q cp + t) + d
    U = [er.make_unary(rng, poses[k], 300, IDENT_Q, ZERO_T) for k in range(2)]
    for u in U:
        u["weight"] = np.ones(len(u["cp"]), np.float32)
    lid = np.concatenate([incre_records(U[k]["cp"], U[k]["nsd"], kf=k) for k in range(2)])
    write_problem(tmp_path / "i.bin", poses, lid, FRONT_CTX, strategy=1)
    r = sc.run_driver(exe, "evaluate", [tmp_path / "i.bin"])[0]
    ref = er.unary_blocks(poses, U, IDENT_Q, ZERO_T, 1.0, 0.1, unit_score=True)
    er.assert_within(r["eval_cost"], ref["cost"].sum(), ref["Mcost"].sum(), "incre cost")
    g = r["gradient"].reshape(2, 6)[:, [3, 4, 5, 0, 1, 2]]                                  # blocks q, t -> t, q
    er.assert_within(g.ravel(), ref["g"].ravel(), ref["Mg"].ravel(), "incre gradient")


def _front_end_check(res, ro):
    so = ro["summary"]
    assert res["termination"] == so.termination
    assert res["n_iters"] == so.num_iterations >= 2
    assert [i[1] for i in res["iters"]] == [int(io["step_is_successful"]) for io in ro["iterations"]]
    for (i, ok, cost, radius), io in zip(res["iters"], ro["iterations"]):
        assert cost == pytest.approx(io["cost"], rel=1e-9)
    assert np.max(np.abs(res["poses"][:, :3] - ro["poses"][:, :3])) <= 1e-6
    assert sc.rot_err(res["poses"][:, 3:], ro["poses"][:, 3:]) <= 1e-8


def _front_end_case(tmp_path, oracle, mode):
    exe = sc.build_driver(tmp_path, "shim_routes_test")
    state, cp, nsd = front_end_problem(oracle)
    prob = oracle.WindowProblem(state, None, IDENT_Q, ZERO_T, huber_delta=0.1)
    prob.add_unary(np.zeros(len(cp), np.int32), cp, nsd, np.ones(len(cp)))
    for max_it in (4, 15):
        path = tmp_path / f"fe{max_it}.bin"
        write_problem(path, state, incre_records(cp, nsd), FRONT_CTX, strategy=1, max_iter=max_it)
        prob.reset_state(state)
        ro = prob.solve(oracle.solver_options(reserved=2, max_num_iterations=max_it), mode=0)
        res = sc.run_driver(exe, mode, [path])[0]
        _front_end_check(res, ro)
        assert res["device_blocks"] == (len(cp) if mode == "device" else 0)
        if mode == "device":
            assert res["device_kinds"] == (len(cp), 0) and res["edge_launches"] == 0


def test_front_end_incre_host_matches_oracle(tmp_path, oracle):
    _front_end_case(tmp_path, oracle, "host")


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_front_end_incre_device_matches_oracle(tmp_path, oracle):
    """every LidarPlaneNormIncreFactor block runs in K2 (unit_score = 1, lidar_const = 1, identity extrinsic, Huber 0.1)"""
    _front_end_case(tmp_path, oracle, "device")


@pytest.mark.gpu
def test_window_with_edges_device_host_and_window_solve(tmp_path, oracle):
    from glio_b200 import api
    exe = sc.build_driver(tmp_path, "shim_routes_test")
    c = window_case(oracle)
    path = tmp_path / "w.bin"
    write_window(path, c)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    n_planes, n_edges = len(c["kf"]), sum(len(e) for e in c["edges"].values())
    assert host["device_blocks"] == 0
    assert dev["device_blocks"] == n_planes + n_edges and dev["device_kinds"] == (n_planes, n_edges)
    assert dev["edge_launches"] >= dev["n_iters"]                 # K2e runs in every evaluation: at least one per iteration
    sc.assert_same_solve(dev, host)

    # the same lists through glio_set_matches / glio_set_edges and glio_window_use_edges(1), host factors in the callback
    P = c["P"]
    ctx = api.Context(0, q_lb=P["q_lb"], t_lb=P["t_lb"], lidar_const=LIDAR_CONST, huber_delta=HUBER)
    try:
        for k in range(4):
            m = c["kf"] == k
            ctx.set_matches(k, c["cp"][m], c["nsd"][m], c["w"][m])
            e = c["E"].get(k)
            if e is None:
                ctx.set_edges(k, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros(0))
            else:
                ctx.set_edges(k, e["cp"], e["pa"], e["pb"], e["s"])
        ctx.window_use_edges(True)
        hf = api.HostFactorSet()
        for a in c["priors"]: hf.add_prior(*a)
        for a in c["betweens"]: hf.add_between(*a)
        for a in c["ranges"]: hf.add_range(*a)
        rw = ctx.window_solve(P["poses_init"], c["sb0"], host_factors=hf)
    finally:
        ctx.close()
    ws = dict(termination=int(rw["summary"].termination), n_iters=rw["summary"].num_iterations,
              iters=[(i["iteration"], int(i["step_is_successful"]), i["cost"], i["trust_region_radius"]) for i in rw["iterations"]],
              cost=(rw["summary"].initial_cost, rw["summary"].final_cost), poses=rw["poses"], sb=rw["speed_bias"])
    sc.assert_same_solve(dev, ws)


@pytest.mark.gpu
def test_blocks_that_stay_on_the_host(tmp_path, oracle):
    """edge blocks the kernels cannot evaluate exactly stay on the host; the count of device blocks is exactly the routable ones
    and the solve agrees with the host-only one"""
    exe = sc.build_driver(tmp_path, "shim_routes_test")
    c = window_case(oracle)
    P = c["P"]
    ql, tl = P["q_lb"], P["t_lb"]
    e0, e3 = c["E"][0], c["E"][3]
    n = 10

    def bad(e, kf=0, cp=None, **kw):
        args = dict(a=e["pa"][:n], b=e["pb"][:n], s=e["s"][:n], q_lb=ql, t_lb=tl, loss=HUBER)
        args.update(kw)
        return lidar_records(EDGE, kf, e["cp"][:n] if cp is None else cp, **args)

    cp_nf = e0["cp"][:n].astype(np.float64) + 1e-9
    assert not np.array_equal(cp_nf.astype(np.float32).astype(np.float64), cp_nf)
    extra = [
        bad(e0, cp=cp_nf),                                   # a point that is not a float
        bad(e0, loss=0.5),                                   # another Huber delta
        bad(e0, loss=-1.0),                                  # no loss
        bad(e0, t_lb=tl + np.array([0.01, 0.0, 0.0])),       # another extrinsic
        bad(e3, kf=1),                                       # keyframe 1's t has a local parameterization
        bad(e0, s=np.full(n, 0.1)),                          # a weight that is not a float
    ]
    extra = np.concatenate(extra)
    t_param = np.array([0, 1, 0, 0]); q_const = np.array([0, 0, 1, 0])   # keyframe 2 (edges only): q constant
    n_planes = len(c["kf"])
    n_good_edges = len(c["E"][0]["cp"]) + len(c["E"][3]["cp"])
    cases = [
        (dict(c["ctx"]), n_planes + n_good_edges, (n_planes, n_good_edges)),
        # the edge route does not depend on the score settings; the plane blocks (score 7.5 w != lidar_const) stay on the host
        (dict(c["ctx"], unit_score=1, lidar_const=2.0), n_good_edges, (0, n_good_edges)),
    ]
    for i, (ctx, n_dev, kinds) in enumerate(cases):
        path = tmp_path / f"m{i}.bin"
        lid = np.concatenate([window_lidar(c), extra])
        write_problem(path, P["poses_init"], lid, ctx, sb=c["sb0"], priors=c["priors"], betweens=c["betweens"], ranges=c["ranges"],
                      t_param=t_param, q_const=q_const)
        dev = sc.run_driver(exe, "device", [path])[0]
        host = sc.run_driver(exe, "host", [path])[0]
        assert host["device_blocks"] == 0
        assert dev["device_blocks"] == n_dev and dev["device_kinds"] == kinds
        sc.assert_same_solve(dev, host)
        assert np.array_equal(dev["poses"][2, 3:], P["poses_init"][2, 3:])          # the constant q stayed put


@pytest.mark.gpu
def test_incre_blocks_outside_a_front_end_context(tmp_path, oracle):
    """LidarPlaneNormIncreFactor blocks go to K2 only in a front-end context: each context below differs from it in exactly one
    field, and the device count then excludes exactly the Incre blocks (the edge blocks of the same problem stay routed)"""
    exe = sc.build_driver(tmp_path, "shim_routes_test")
    state, cp, nsd = front_end_problem(oracle)
    e = er.make_edges(np.random.default_rng(23), state[0], 200, IDENT_Q, ZERO_T, noise=0.03)
    cases = [
        ("front_end", FRONT_CTX, True),
        ("unit_score_0", dict(FRONT_CTX, unit_score=0), False),
        ("lidar_const_2", dict(FRONT_CTX, lidar_const=2.0), False),
        ("t_lb", dict(FRONT_CTX, t_lb=np.array([0.0, 0.0, 0.28])), False),     # identity q, non-zero t_lb
    ]
    for name, ctx, incre_dev in cases:
        # the edge blocks carry the context's extrinsic, so they are routable in every case
        edges = lidar_records(EDGE, 0, e["cp"], a=e["pa"], b=e["pb"], s=e["s"], q_lb=ctx["q_lb"], t_lb=ctx["t_lb"], loss=0.1)
        path = tmp_path / f"{name}.bin"
        write_problem(path, state, [incre_records(cp, nsd), edges], ctx, strategy=1)
        dev = sc.run_driver(exe, "device", [path])[0]
        host = sc.run_driver(exe, "host", [path])[0]
        assert dev["device_kinds"] == ((len(cp) if incre_dev else 0), len(e["cp"])), name
        assert dev["device_blocks"] == (len(cp) if incre_dev else 0) + len(e["cp"])
        sc.assert_same_solve(dev, host, sb=False)


def _shim_problem(tmp_path, oracle, binary):
    P, kf, cp, nsd, w, sb0, priors, betweens, ranges = sc.make_problem(oracle, synth)
    lid = [lidar_records(PLANE, kf, cp, a=nsd[:, :3], d=nsd[:, 3], s=LIDAR_CONST * w.astype(np.float64), q_lb=P["q_lb"], t_lb=P["t_lb"], loss=HUBER)]
    nb = 0
    args = (P["poses_init"], sb0, P["q_lb"], P["t_lb"], LIDAR_CONST, HUBER, kf, cp, nsd, w, priors, betweens, ranges)
    path_old = tmp_path / f"old{int(binary)}.bin"
    if binary:
        bkc, bko, bcp, bnc, bsc = sc.make_binary(oracle, synth, P)
        lid.append(lidar_records(BINARY, bkc, bcp, a=bnc[:, :3], b=bnc[:, 3:], s=bsc, kf2=bko))
        nb = len(bkc)
        sc.write_problem(str(path_old), *args, binary=(bkc, bko, bcp, bnc, bsc))
    else:
        sc.write_problem(str(path_old), *args)
    path = tmp_path / f"new{int(binary)}.bin"
    write_problem(path, P["poses_init"], np.concatenate(lid), dict(q_lb=P["q_lb"], t_lb=P["t_lb"], lidar_const=LIDAR_CONST, huber=HUBER, unit_score=0),
                  sb=sb0, priors=priors, betweens=betweens, ranges=ranges)
    return path, path_old, len(kf), nb


@pytest.mark.gpu
@pytest.mark.parametrize("binary", [False, True])
def test_plane_only_problems_launch_no_edge_kernel(tmp_path, oracle, binary):
    """test_shim.py's two problems: the device block counts are unchanged and no K2e kernel is launched"""
    exe = sc.build_driver(tmp_path, "shim_routes_test")
    old = sc.build_driver(tmp_path, "shim_test")
    path, path_old, nu, nb = _shim_problem(tmp_path, oracle, binary)
    dev = sc.run_driver(exe, "device", [path])[0]
    ref = sc.run_driver(old, "device", [path_old])[0]
    assert dev["device_blocks"] == ref["device_blocks"] == nu + nb
    assert dev["edge_launches"] == 0
    assert dev["n_iters"] == ref["n_iters"]
    assert np.max(np.abs(dev["poses"] - ref["poses"])) <= 1e-9 and np.max(np.abs(dev["sb"] - ref["sb"])) <= 1e-9


@pytest.mark.gpu
def test_solve_sequences_on_one_context(tmp_path, oracle):
    """edges at W = 4 (slots 0, 2, 3), planes only at W = 3, edges on fewer slots (W = 2, slot 0), then edges on keyframe 0 only
    with keyframe 2 empty -- its slot 2 held keyframe 2's edges two solves earlier and now holds keyframe 3's planes, and an edge
    list left in it would be evaluated: every solve on one context is bit-identical to the same solve on a fresh context, with or
    without glio_window_use_edges(1) set beforehand, and after a direct caller left selected edge lists in every slot
    (glio_set_edges + glio_select_random_edges; the first solve has to clear slot 1's)"""
    exe = sc.build_driver(tmp_path, "shim_routes_test")
    c = window_case(oracle)
    paths = [tmp_path / f"s{i}.bin" for i in range(4)]
    write_window(paths[0], c, W=4)
    write_window(paths[1], c, W=3, with_edges=False)
    write_window(paths[2], c, W=2)
    write_window(paths[3], c, W=4, with_edges={0})
    fresh = [sc.run_driver(exe, "device", [p])[0] for p in paths]
    assert [f["device_kinds"][1] for f in fresh] == [sum(len(e) for e in c["edges"].values()), 0, len(c["edges"][0]), len(c["edges"][0])]
    assert [f["edge_launches"] > 0 for f in fresh] == [True, False, True, True]
    assert fresh[3]["cost"][0] < fresh[0]["cost"][0]      # the last problem really lacks the edges of slots 2 and 3
    for flags in ((), ("--use-edges",), ("--use-edges", "--preload-edges", "150")):
        seq = sc.run_driver(exe, "device", paths, *flags)
        assert len(seq) == 4
        if "--preload-edges" in flags:
            assert seq[0]["preload_cost"] > 1.0               # the left-over lists would add cost if they were evaluated
        for a, b in zip(seq, fresh):
            assert a["text"] == b["text"]
