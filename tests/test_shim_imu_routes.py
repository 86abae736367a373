"""Ceres-API shim route for the batch refinement's IMU factors (K2i: ImuFactor), driven by tests/cpp/shim_imu_routes_test.cpp:
the restated host factor against the longdouble reference, the trait's descriptions, level-1 problems built with
optimizeBatchWithLandMark's call sequence giving the same iterates host-only, device-routed and through glio_batch_solve, blocks
K2i cannot take staying on the host, and problems without IMU blocks launching no K2i kernel."""
import struct

import numpy as np
import pytest

from glio_b200 import synth
from tests import eval_reference as er
from tests import imu_factor_reference as ir
from tests import shim_common as sc
from tests.test_shim_pose_routes import binary_records

BIN_DTYPE = np.dtype([("kc", "<i4"), ("ko", "<i4"), ("cp", "<f8", (3,)), ("nc", "<f8", (6,)), ("score", "<f8")])
JAC = ("dp_dba", "dp_dbg", "dq_dbg", "dv_dba", "dv_dbg")
# the glio_imu_factor doubles from sum_dt on, in record order: what the driver's describe prints
DESC_FIELDS = (("sum_dt", 1), ("g_vec", 3), ("delta_p", 3), ("delta_q", 4), ("delta_v", 3), ("linearized_ba", 3), ("linearized_bg", 3),
               ("dp_dba", 9), ("dp_dbg", 9), ("dq_dbg", 9), ("dv_dba", 9), ("dv_dbg", 9), ("sqrt_info", 225))


# ---------------------------------------------------------------------------------------------------------------------------
# problem files
# ---------------------------------------------------------------------------------------------------------------------------
def imu_records(P, **over):
    """driver IMU records (dicts) from synth.imu_problem's factor columns and covariances; `over` sets a field on all"""
    I, out = P["imu"], []
    for n in range(len(I["i"])):
        d = dict(i=int(I["i"][n]), j=int(I["j"][n]), alt_q=-1, as_base=0, loss=-1.0, cov=P["cov"][n])
        d["sb_i"], d["sb_j"] = d["i"], d["j"]
        for k in ("sum_dt", "g_vec", "delta_p", "delta_q", "delta_v", "linearized_ba", "linearized_bg") + JAC:
            d[k] = np.array(I[k][n], np.float64)
        d.update(over)
        out.append(d)
    return out


def write_problem(path, poses, sb, att=None, binary=None, planes=(), priors=(), imu=(), t_const=None, q_const=None, sb_const=None,
                  q_alt=None, max_iter=10, time_limit=1e9):
    """att: (i, j, dq) columns of the attitude factors; planes: (k, cp, n, d, score, q_lb, t_lb, loss) LidarPlaneNormFactor blocks;
    priors: (k, sb0, w) host speed-bias priors; imu: driver records"""
    poses = np.asarray(poses, np.float64).reshape(-1, 7); K = len(poses)
    sb = np.asarray(sb, np.float64).reshape(K, 9)
    q_alt = np.zeros((0, 4)) if q_alt is None else np.asarray(q_alt, np.float64).reshape(-1, 4)
    binary = np.zeros(0, BIN_DTYPE) if binary is None else binary
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", K, len(q_alt)))
        f.write(poses.tobytes()); f.write(sb.tobytes())
        for c in (t_const, q_const, sb_const):
            f.write(np.asarray(np.zeros(K) if c is None else c, np.int32).tobytes())
        f.write(q_alt.tobytes())
        n = 0 if att is None else len(att[0])
        f.write(struct.pack("<i", n))
        for k in range(n):
            f.write(struct.pack("<ii", int(att[0][k]), int(att[1][k]))); f.write(np.asarray(att[2][k], np.float64).tobytes())
        f.write(struct.pack("<i", len(binary))); f.write(np.ascontiguousarray(binary, BIN_DTYPE).tobytes())
        f.write(struct.pack("<i", len(planes)))
        for (k, cp, nrm, d, score, q_lb, t_lb, loss) in planes:
            f.write(struct.pack("<i", k)); f.write(np.asarray([*cp, *nrm, d, score, *q_lb, *t_lb, loss], np.float64).tobytes())
        f.write(struct.pack("<i", len(priors)))
        for (k, sb0, w) in priors:
            f.write(struct.pack("<i", k)); f.write(np.asarray([*sb0, w], np.float64).tobytes())
        f.write(struct.pack("<i", len(imu)))
        for d in imu:
            f.write(struct.pack("<iiiiiid", d["i"], d["j"], d["sb_i"], d["sb_j"], d["alt_q"], d["as_base"], d["loss"]))
            f.write(np.concatenate([np.ravel(d[k]) for k in ("sum_dt", "g_vec", "delta_p", "delta_q", "delta_v", "linearized_ba",
                                                             "linearized_bg") + JAC + ("cov",)]).astype(np.float64).tobytes())
        f.write(struct.pack("<id", max_iter, time_limit))


def describe(exe, path):
    """each IMU record's trait description: (ok, i, j, active, {field: array})"""
    out = []
    for ok, i, j, act, v in sc.run_driver(exe, "describe", [path], desc_ints=4)[0]["desc"]:
        fields, o = {}, 0
        for name, n in DESC_FIELDS:
            fields[name] = np.array(v[o:o + n]); o += n
        assert o == len(v)
        out.append((ok, i, j, act, fields))
    return out


def factor_array(imu, desc):
    """the glio_imu_factor array of driver records, with the sqrt_info the trait formed"""
    from glio_b200 import api
    cols = {k: np.array([d[k] for d in imu]) for k in ("i", "j", "sum_dt", "g_vec", "delta_p", "delta_q", "delta_v", "linearized_ba",
                                                       "linearized_bg") + JAC}
    cols["sqrt_info"] = np.array([x[4]["sqrt_info"] for x in desc]).reshape(-1, 15, 15)
    return api.imu_factor_records(**cols)


# ---------------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------------
def level1(K, seed=synth.SEED0 + 18, binary=True):
    """the shipped sms_fusion_level 1 problem in the Estimator's order: per keyframe t, q and sb, the attitude factors, the
    BinaryLidarPlaneNormFactor blocks of the batch pairs, then the IMU chain (synth.imu_problem)"""
    P = synth.imu_problem(K=K, seed=seed)
    B = binary_records(P) if binary else None
    return dict(P=P, poses=P["poses_init"], sb=P["sb_init"], att=(P["i"], P["j"], P["dq"]), binary=B, imu=imu_records(P))


def write_case(path, c, **kw):
    args = dict(att=c.get("att"), binary=c.get("binary"), imu=c["imu"], planes=c.get("planes", ()), priors=c.get("priors", ()))
    args.update(kw)
    write_problem(path, c["poses"], c["sb"], **args)


def window(K=8, seed=synth.SEED0 + 21, n=60):
    """a window-shaped problem: LidarPlaneNormFactor blocks (HuberLoss(1), the context's extrinsic and lidar_const, float-exact
    data: K2's) on every keyframe, the IMU chain, and a host prior on keyframe 0's speed-bias"""
    P = synth.imu_problem(K=K, seed=seed)
    rng = np.random.default_rng(seed)
    T = P["poses_true"]
    q_lb, t_lb = np.array([1.0, 0, 0, 0]), np.array([0, 0, 0.28])
    planes = []
    for k in range(K):
        R = synth.quat_to_R(T[k, 3:])
        for _ in range(n):
            cp = rng.uniform(-15, 15, 3).astype(np.float32).astype(np.float64)
            nrm = rng.normal(0, 1, 3); nrm = (nrm / np.linalg.norm(nrm)).astype(np.float32).astype(np.float64)
            pw = R @ (cp - t_lb) + T[k, :3]
            d = float(np.float32(-nrm @ pw + rng.normal(0, 0.02)))
            w = float(np.float32(rng.uniform(0.3, 1.0)))
            planes.append((k, cp, nrm, d, 7.5 * w, q_lb, t_lb, 1.0))
    priors = [(0, P["sb_true"][0], 3.0)]
    return dict(P=P, poses=P["poses_init"], sb=P["sb_init"], att=None, imu=imu_records(P), planes=planes, priors=priors)


def quirky(P, seed):
    """P's initial states with non-unit and w < 0 quaternions, 20 km offsets, Bg_i away from linearized_bg"""
    rng = np.random.default_rng(seed)
    K = len(P["poses_init"])
    poses = P["poses_init"].copy(); sb = P["sb_init"].copy()
    poses[:, 3:] *= rng.uniform(0.7, 1.4, (K, 1)); poses[1::3, 3:] *= -1.0
    poses[:, :3] += np.array([20_000.0, -12_000.0, 150.0])
    sb[:, 6:] += rng.normal(0.0, 0.01, (K, 3))
    return poses, sb


def routable_imu(imu, K, t_const=None, q_const=None, sb_const=None, finite=None):
    """the shim's IMU routing rule, restated: no loss, a trait, all six blocks active, two different keyframes, a finite
    description; then on the candidates, each side's t paired with its q alone (and the q with that t alone), its sb used with that
    keyframe alone and the keyframe with that sb alone.  Returns a bool per record."""
    tc, qc, sc_ = (np.zeros(K, bool) if x is None else np.asarray(x, bool) for x in (t_const, q_const, sb_const))

    def sides(d):
        qi = ("alt", d["alt_q"]) if d["alt_q"] >= 0 else ("q", d["i"])
        return [(d["i"], qi, d["sb_i"]), (d["j"], ("q", d["j"]), d["sb_j"])]

    def active(t, q, s):
        return not tc[t] and not (q[0] == "q" and qc[q[1]]) and not sc_[s]
    cand = [d["loss"] < 0 and not d["as_base"] and (finite is None or finite[n]) and all(active(*x) for x in sides(d)) and
            not (d["i"] == d["j"] and d["alt_q"] < 0) for n, d in enumerate(imu)]
    qs_of_t, ts_of_q, kfs_of_sb, sbs_of_kf = {}, {}, {}, {}
    for d, c in zip(imu, cand):
        if c:
            for t, q, s in sides(d):
                qs_of_t.setdefault(t, set()).add(q); ts_of_q.setdefault(q, set()).add(t)
                kfs_of_sb.setdefault(s, set()).add((t, q)); sbs_of_kf.setdefault((t, q), set()).add(s)
    return [c and all(len(qs_of_t[t]) == 1 and len(ts_of_q[q]) == 1 and len(kfs_of_sb[s]) == 1 and len(sbs_of_kf[(t, q)]) == 1
                      for t, q, s in sides(d)) for d, c in zip(imu, cand)]


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", ["init", "quirky"])
def test_host_evaluate_imu_factor(tmp_path, state):
    """Problem::Evaluate of an IMU-only problem (the restated ImuFactor, host): residuals, cost and gradient against the longdouble
    reference within its error bound, at the initial states and at states with non-unit and w < 0 quaternions, 20 km offsets and
    every other factor's sides swapped (i > j)"""
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    K = 9
    P = synth.imu_problem(K=K, seed=synth.SEED0 + 30)
    poses, sb = P["poses_init"], P["sb_init"]
    imu = imu_records(P)
    if state == "quirky":
        poses, sb = quirky(P, 3)
        for d in imu[1::2]:
            d["i"], d["j"] = d["j"], d["i"]; d["sb_i"], d["sb_j"] = d["i"], d["j"]
    path = tmp_path / "e.bin"
    write_problem(path, poses, sb, imu=imu)
    f = factor_array(imu, describe(exe, path))
    r = sc.run_driver(exe, "evaluate", [path])[0]
    ref = ir.imu_blocks(poses, sb, f)
    res = ir.factor_residuals(poses, sb, f)
    got_r = np.array([float(x) for x in next(t for t in r["text"] if t.startswith("residuals")).split()[1:]]).reshape(-1, 15)
    er.assert_within(got_r, res["r"].astype(np.float64), res["Mr"].astype(np.float64), "residuals")
    er.assert_within(r["eval_cost"], ref["cost"], ref["Mcost"], "cost")
    er.assert_within(r["gradient"].reshape(K, 15), ref["g"], ref["Mg"], "gradient")     # per keyframe t, q (tangent), sb
    assert ref["cost"] > 0 and np.abs(ref["g"]).max() > 0


def test_descriptions_are_the_preintegration(tmp_path):
    """the trait copies the Preintegration's fields bit for bit and leaves i, j and active to the shim; its sqrt_info, formed from the
    covariance as ImuFactor forms it, matches numpy's Cholesky factor of the inverse to 1e-11 of the largest entry (15 x 15
    inverses of covariances with condition numbers up to about 1e3 after the sigma scaling is taken out)"""
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    P = synth.imu_problem(K=40, seed=synth.SEED0 + 31)
    imu = imu_records(P)
    imu[3]["delta_p"] = np.array([-0.0, 5e-324, np.pi * 1e7]); imu[3]["sum_dt"] = 1.0 - 2.0 ** -53
    path = tmp_path / "d.bin"
    write_problem(path, P["poses_init"], P["sb_init"], imu=imu)
    desc = describe(exe, path)
    assert len(desc) == len(imu)
    for d, (ok, i, j, act, v) in zip(imu, desc):
        assert ok == 1 and (i, j, act) == (0, 0, 0)
        for name, _ in DESC_FIELDS[:-1]:
            assert v[name].tobytes() == np.ravel(np.asarray(d[name], np.float64)).tobytes(), name
        S = np.linalg.cholesky(np.linalg.inv(d["cov"])).T
        assert np.max(np.abs(v["sqrt_info"].reshape(15, 15) - S)) <= 1e-11 * np.max(np.abs(S))
        assert np.all(np.tril(v["sqrt_info"].reshape(15, 15), -1) == 0)


def test_host_solve_level1(tmp_path):
    """the level-1 problem (attitude, binary-plane and IMU blocks) solved on the host only (no context): no device block, and the
    solve converges"""
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    c = level1(12)
    write_case(tmp_path / "h.bin", c, max_iter=50)
    r = sc.run_driver(exe, "host", [tmp_path / "h.bin"])[0]
    assert r["device_blocks"] == 0 and r["device_imu"] == 0 and r["imu_launches"] == 0
    assert r["blocks"] == len(c["att"][0]) + len(c["binary"]) + len(c["imu"]) == r["blocks"]
    assert r["termination"] == 0
    assert r["cost"][1] < 1e-2 * r["cost"][0]


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 7, 40, 200])
def test_device_matches_host(tmp_path, K):
    """level-1 problems (attitude, binary-plane and IMU blocks): every residual block is routed, the IMU count is the chain length,
    K2i runs in every evaluation, and the device-routed solve agrees with the host-routed one"""
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    # K = 40 uses seed SEED0 + 24 in place of the default SEED0 + 18: ImuFactor's Jacobian is not the exact derivative, so the
    # level-1 problems above a dozen keyframes converge linearly and end their 10 iterations without convergence; the default seed's
    # final cost then carried the two evaluation orders' rounding to 3.8e-9 of itself, seed 24's to 1.3e-10
    c = level1(K, seed=synth.SEED0 + (24 if K == 40 else 18))
    path = tmp_path / "p.bin"
    write_case(path, c)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    assert host["device_blocks"] == 0
    assert dev["device_blocks"] == dev["blocks"] == len(c["att"][0]) + len(c["binary"]) + K - 1
    assert dev["device_imu"] == K - 1 and dev["device_pose"] == len(c["att"][0])
    assert dev["imu_launches"] >= dev["n_iters"]
    # iterate_abs: the attitude factors (weight 10^4) make the first step drop the cost by orders of magnitude, and each later
    # iterate's cost carries the rounding of the host and device evaluation orders at the scale of the initial cost
    sc.assert_same_solve(dev, host, sb=True, iterate_abs=1e-10)


@pytest.mark.gpu
def test_device_matches_glio_batch_solve(tmp_path):
    """attitude and IMU blocks: the device-routed solve against glio_batch_solve with glio_batch_use_pose_factors(1) and
    glio_batch_use_imu_factors(1) on the same lists (the IMU list with the trait's sqrt_info) and the speed-bias states"""
    from glio_b200 import api
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    max_iter = 8
    c = level1(40, binary=False)
    path = tmp_path / "p.bin"
    write_case(path, c, max_iter=max_iter)
    dev = sc.run_driver(exe, "device", [path])[0]
    f = factor_array(c["imu"], describe(exe, path))
    P = c["P"]
    ctx = api.Context(0)
    try:
        ctx.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"]))
        ctx.batch_use_pose_factors(True)
        ctx.batch_set_imu_factors(f)
        ctx.batch_use_imu_factors(True)
        out = ctx.batch_solve(c["poses"], c["sb"], options=api.batch_solver_options(max_num_iterations=max_iter), max_log=64)
    finally:
        ctx.close()
    summ = out["summary"]
    bs = dict(termination=int(summ.termination), n_iters=summ.num_iterations, cost=(summ.initial_cost, summ.final_cost), poses=out["poses"],
              sb=out["speed_bias"], iters=[(i["iteration"], int(i["step_is_successful"]), i["cost"], i["trust_region_radius"]) for i in out["iterations"]])
    assert dev["device_imu"] == len(c["imu"]) and dev["device_blocks"] == dev["blocks"]
    sc.assert_same_solve(dev, bs, sb=True, iterate_abs=1e-10)       # iterate_abs as in test_device_matches_host


@pytest.mark.gpu
def test_window_shaped_problem(tmp_path):
    """LidarPlaneNormFactor blocks on K2, the IMU chain on K2i and a host speed-bias prior: the plane and IMU blocks are routed, the
    prior stays on the host, and the solve agrees with the host one"""
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    c = window()
    path = tmp_path / "w.bin"
    write_case(path, c)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    assert dev["device_imu"] == len(c["imu"])
    assert dev["device_blocks"] == len(c["planes"]) + len(c["imu"]) == dev["blocks"] - 1
    sc.assert_same_solve(dev, host, sb=True, iterate_abs=1e-10)     # iterate_abs as in test_device_matches_host


@pytest.mark.gpu
def test_blocks_that_stay_on_the_host(tmp_path):
    """IMU blocks K2i cannot take stay on the host, next to routed ones: a loss, a constant t, q and sb, an sb shared by two
    keyframes, a t paired with two q blocks, the same keyframe on both sides, and a factor added through a ceres::CostFunction*.  The
    IMU device count is exactly the routable number, and the solve agrees with the host one.  A non-finite description stays on the
    host too: glio_batch_set_imu_factors never sees it, and both solves end alike at the non-finite initial cost."""
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    K = 30
    c = level1(K, binary=False)
    imu = c["imu"]
    t_const, q_const, sb_const = np.zeros(K, int), np.zeros(K, int), np.zeros(K, int)
    t_const[3] = 1; q_const[7] = 1; sb_const[11] = 1
    imu[14]["loss"] = 0.5
    imu[17]["sb_j"] = 19                                          # sb_19 with keyframes 18 and 19; keyframe 18 with sb_18 and sb_19
    extra = [dict(imu[22], alt_q=0),                              # t_22 with q_22 and another q
             dict(imu[25], j=25, sb_j=25),                        # keyframe 25 on both sides
             dict(imu[27], as_base=1)]                            # through a ceres::CostFunction*
    imu = imu + extra
    q_alt = c["poses"][22:23, 3:]
    flags = dict(t_const=t_const, q_const=q_const, sb_const=sb_const)
    expect = sum(routable_imu(imu, K, **flags))
    assert 0 < expect < len(c["imu"]) - 10
    path = tmp_path / "m.bin"
    write_case(path, c, imu=imu, q_alt=q_alt, **flags)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    assert host["device_blocks"] == 0
    assert dev["device_imu"] == expect
    assert dev["device_blocks"] == dev["device_imu"] + dev["device_pose"] < dev["blocks"]
    sc.assert_same_solve(dev, host, sb=True, iterate_abs=1e-10)     # iterate_abs as in test_device_matches_host
    assert np.array_equal(dev["poses"][3, :3], c["poses"][3, :3]) and np.array_equal(dev["sb"][11], c["sb"][11])
    base = sc.run_driver(exe, "device", [path], "--imu-as-cost-function")[0]     # every ImuFactor through a ceres::CostFunction*
    assert base["device_imu"] == 0 and base["imu_launches"] == 0

    bad = imu_records(c["P"])
    bad[5]["cov"] = bad[5]["cov"].copy(); bad[5]["cov"][2, 2] = np.nan
    path2 = tmp_path / "n.bin"
    write_case(path2, c, imu=bad)
    dev = sc.run_driver(exe, "device", [path2])[0]
    host = sc.run_driver(exe, "host", [path2])[0]
    finite = [n != 5 for n in range(len(bad))]
    assert dev["device_imu"] == sum(routable_imu(bad, K, finite=finite)) == len(bad) - 1
    assert dev["termination"] == host["termination"] and dev["n_iters"] == host["n_iters"]
    assert dev["text"][dev["text"].index(next(t for t in dev["text"] if t.startswith("cost"))):] == \
        host["text"][host["text"].index(next(t for t in host["text"] if t.startswith("cost"))):]


@pytest.mark.gpu
def test_solve_sequences_on_one_context(tmp_path):
    """IMU problem -> problem without IMU blocks -> IMU problem on one context print the same text (%.17g) as fresh contexts, also
    with glio_batch_use_imu_factors on and after a direct caller left another IMU list with the switch on; the problem without IMU
    blocks launches no K2i kernel"""
    exe = sc.build_driver(tmp_path, "shim_imu_routes_test")
    paths = [tmp_path / f"s{i}.bin" for i in range(3)]
    write_case(paths[0], level1(40))
    write_case(paths[1], level1(30, seed=synth.SEED0 + 19), imu=[])
    write_case(paths[2], window())
    fresh = [sc.run_driver(exe, "device", [p])[0] for p in paths]
    assert [f["imu_launches"] > 0 for f in fresh] == [True, False, True]
    assert fresh[1]["device_imu"] == 0 and fresh[1]["device_pose"] > 0
    for flags in ((), ("--use-imu",), ("--preload-imu", "40")):
        seq = sc.run_driver(exe, "device", paths, *flags)
        assert len(seq) == 3
        for a, b in zip(seq, fresh):
            assert a["text"] == b["text"]
