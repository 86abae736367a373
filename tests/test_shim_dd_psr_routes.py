"""Ceres-API shim route for the batch refinement's DD pseudorange factors (K2g: dd_psr_factor_20), driven by
tests/cpp/shim_dd_psr_routes_test.cpp: problems built with optimizeBatchWithLandMark's call sequence give the same iterates
host-only and device-routed and through glio_batch_solve, a level-0 problem routes every residual block, blocks K2g cannot
evaluate exactly stay on the host, and problems without DD blocks launch no K2g kernel."""
import struct

import numpy as np
import pytest

from glio_b200 import synth
from tests import dd_psr_reference as dr
from tests import eval_reference as er
from tests import shim_common as sc
from tests.test_shim_pose_routes import binary_records, curved_pose_graph

YAW = 0.3
REL, DQ = 0, 1                                  # the driver's pose record kinds (synth's kind column: 1 = attitude)
BIN_DTYPE = np.dtype([("kc", "<i4"), ("ko", "<i4"), ("cp", "<f8", (3,)), ("nc", "<f8", (6,)), ("score", "<f8")])


# ---------------------------------------------------------------------------------------------------------------------------
# problem files
# ---------------------------------------------------------------------------------------------------------------------------
def dd_from_records(f, sats, W=None, **over):
    """driver DD records (dicts) from a glio_dd_psr_factor array, its satellites and weights; `over` sets a field on all"""
    out = []
    for F in f:
        n, o = int(F["n_sat"]), int(F["sat_offset"])
        S = sats[o:o + n]
        d = dict(i=int(F["i"]), j=int(F["j"]), master=int(F["master"]), ratio=float(F["ratio"]), threshold=float(F["threshold"]),
                 station=np.array(F["station"], np.float64), frame=0, as_base=0, loss=-1.0,
                 user=np.column_stack([S["sat_user"], S["psr_user"]]), ref=np.column_stack([S["sat_ref"], S["psr_ref"]]), W=None)
        if W is not None and int(F["w_offset"]) >= 0:
            d["W"] = np.asarray(W[int(F["w_offset"]):int(F["w_offset"]) + (n - 1) ** 2], np.float64).reshape(n - 1, n - 1)
        d.update(over)
        out.append(d)
    return out


def records_from_dd(dds):
    """the glio_dd_psr_factor list, satellites and weights a Level-2 caller passes for driver records (all frame 0)"""
    from glio_b200 import api
    n_sat = np.array([len(d["user"]) for d in dds], np.int32)
    W, w_off = [], []
    for d in dds:
        w_off.append(-1 if d["W"] is None else sum(len(x) for x in W))
        if d["W"] is not None:
            W.append(np.asarray(d["W"]).ravel())
    f = api.dd_psr_factor_records([d["i"] for d in dds], [d["j"] for d in dds], n_sat, [d["master"] for d in dds], [d["ratio"] for d in dds],
                                  [d["threshold"] for d in dds], np.array([d["station"] for d in dds]), w_offset=w_off)
    U = np.concatenate([d["user"] for d in dds]); Rf = np.concatenate([d["ref"] for d in dds])
    sats = api.dd_psr_sat_records(U[:, :3], Rf[:, :3], U[:, 3], Rf[:, 3])
    return f, sats, (np.concatenate(W) if W else None)


def write_problem(path, poses, pose=None, binary=None, dds=(), frames=None, t_const=None, q_alt=None, max_iter=10, time_limit=1e9):
    """pose: columns (kind, i, j, dq, dp[, alt_q]) as synth's pose lists; frames: (yaw, anchor, yaw_const, anchor_const), default
    one constant frame at dd_psr_reference.frame's anchor"""
    poses = np.asarray(poses, np.float64).reshape(-1, 7); K = len(poses)
    if frames is None:
        frames = [(YAW, dr.frame(YAW)[1], 1, 1)]
    q_alt = np.zeros((0, 4)) if q_alt is None else np.asarray(q_alt, np.float64).reshape(-1, 4)
    binary = np.zeros(0, BIN_DTYPE) if binary is None else binary
    with open(path, "wb") as f:
        f.write(struct.pack("<iii", K, len(q_alt), len(frames)))
        f.write(poses.tobytes())
        f.write(np.asarray(t_const if t_const is not None else np.zeros(K), np.int32).tobytes())
        for yaw, anchor, yc, ac in frames:
            f.write(struct.pack("<d", yaw)); f.write(np.asarray(anchor, np.float64).tobytes()); f.write(struct.pack("<ii", yc, ac))
        f.write(q_alt.tobytes())
        n = 0 if pose is None else len(pose["i"])
        f.write(struct.pack("<i", n))
        for k in range(n):
            alt = int(pose["alt_q"][k]) if "alt_q" in pose else -1
            f.write(struct.pack("<iiii", REL if pose["kind"][k] == 0 else DQ, int(pose["i"][k]), int(pose["j"][k]), alt))
            f.write(np.asarray(pose["dq"][k], np.float64).tobytes()); f.write(np.asarray(pose["dp"][k], np.float64).tobytes())
        f.write(struct.pack("<i", len(binary))); f.write(np.ascontiguousarray(binary, BIN_DTYPE).tobytes())
        f.write(struct.pack("<i", len(dds)))
        for d in dds:
            W = d.get("W")
            w_rows = 0 if W is None else np.asarray(W).shape[0]
            f.write(struct.pack("<iiiiiiii", d["i"], d["j"], len(d["user"]), len(d["ref"]), d["master"], d.get("frame", 0), d.get("as_base", 0), w_rows))
            f.write(struct.pack("<dd", d["ratio"], d["threshold"])); f.write(np.asarray(d["station"], np.float64).tobytes())
            f.write(struct.pack("<d", d.get("loss", -1.0)))
            f.write(np.ascontiguousarray(d["user"], np.float64).tobytes()); f.write(np.ascontiguousarray(d["ref"], np.float64).tobytes())
            if w_rows:
                f.write(np.ascontiguousarray(W, np.float64).tobytes())
        f.write(struct.pack("<id", max_iter, time_limit))


# ---------------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------------
def gnss_dd(truth, init, seed, outer_pass):
    """synth.dd_psr_problem's GNSS part on a given trajectory: keyframe times about 3 Hz, synth.gnss_epochs at 10 Hz and the DD list of
    outer pass `outer_pass` built against the initial states"""
    K = len(truth)
    rng = np.random.default_rng([seed, 1])
    kf_times = 1_600_000_000.0 + np.concatenate([[0.0], np.cumsum(rng.uniform(0.25, 0.45, K - 1))])
    R, anchor, station = dr.frame(YAW)
    epochs = synth.gnss_epochs(kf_times, truth[:, :3], R, anchor, station, rng)
    cols, sats = synth.dd_psr_factors(epochs, kf_times, init[:, :3], station, synth.DD_PSR_THRESHOLDS[outer_pass])
    from glio_b200 import api
    if len(cols["i"]) == 0:
        return []
    f = api.dd_psr_factor_records(cols["i"], cols["j"], cols["n_sat"], cols["master"], cols["ratio"], cols["threshold"], cols["station"])
    return dd_from_records(f, api.dd_psr_sat_records(sats["sat_user"], sats["sat_ref"], sats["psr_user"], sats["psr_ref"]))


def random_dd(truth, ij, seed, n_sat=None, with_w=False, thresholds=(1e9, 10.0, 8.0, 6.0)):
    rng = np.random.default_rng(seed)
    ij = np.asarray(ij, np.int32).reshape(-1, 2)
    n_sat = rng.integers(4, 13, len(ij)) if n_sat is None else n_sat
    f, sats, W, _, _ = dr.random_list(rng, truth, ij, n_sat, thresholds=thresholds, with_w=with_w)
    return dd_from_records(f, sats, W)


def level0(K, seed=synth.SEED0 + 16, outer_pass=1):
    """the shipped sms_fusion_level 0 problem: attitude then relative factors on a trajectory that curves in y and z (see
    tests/test_shim_pose_routes.py), constant yaw and anchor, then the DD factors per epoch and constellation.  Below 4 keyframes
    the generator's epochs fall outside the bracketing rule; such problems get DD factors between keyframes 0 and 1 instead."""
    P = curved_pose_graph(K, seed)
    dds = gnss_dd(P["poses_true"], P["poses_init"], seed, outer_pass)
    if not dds:
        dds = random_dd(P["poses_true"], [[0, 1]] * 4, seed, thresholds=(synth.DD_PSR_THRESHOLDS[outer_pass],))
    return dict(P=P, poses=P["poses_init"], pose=P, dds=dds)


def dd_chain(n_pairs, seed, per_pair=3, with_w=False):
    """a DD-only problem: K = n_pairs + 1 translation-only keyframes, per_pair factors on each neighbour pair"""
    K = n_pairs + 1
    rng = np.random.default_rng(seed)
    truth = synth.trajectory(K, rng)
    init = truth.copy(); init[:, :3] += rng.normal(0, 0.5, (K, 3))
    ij = [[k, k + 1] if n % 2 else [k + 1, k] for k in range(n_pairs) for n in range(per_pair)]
    return dict(poses=init, truth=truth, dds=random_dd(truth, ij, seed, with_w=with_w))


def write_case(path, c, **kw):
    args = dict(pose=c.get("pose"), dds=c["dds"]); args.update(kw)
    write_problem(path, c["poses"], **args)


def n_pose(c):
    return 0 if c.get("pose") is None else len(c["pose"]["i"])


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_host_evaluate_dd_factor(tmp_path):
    """Problem::Evaluate of a DD-only problem (the restated factor, host) against the longdouble reference: n_sat 2 .. 20, the master
    anywhere, i < j and i > j, identity and dense W, the 1e9 / 10 / 8 / 6 gates"""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    rng = np.random.default_rng(21)
    K = 6
    truth = synth.trajectory(K, rng)
    poses = truth.copy(); poses[:, :3] += rng.normal(0, 2.0, (K, 3))
    ij = np.array([[0, 1], [2, 1], [3, 4], [5, 4], [1, 3], [0, 5], [2, 3], [4, 2]])
    f, sats, W, _, anchor = dr.random_list(rng, truth, ij, np.array([2, 3, 19, 20, 7, 11, 5, 9]), with_w=True)
    dds = dd_from_records(f, sats, W)
    write_problem(tmp_path / "e.bin", poses, dds=dds)
    frame = sc.run_driver(exe, "describe", [tmp_path / "e.bin"], desc_ints=4)[0]["frames"][0]
    r = sc.run_driver(exe, "evaluate", [tmp_path / "e.bin"])[0]
    ref = dr.dd_blocks(poses, f, sats, frame, anchor, W)
    er.assert_within(r["eval_cost"], ref["cost"], ref["Mcost"], "cost")
    g = r["gradient"][:6 * K].reshape(K, 6)                        # per keyframe t, q (tangent); then yaw and anchor
    er.assert_within(g[:, :3], ref["g"][:, :3], ref["Mg"][:, :3], "gradient")
    assert np.all(g[:, 3:] == 0) and np.all(r["gradient"][6 * K:] == 0)
    assert ref["cost"] > 0


def test_ecef2rotation_matches_synth(tmp_path):
    """the driver's gnss_comm ecef2rotation * R_enu_local(yaw) (the trait's frame()) against synth.ecef_local_rotation"""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    frames = [(y, synth.geo_to_ecef(lat, lon, h), 1, 1) for y, lat, lon, h in
              ((0.3, 22.3, 114.18, 5.0), (-2.0, -33.9, 151.2, 40.0), (1.1, 64.1, -21.9, 0.0), (0.0, 0.5, -179.0, 1200.0), (3.0, -80.0, 10.0, 5.0))]
    write_problem(tmp_path / "f.bin", np.tile([0, 0, 0, 1, 0, 0, 0], (2, 1)), frames=frames)
    got = sc.run_driver(exe, "describe", [tmp_path / "f.bin"], desc_ints=4)[0]["frames"]
    assert len(got) == len(frames)
    for R, (yaw, anchor, _, _) in zip(got, frames):
        np.testing.assert_allclose(R, synth.ecef_local_rotation(anchor, yaw), rtol=0, atol=4e-16)
        np.testing.assert_allclose(R @ R.T, np.eye(3), rtol=0, atol=2e-15)


def _desc_case(rng, n_sat, master, W=None, n_ref=None):
    user = np.column_stack([rng.normal(0, 2e7, (n_sat, 3)), rng.normal(2e7, 1e5, n_sat)])
    ref = np.column_stack([rng.normal(0, 2e7, (n_ref or n_sat, 3)), rng.normal(2e7, 1e5, n_ref or n_sat)])
    return dict(i=0, j=1, master=master, ratio=float(rng.uniform()), threshold=float(rng.choice([1e9, 10.0, 8.0, 6.0])),
                station=rng.normal(0, 6e6, 3), user=user, ref=ref, W=W)


def test_descriptions_are_the_constructor_arguments(tmp_path):
    """the trait returns the factor's private data bit for bit, read through the explicit-instantiation idiom; it refuses what K2g
    cannot evaluate: n_sat 1 and 21, a master out of range, a W of the wrong size, station data of another length"""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    rng = np.random.default_rng(5)
    good = []
    for n_sat in (2, 3, 19, 20):
        for master in sorted({0, n_sat // 2, n_sat - 1}):
            good.append(_desc_case(rng, n_sat, master))
            good.append(_desc_case(rng, n_sat, master, W=np.eye(n_sat - 1) + rng.normal(0, 0.1, (n_sat - 1, n_sat - 1))))
    good.append(_desc_case(rng, 5, 2, W=np.eye(4)))                                 # an identity given densely
    nearly = np.eye(4); nearly[1, 2] = -0.0; nearly[3, 0] = 5e-324
    good.append(_desc_case(rng, 5, 1, W=nearly))                                   # a subnormal off the diagonal: not identity
    good[0]["station"] = np.array([-0.0, 1e-300, np.pi * 1e7]); good[0]["ratio"] = 1.0 - 2.0 ** -53
    bad = [_desc_case(rng, 1, 0), _desc_case(rng, 21, 3), _desc_case(rng, 6, 6), _desc_case(rng, 6, -1),
           _desc_case(rng, 6, 2, W=np.eye(4)), _desc_case(rng, 6, 2, W=np.eye(6)), _desc_case(rng, 6, 2, n_ref=7), _desc_case(rng, 6, 2, n_ref=5)]
    write_problem(tmp_path / "d.bin", np.tile([0, 0, 0, 1, 0, 0, 0], (2, 1)), dds=good + bad)
    desc = sc.run_driver(exe, "describe", [tmp_path / "d.bin"], desc_ints=4)[0]["desc"]
    assert len(desc) == len(good) + len(bad)
    for d, (ok, n_sat, master, ident, v) in zip(good, desc):
        n = len(d["user"])
        assert ok == 1 and n_sat == n and master == d["master"]
        W = np.eye(n - 1) if d["W"] is None else d["W"]
        assert ident == int(np.array_equal(W, np.eye(n - 1)))                     # -0.0 == 0.0: still the identity
        head = np.array(v[:5]); sat = np.array(v[5:5 + 8 * n]).reshape(n, 8); w = np.array(v[5 + 8 * n:])
        assert head.tobytes() == np.array([d["ratio"], d["threshold"], *d["station"]]).tobytes()
        assert sat[:, :4].tobytes() == np.ascontiguousarray(d["user"]).tobytes()
        assert sat[:, 4:].tobytes() == np.ascontiguousarray(d["ref"]).tobytes()
        assert w.tobytes() == np.ascontiguousarray(W, np.float64).ravel().tobytes()
    assert desc[len(good) - 1][3] == 0 and desc[len(good) - 2][3] == 1             # the subnormal case; the dense identity
    for ok, *_ in desc[len(good):]:
        assert ok == 0


def test_host_solve_level0(tmp_path):
    """the level-0 problem with its DD factors solved on the host only (no context): no device block, a cost that drops, and a gate
    margin the driver reports"""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    c = level0(30)
    write_case(tmp_path / "h.bin", c)
    r = sc.run_driver(exe, "host", [tmp_path / "h.bin"])[0]
    assert r["device_blocks"] == 0 and r["device_dd"] == 0 and r["dd_launches"] == 0
    assert r["blocks"] == n_pose(c) + len(c["dds"]) and len(c["dds"]) > 0
    assert r["cost"][1] < 1e-2 * r["cost"][0]
    assert 0 < r["gate_margin"] < np.inf


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
def assert_gate_clear(h):
    """no comparison is decided by a gate flip at rounding level: every DD row the host evaluated is 1e-6 m or more from its
    threshold"""
    assert h["gate_margin"] > 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("outer_pass", [0, 1, 2, 3])
@pytest.mark.parametrize("K", [2, 7, 40, 200])
def test_device_matches_host(tmp_path, K, outer_pass):
    """level-0 problems (attitude, relative and DD blocks) at each outer pass's threshold: every residual block is routed, and the
    device-routed solve agrees with the host-routed one"""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    # K = 7 uses seed SEED0 + 29 in place of the default SEED0 + 16: at that size the pass-0 problem (every outlier row at full
    # weight) of the default seed ends without convergence after its 10 iterations, and its nonmonotonic steps carried the DD
    # rows' rounding (a few 1e-11 of the cost per evaluation) to 3e-9 of an iterate's cost; seed 29's problems converge at every pass
    c = level0(K, seed=synth.SEED0 + (29 if K == 7 else 16), outer_pass=outer_pass)
    path = tmp_path / "p.bin"
    write_case(path, c)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    n_dd = len(c["dds"])
    assert n_dd > 0 and host["device_blocks"] == 0
    assert dev["device_blocks"] == dev["blocks"] == n_pose(c) + n_dd
    assert dev["device_dd"] == n_dd and dev["device_pose"] == n_pose(c)
    assert dev["dd_launches"] >= dev["n_iters"]                     # K2g runs in every evaluation
    assert_gate_clear(host)
    sc.assert_same_solve(dev, host, sb=False, iterate_abs=1e-10)


@pytest.mark.gpu
@pytest.mark.parametrize("outer_pass", [1, 3])
def test_device_matches_glio_batch_solve(tmp_path, outer_pass):
    """the device-routed solve against glio_batch_solve with glio_batch_use_pose_factors(1) and glio_batch_use_dd_psr_factors(1) on
    the same pose and DD lists, with the R the trait's frame() gives"""
    from glio_b200 import api
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    max_iter = 8
    c = level0(40, outer_pass=outer_pass)
    path = tmp_path / "p.bin"
    write_case(path, c, max_iter=max_iter)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    R = sc.run_driver(exe, "describe", [path], desc_ints=4)[0]["frames"][0]
    P = c["P"]
    f, sats, W = records_from_dd(c["dds"])
    ctx = api.Context(0)
    try:
        ctx.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"]))
        ctx.batch_use_pose_factors(True)
        ctx.batch_set_dd_psr_factors(f, sats, R, dr.frame(YAW)[1], W)
        ctx.batch_use_dd_psr_factors(True)
        out = ctx.batch_solve(c["poses"], options=api.batch_solver_options(max_num_iterations=max_iter), max_log=64)
    finally:
        ctx.close()
    summ = out["summary"]
    bs = dict(termination=int(summ.termination), n_iters=summ.num_iterations, cost=(summ.initial_cost, summ.final_cost), poses=out["poses"],
              iters=[(i["iteration"], int(i["step_is_successful"]), i["cost"], i["trust_region_radius"]) for i in out["iterations"]])
    assert dev["device_dd"] == len(c["dds"]) and dev["device_blocks"] == dev["blocks"]
    assert_gate_clear(host)
    sc.assert_same_solve(dev, bs, sb=False, iterate_abs=1e-10)


@pytest.mark.gpu
def test_dd_pair_counts_and_translation_only_keyframes(tmp_path):
    """DD-only problems (every keyframe translation-only: its q blocks are unused) with exactly 1, 3, 4, 5, 8 and 9 distinct DD pairs
    (K2g gives 4 pairs to a block), i < j and i > j, solved in turn on one context and on the host; one of them with dense W"""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    paths = []
    for n_pairs in (1, 3, 4, 5, 8, 9):
        c = dd_chain(n_pairs, synth.SEED0 + 60 + n_pairs, with_w=n_pairs == 5)
        assert len({(min(d["i"], d["j"]), max(d["i"], d["j"])) for d in c["dds"]}) == n_pairs
        path = tmp_path / f"c{n_pairs}.bin"
        write_case(path, c)
        paths.append((path, len(c["dds"])))
    dev = sc.run_driver(exe, "device", [p for p, _ in paths])
    host = sc.run_driver(exe, "host", [p for p, _ in paths])
    for d, h, (_, n) in zip(dev, host, paths):
        assert d["device_dd"] == d["device_blocks"] == d["blocks"] == n and d["device_pose"] == 0
        assert_gate_clear(h)
        sc.assert_same_solve(d, h, sb=False, iterate_abs=1e-10)


@pytest.mark.gpu
def test_level1_shape_and_dense_weights(tmp_path):
    """a level-1-shaped problem (BinaryLidarPlaneNormFactor blocks of the batch pairs, attitude and DD blocks: DD keyframes shared
    with the binary-plane keyframes), and a level-0 problem whose DD factors carry dense, non-identity weights"""
    from glio_b200.dist import batch_pairs
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    K = 30
    c = level0(K, seed=synth.SEED0 + 18)
    P = dict(c["P"]); P["pairs"] = batch_pairs(K, 6)
    att = P["kind"] == 1
    pose = {k: P[k][att] for k in ("i", "j", "kind", "dq", "dp")}
    B = binary_records(P)
    path1 = tmp_path / "l1.bin"
    write_problem(path1, c["poses"], pose=pose, binary=B, dds=c["dds"])
    rng = np.random.default_rng(9)
    dds = [dict(d) for d in c["dds"]]
    for d in dds[::2]:
        m = len(d["user"]) - 1
        d["W"] = np.eye(m) + rng.normal(0, 0.1, (m, m))
    path2 = tmp_path / "w.bin"
    write_case(path2, c, dds=dds)
    dev = sc.run_driver(exe, "device", [path1, path2])
    host = sc.run_driver(exe, "host", [path1, path2])
    assert dev[0]["device_blocks"] == dev[0]["blocks"] == len(B) + int(att.sum()) + len(c["dds"])
    assert dev[1]["device_blocks"] == dev[1]["blocks"] and dev[1]["device_dd"] == len(dds)
    for d, h in zip(dev, host):
        assert_gate_clear(h)
        sc.assert_same_solve(d, h, sb=False, iterate_abs=1e-10)


@pytest.mark.gpu
def test_blocks_that_stay_on_the_host(tmp_path):
    """DD blocks K2g cannot evaluate exactly stay on the host, next to routed ones: a variable yaw, a variable anchor, a loss, t_i ==
    t_j, a constant t (keyframe 0 gauge-fixed), a second constant (yaw, anchor) pair, a t paired with two q blocks, and a factor
    added through a ceres::CostFunction*.  The DD device count is exactly the routable one, and the solve agrees with the host one."""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    K = 30
    c = level0(K)
    base = c["dds"]
    anchor = dr.frame(YAW)[1]
    frames = [(YAW, anchor, 1, 1), (YAW + 0.01, anchor + 50.0, 1, 1), (YAW, anchor, 0, 1), (YAW, anchor, 1, 0)]
    pick = [d for d in base if 0 not in (d["i"], d["j"]) and 20 not in (d["i"], d["j"])][:8]
    extra = [dict(pick[0], frame=2), dict(pick[1], frame=3), dict(pick[2], loss=0.5), dict(pick[3], j=pick[3]["i"]),
             dict(pick[4], frame=1), dict(pick[5], as_base=1), dict(pick[6], i=20), dict(pick[7], j=0)]
    dds = base + extra
    t_const = np.zeros(K, int); t_const[0] = 1                                       # gauge-fixed keyframe 0
    P = c["P"]
    pose = {k: np.asarray(P[k]) for k in ("i", "j", "kind", "dq", "dp")}
    pose["alt_q"] = np.full(len(pose["i"]), -1)
    rel = np.nonzero((pose["kind"] == 0) & (pose["i"] == 20))[0][0]                 # t_20 paired with q_20 and another q
    for k in ("i", "j", "kind", "dq", "dp"):
        pose[k] = np.concatenate([pose[k], pose[k][rel:rel + 1]])
    pose["alt_q"] = np.concatenate([pose["alt_q"], [0]])
    q_alt = c["poses"][20:21, 3:]

    def routable(d):
        return (d.get("frame", 0) == 0 and d.get("loss", -1.0) < 0 and d["i"] != d["j"] and not d.get("as_base", 0) and
                0 not in (d["i"], d["j"]) and 20 not in (d["i"], d["j"]))
    expect = sum(routable(d) for d in dds)
    assert 0 < expect < len(dds) - len(extra) + 1 and expect < len(base)
    path = tmp_path / "m.bin"
    write_problem(path, c["poses"], pose=pose, dds=dds, frames=frames, t_const=t_const, q_alt=q_alt)
    dev = sc.run_driver(exe, "device", [path])[0]
    host = sc.run_driver(exe, "host", [path])[0]
    assert host["device_blocks"] == 0
    assert dev["device_dd"] == expect
    assert dev["device_blocks"] == dev["device_dd"] + dev["device_pose"] < dev["blocks"]
    assert_gate_clear(host)
    sc.assert_same_solve(dev, host, sb=False, iterate_abs=1e-10)
    assert np.array_equal(dev["poses"][0, :3], c["poses"][0, :3])                  # the constant t stayed put


@pytest.mark.gpu
def test_solve_sequences_on_one_context(tmp_path):
    """DD problem -> pose-only problem -> DD-only problem -> DD problem on one context print the same text (%.17g) as fresh contexts,
    also with both switches on and after a direct caller left another DD list with the switch on; the pose-only problem launches no
    K2g kernel"""
    exe = sc.build_driver(tmp_path, "shim_dd_psr_routes_test")
    paths = [tmp_path / f"s{i}.bin" for i in range(4)]
    write_case(paths[0], level0(40))
    c1 = level0(30, seed=synth.SEED0 + 19)
    write_case(paths[1], c1, dds=[])
    write_case(paths[2], dd_chain(9, synth.SEED0 + 70))
    write_case(paths[3], level0(25, seed=synth.SEED0 + 17, outer_pass=3))
    fresh = [sc.run_driver(exe, "device", [p])[0] for p in paths]
    assert [f["dd_launches"] > 0 for f in fresh] == [True, False, True, True]
    assert fresh[1]["device_dd"] == 0 and fresh[1]["device_pose"] > 0
    for flags in ((), ("--use-pose", "--use-dd"), ("--preload-dd", "40")):
        seq = sc.run_driver(exe, "device", paths, *flags)
        assert len(seq) == 4
        for a, b in zip(seq, fresh):
            assert a["text"] == b["text"]
