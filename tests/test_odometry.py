"""The front end's LidarOdometry node (GLIO/src/LidarOdometry.cpp:661-695) as the CPU oracle restates it: its state machine on
hand-made cases, its arithmetic against independent numpy formulations, and a seeded 40-sweep drive through
prepare -> features -> odometry that must track the ground truth.  No GPU."""
import math

import numpy as np
import pytest

from glio_b200 import synth


@pytest.fixture(scope="module")
def od(oracle):
    from oracle import pyoracle_odom
    return pyoracle_odom


def _plane_cloud(n, rng, intensity=5.05):
    """Points on three orthogonal planes (a corner), float32 x,y,z,intensity: a map the matcher can lock onto."""
    k = n // 3
    a = rng.uniform(-4, 4, (k, 2))
    pts = np.concatenate([np.c_[a[:, 0] + 6, a[:, 1], np.full(k, -1.5)],          # floor
                          np.c_[np.full(k, 10.0), a[:, 0], a[:, 1] + 1],           # wall x = 10
                          np.c_[a[:, 0] + 6, np.full(k, 5.0), a[:, 1] + 1]])        # wall y = 5
    pts += rng.uniform(-1e-3, 1e-3, pts.shape)
    return np.c_[pts, np.full(len(pts), intensity)].astype(np.float32)


def test_keyframe_truth_table(od):
    I = (1.0, 0.0, 0.0, 0.0)
    far, near = (0.3, 0.0, 0.0), (0.1, 0.0, 0.0)
    turned = tuple(synth.quat_from_rotvec(np.array([0, 0, 0.15])))
    # (t_cur, q_cur, size, kf_num) -> expected, with the literal precedence
    cases = [((near, I, 5, 4), False),        # small motion, 1 sweep since the keyframe
             ((far, I, 5, 4), False),         # moved, but size - kf_num = 1 is not > 1
             ((far, I, 6, 4), True),          # moved and size - kf_num = 2 > 1
             ((near, turned, 6, 4), True),    # turned by 0.15 rad > 0.1
             ((near, I, 6, 4), False),        # neither moved nor turned, size - kf_num = 2 is not > 2
             ((near, I, 7, 4), True),         # size - kf_num = 3 > 2 whatever the motion
             ((near, I, 1, 0), True),         # size <= 1
             ((far, I, 2, 1), False)]         # size 2 is not <= 1 and 2 - 1 is not > 1
    for (t, q, size, kfn), want in cases:
        assert od.keyframe_rule(t, q, (0.0, 0.0, 0.0), I, size, kfn) is want, (t, q, size, kfn)
    # a rounding-induced w above 1: acos gives NaN and NaN > 0.1 is false - only the distance can make it a keyframe
    q_big = (1.0 + 2.0 ** -52, 0.0, 0.0, 0.0)
    w = od.quat_mul(od.quat_inverse(I), q_big)[0]
    assert w > 1.0
    assert od.keyframe_rule(near, q_big, (0.0, 0.0, 0.0), I, 6, 4) is False
    assert od.keyframe_rule(far, q_big, (0.0, 0.0, 0.0), I, 6, 4) is True


def test_eigen_inverse_divides_by_squared_norm(od):
    q = (2.0, 0.0, 0.0, 0.0)                         # not unit: inverse is conj / 4, not conj
    assert od.quat_inverse(q) == (0.5, -0.0, -0.0, -0.0)
    q = (0.3, -0.2, 0.5, 0.7)
    n2 = ((q[1] * q[1] + q[2] * q[2]) + q[3] * q[3]) + q[0] * q[0]
    assert od.quat_inverse(q) == (q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2)
    assert od.quat_inverse((0.0, 0.0, 0.0, 0.0)) == (0.0, 0.0, 0.0, 0.0)
    # computeRelative uses it: with a non-unit previous quaternion (0, 0, 0, 2) the relative pose differs from the conjugate's
    p1 = (0.0, 0.0, 0.0, 2.0, 1.0, 2.0, 3.0); p2 = (0.0, 0.0, 0.0, 2.0, 2.0, 2.0, 3.0)
    r = od.relative(p1, p2)
    assert r[:4] == (4.0 / 4.0, 0.0, 0.0, 0.0) and r[4:] == (0.5, 0.0, 0.0)   # the conjugate alone would give w = 4, x = -7


def test_unify_quaternion(od):
    assert od.unify_quaternion((-0.5, 0.5, -0.5, 0.5)) == (0.5, -0.5, 0.5, -0.5)
    assert od.unify_quaternion((0.0, -1.0, 0.0, 0.0)) == (0.0, -1.0, 0.0, 0.0)      # w >= 0 is kept as it is


def test_prediction_and_relative_against_numpy(od):
    rng = np.random.default_rng(5)
    for _ in range(50):
        q0 = synth.quat_from_rotvec(rng.normal(0, 0.5, 3)); t0 = rng.normal(0, 10, 3)
        dq = synth.quat_from_rotvec(rng.normal(0, 0.05, 3)); dt = rng.normal(0, 0.5, 3)
        p = od.predict(tuple(q0) + tuple(t0), tuple(dq) + tuple(dt))
        assert np.allclose(p[4:], synth.quat_to_R(q0) @ dt + t0, rtol=0, atol=1e-12)
        assert np.allclose(p[:4], synth.quat_mul(q0, dq), rtol=0, atol=1e-15)
        r = od.relative(tuple(q0) + tuple(t0), p)
        assert np.allclose(r[:4], dq, atol=1e-12) and np.allclose(r[4:], dt, atol=1e-10)


def test_deskew_against_numpy(od):
    rng = np.random.default_rng(6)
    c = np.c_[rng.normal(0, 20, (5000, 3)), rng.integers(0, 32, 5000) + rng.uniform(0, 0.12, 5000)].astype(np.float32)
    trans = rng.normal(0, 0.5, 3)
    got = od.deskew(c, trans)
    frac = np.array([np.float32(v - np.float32(int(v))) for v in c[:, 3]], np.float64)
    ratio = np.minimum(frac / 0.1, 1.0)
    want = (c[:, :3].astype(np.float64) + ratio[:, None] * trans[None, :]).astype(np.float32)
    assert np.array_equal(got[:, :3], want) and np.array_equal(got[:, 3], c[:, 3])
    assert (ratio == 1.0).any() and (ratio < 1.0).any()


def test_first_sweeps_quirks(od):
    rng = np.random.default_rng(7)
    o = od.OdometryOracle()
    c1 = _plane_cloud(3000, rng)
    full = _plane_cloud(6000, rng, 3.02)
    r1 = o.step(c1, full)
    # sweep 1: clouds pass through, no odometry, an EMPTY scan frame saved with the identity pose
    assert r1["initialised"] and not r1["rounds"] and np.array_equal(r1["surf"], c1) and np.array_equal(r1["full"], full)
    assert len(o.surf_frames) == 1 and len(o.surf_frames[0]) == 0 and o.pose_info[0] == (1.0, 0, 0, 0, 0, 0, 0)
    # sweep 2: the map is the sweep's own surf cloud (scan frame) filtered, 8 rounds, always a keyframe
    c2 = _plane_cloud(3000, rng)
    r2 = o.step(c2, full)
    assert len(r2["rounds"]) == 8 and r2["keyframe"] and np.array_equal(r2["map"], od.voxel(c2[:, :3]))
    assert all(rd["n_match"] > 500 for rd in r2["rounds"])
    assert np.max(np.abs(r2["pose"][:3])) < 1e-3                      # matched against itself
    # sweep 3: the map is sweep 2's filtered scan moved by sweep 2's final pose (sweep 1's empty frame never enters)
    r3 = o.step(_plane_cloud(3000, rng))
    assert len(o.recent) == 1 and len(r3["rounds"]) == 1
    p = o.pose_info[1]
    from oracle import pyoracle as po
    assert np.array_equal(r3["map"], od.voxel(po.transform_points(r2["scan"], p[4:], p[:4])))


def test_twenty_sweep_window(od):
    rng = np.random.default_rng(8)
    o = od.OdometryOracle()
    base = _plane_cloud(1500, rng)
    for k in range(26):
        o.step(base + np.float32(rng.uniform(-1e-3, 1e-3, base.shape)) * np.array([1, 1, 1, 0], np.float32))
        assert len(o.recent) == min(max(k - 1, 0), 20)
    # the window holds the last 20 SWEEPS (latest_frame_idx changes every sweep), keyframe or not
    assert o.latest_frame_idx == len(o.pose_info) - 2


def test_small_map_keeps_prediction_and_kf(od):
    rng = np.random.default_rng(9)
    o = od.OdometryOracle()
    o.step(_plane_cloud(3000, rng))
    r = o.step(_plane_cloud(3000, rng))
    assert r["keyframe"]
    o.rel_pose = (1.0, 0.0, 0.0, 0.0, 0.3, 0.0, 0.0)                 # a motion to predict with
    pred = od.predict(o.abs_pose, o.rel_pose)
    o.recent.clear(); o.surf_frames[-1] = np.zeros((0, 3), np.float32)   # next map: an empty previous scan -> fewer than 10 points
    r = o.step(np.zeros((0, 4), np.float32))
    assert r["skipped"] and not r["rounds"] and r["n_map"] < 10
    assert tuple(r["pose"][3:]) + tuple(r["pose"][:3]) == pred      # the prediction stands
    assert r["keyframe"]                                             # kf keeps its previous value (true)


def test_zero_matches_keep_pose(od):
    rng = np.random.default_rng(10)
    o = od.OdometryOracle()
    o.step(_plane_cloud(3000, rng)); o.step(_plane_cloud(3000, rng))
    far = _plane_cloud(3000, rng); far[:, :3] += np.float32(500.0)    # nothing within the 1 m gate
    before = od.predict(o.abs_pose, o.rel_pose)
    r = o.step(far)
    assert [rd["n_match"] for rd in r["rounds"]] == [0] and r["rounds"][0]["message"] == od.NO_BLOCKS
    assert tuple(r["pose"][3:]) + tuple(r["pose"][:3]) == before


@pytest.fixture(scope="module")
def drive_run(od):
    """The 40-sweep seeded drive through the CPU chain: scan preparation -> feature extraction -> odometry."""
    from oracle import pyoracle as po, pyoracle_scanprep as ps
    D = synth.raw_drive(40)
    st = ps.ImuState(); o = od.OdometryOracle()
    out = []
    for k in range(40):
        q = ps.imu_sweep_rotation(st, D["stamps"], D["gyro"], D["t_scan_next"][k])
        p = ps.prepare_scan(D["sweeps"][k], 32, q_imu=q, q_lb=synth.Q_LB)
        f = po.extract_features(p["cloud"], p["scan_start"], p["scan_end"], 1, 1.0, 0.1, 0.4)
        out.append(o.step(f["less_flat_ds"], p["cloud"]))
    return D, out


def test_drive_tracks_ground_truth(drive_run):
    D, res = drive_run
    T = D["poses"]
    terr, yerr = [], []
    for k in range(3, 40):              # sweep 2 starts from a zero-motion prediction (rel_pose of sweep 1 is the identity)
        dp = synth.quat_to_R(T[k - 1, 3:]).T @ (T[k, :3] - T[k - 1, :3])
        dyaw = 2 * math.atan2(T[k, 6], T[k, 3]) - 2 * math.atan2(T[k - 1, 6], T[k - 1, 3])
        rel = res[k]["rel_pose"]
        terr.append(np.linalg.norm(rel[:3] - dp)); yerr.append(abs(2 * math.atan2(rel[6], rel[3]) - dyaw))
    # Bars from an oracle run of this drive (0.5 m per sweep at 5 m/s; the translation inside a sweep is not de-skewed): the worst
    # per-sweep translation error was 0.0077 m and the worst yaw error 5.3e-5 rad, with 13 keyframes and at least 9230 matches per
    # round.  The bars allow about 2x the errors: a regression that loses the track breaks them by orders of magnitude.
    assert max(terr) < 0.015 and max(yerr) < 1e-4, (max(terr), max(yerr))
    assert sum(r["keyframe"] for r in res) >= 8                          # keyframes occur
    assert all(rd["n_match"] >= 300 for r in res[1:] for rd in r["rounds"])   # every round has hundreds of matches
    assert all(len(r["rounds"]) == (8 if k == 1 else 1) for k, r in enumerate(res[1:], 1))
