"""The loop-closure oracle (oracle/loop/go_loop.cpp, oracle/pyoracle_loop.py) against independent formulations: its 3x3 Jacobi SVD
against LAPACK, umeyama on exact correspondences, every convergence exit of PCL's criteria, the candidate search and the cloud index
ranges against a numpy restatement, the whole ICP against a float64 Kabsch ICP on a scipy kd-tree, and its 1-NN against OpenCV's
bundled FLANN.  CPU only."""
import numpy as np
import pytest

from glio_b200 import synth


@pytest.fixture(scope="module")
def pl():
    from oracle import pyoracle_loop
    pyoracle_loop.build()
    return pyoracle_loop


def _moved(pts, yaw, t, roll=0.0, pitch=0.0):
    R = synth.quat_to_R(synth.quat_from_rpy(roll, pitch, yaw))
    return (np.asarray(pts, np.float64) @ R.T + np.asarray(t)).astype(np.float32), R


# ---- the Jacobi SVD --------------------------------------------------------------------------------------------------
def _svd_cases():
    rng = np.random.default_rng(3)
    cases = [rng.normal(size=(3, 3)) for _ in range(20)]
    cases += [np.diag([3.0, -1.0, 0.5]), np.diag([0.0, 2.0, 1.0])]
    u = rng.normal(size=3); v = rng.normal(size=3)
    cases.append(np.outer(u, v))                                                # rank 1
    cases.append(np.outer(u, v) + np.outer(rng.normal(size=3), rng.normal(size=3)))   # rank 2
    cases.append(np.zeros((3, 3)))
    R = synth.quat_to_R(synth.quat_from_rpy(0.3, -0.2, 1.1))
    cases.append(R @ np.diag([1.0, 1.0, -1.0]))                                 # a reflection, det < 0
    cases.append(1e-3 * rng.normal(size=(3, 3)))
    return [np.asarray(c, np.float32) for c in cases]


@pytest.mark.parametrize("k", range(len(_svd_cases())))
def test_svd3_against_lapack(pl, k):
    A = _svd_cases()[k]
    U, S, V = pl.svd3(A)
    ref = np.linalg.svd(A.astype(np.float64), compute_uv=False)
    na = max(float(np.abs(A).max()), 1e-30)
    eps = np.finfo(np.float32).eps
    assert np.all(np.diff(S) <= 0), "sorted descending"
    assert np.all(S >= 0)
    assert np.max(np.abs(S - ref)) <= 16 * eps * na
    assert np.max(np.abs(U.T.astype(np.float64) @ U - np.eye(3))) <= 16 * eps
    assert np.max(np.abs(V.T.astype(np.float64) @ V - np.eye(3))) <= 16 * eps
    assert np.max(np.abs(U.astype(np.float64) @ np.diag(S) @ V.T - A)) <= 32 * eps * na


def test_umeyama_recovers_a_known_motion(pl):
    rng = np.random.default_rng(4)
    src = rng.uniform(-20.0, 20.0, (5000, 3)).astype(np.float32)
    for yaw, t in ((0.4, [1.0, -2.0, 0.5]), (-2.5, [10.0, 3.0, -1.0]), (0.0, [0.0, 0.0, 0.0])):
        dst, R = _moved(src, yaw, t, roll=0.05, pitch=-0.1)
        T = pl.umeyama(src, dst)
        assert np.max(np.abs(T[:3, :3] - R)) <= 2e-6
        assert np.max(np.abs(T[:3, 3] - t)) <= 2e-5
        assert np.array_equal(T[3], [0, 0, 0, 1])


def test_summation_order(pl):
    rng = np.random.default_rng(5)
    for n in (0, 1, 63, 64, 65, 4095, 4096, 4097, 300_000):
        v = rng.normal(size=n).astype(np.float32)
        l0 = []
        for r in range(0, n, 64):
            a = np.float32(0)
            for x in v[r:r + 64]:
                a = np.float32(a + x)
            l0.append(a)
        l1 = []
        for r in range(0, len(l0), 64):
            a = np.float32(0)
            for x in l0[r:r + 64]:
                a = np.float32(a + x)
            l1.append(a)
        a = np.float32(0)
        for x in l1:
            a = np.float32(a + x)
        assert pl.hsum(v) == a
        assert abs(pl.hsum(v.astype(np.float64)) - float(np.sum(v.astype(np.float64)))) <= 1e-9 * max(1.0, n)


# ---- convergence exits -------------------------------------------------------------------------------------------
def test_every_convergence_exit(pl):
    rng = np.random.default_rng(21)
    cube = rng.uniform(-5.0, 5.0, (800, 3)).astype(np.float32)
    r = pl.icp(cube.copy(), cube)
    assert (r["converged"], r["state"], r["iterations"]) == (True, pl.TRANSFORM, 1)
    r = pl.icp(cube.copy(), cube, transformation_epsilon=0.0, euclidean_fitness_epsilon=0.0)
    assert (r["converged"], r["state"]) == (True, pl.ABS_MSE)
    rng = np.random.default_rng(22)
    sc = synth.Scene(-30.0, 30.0, rng)
    tgt = sc.sample(5000, rng, -20.0, 20.0).astype(np.float32)
    src, _ = _moved(sc.sample(2000, rng, -15.0, 15.0), 0.02, [0.4, 0.1, 0.0])
    r = pl.icp(src, tgt, transformation_epsilon=0.0, euclidean_fitness_epsilon=1e-3)
    assert (r["converged"], r["state"]) == (True, pl.REL_MSE) and r["iterations"] > 2
    r = pl.icp(src, tgt, max_iterations=3)
    assert (r["converged"], r["state"], r["iterations"]) == (True, pl.ITERATIONS, 3)
    far = (src + np.float32(100.0)).astype(np.float32)
    r = pl.icp(far, tgt)
    assert (r["converged"], r["state"], r["iterations"]) == (False, pl.NO_CORRESPONDENCES, 0)
    assert r["fitness"] > 900.0
    r = pl.icp(src[:0], tgt)
    assert r["state"] == pl.NO_CORRESPONDENCES and r["fitness"] == np.finfo(np.float64).max
    # the log: one record per iteration, MSE = double mean of the float distances, the transforms compose to final
    r = pl.icp(src, tgt)
    F = np.eye(4, dtype=np.float64)
    for T, n, mse in r["log"]:
        F = T.astype(np.float64) @ F
        assert 3 <= n <= len(src) and mse >= 0.0
    assert np.max(np.abs(F - r["final"])) <= 1e-5
    q, m, d = r["corr"]
    assert np.all(np.diff(q) > 0) and np.all(d <= 900.0)


# ---- detection ----------------------------------------------------------------------------------------------------
def _np_detect(pos, times, sel, t_new, radius, time_thres):
    p = np.asarray(pos, np.float32); s = np.asarray(sel, np.float32)
    dd = np.zeros(len(p), np.float32)                                # ((0 + dx^2) + dy^2) + dz^2 in float
    for a in range(3):
        dd = (dd + (s[a] - p[:, a]) * (s[a] - p[:, a])).astype(np.float32)
    hit = np.nonzero(dd < np.float32(radius * radius))[0]
    order = hit[np.lexsort((hit, dd[hit]))]
    for k in order:
        if abs(times[k] - t_new) > time_thres:
            return int(k), order
    return -1, order


def test_detection_against_numpy(pl):
    rng = np.random.default_rng(30)
    K = 400
    pos = rng.uniform(-40.0, 40.0, (K, 3)).astype(np.float32)
    pos[50] = pos[60]                                               # a tie in distance: index order
    times = np.sort(rng.uniform(0.0, 300.0, K))
    for i in range(200):
        sel = rng.uniform(-40.0, 40.0, 3).astype(np.float32)
        if i % 7 == 0:
            sel = pos[50].copy()
        t_new = float(rng.uniform(0.0, 300.0))
        for radius, thr in ((25.0, 30.0), (7.0, 30.0), (25.0, 0.0), (40.0, 1000.0)):
            c, order = pl.detect(pos, times, sel, t_new, radius, thr)
            c2, order2 = _np_detect(pos, times, sel, t_new, radius, thr)
            assert c == c2 and np.array_equal(order, order2)


def test_loop_oracle_rules_and_index_clipping(pl):
    # keyframe k has 20 + k points: the concatenated sizes tell which keyframes a cloud holds
    rng = np.random.default_rng(31)
    K = 40
    L = pl.LoopOracle(lc_map_width=3)
    for k in range(K):
        L.add_keyframe(rng.uniform(-1.0, 1.0, (20 + k, 3)), [0.5 * k, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0], 10.0 * k)
    size = lambda ids: sum(20 + k for k in ids)                                     # noqa: E731
    # a candidate at index 0: the history window is clipped below
    r = L.step(np.array([0.0, 0.0, 0.0], np.float32), 10.0 * 34)
    assert r["detected"] and r["closest_his_idx"] == 0 and r["latest_frame_idx"] == K - 5
    assert r["n_his"] == size(range(0, 4)) and r["n_latest"] == size(range(K - 5 - 5, K - 5 + 1))
    # the 0.2 s rule: a candidate less than 0.2 s from the last accepted loop is not registered
    L.time_last_loop = 500.0
    r2 = L.step(np.array([0.0, 0.0, 0.0], np.float32), 500.1)
    assert r2["closest_his_idx"] == 0 and not r2["detected"] and r2["icp"] is None
    r2 = L.step(np.array([0.0, 0.0, 0.0], np.float32), 500.3)
    assert r2["closest_his_idx"] == 0 and r2["detected"]
    # the time threshold skips recent neighbours: the nearest keyframe that is old enough wins
    r3 = L.step(np.array([10.0, 0.0, 0.0], np.float32), 10.0 * 22)
    assert r3["closest_his_idx"] == 18          # keyframe 20 is at distance 0, 19 / 21 / 22 are younger than 30 s
    # fewer than six keyframes: negative indices skipped; fewer than slide_window_width: both clouds empty
    S = pl.LoopOracle(lc_time_thres=0.5)
    for k in range(7):
        S.add_keyframe(rng.uniform(-1.0, 1.0, (20 + k, 3)), [0.5 * k, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0], 10.0 * k)
    r = S.step(np.array([0.0, 0.0, 0.0], np.float32), 10.0 * 6)
    assert r["detected"] and r["latest_frame_idx"] == 2 and r["n_latest"] == size([2, 1, 0]) and r["n_his"] == size([0, 1, 2])
    T = pl.LoopOracle(lc_time_thres=0.5)
    for k in range(3):
        T.add_keyframe(rng.uniform(-1.0, 1.0, (20, 3)), [0.5 * k, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0], 10.0 * k)
    r = T.step(np.array([0.0, 0.0, 0.0], np.float32), 10.0 * 2)
    assert r["detected"] and r["latest_frame_idx"] == -2 and r["n_latest"] == 0 and r["n_his"] == 0
    assert r["icp"]["state"] == pl.NO_CORRESPONDENCES and not r["accepted"]


def test_pose_arithmetic(pl):
    for rpy in ((0.1, -0.2, 0.3), (0.0, 0.0, np.pi), (np.pi - 1e-3, 0.2, -0.4), (0.0, 0.0, 0.0)):
        q = synth.quat_from_rpy(*rpy)
        qq = pl.quat_from_R(synth.quat_to_R(q))
        assert min(np.max(np.abs(np.array(qq) - q)), np.max(np.abs(np.array(qq) + q))) <= 1e-12
    F = np.eye(4, dtype=np.float32); F[:3, :3] = synth.quat_to_R(synth.quat_from_rpy(0.0, 0.0, 0.1)); F[:3, 3] = [1.0, 2.0, 0.5]
    latest = np.array([3.0, -1.0, 0.2, *synth.quat_from_rpy(0.0, 0.0, 0.5)])
    pf = pl.pose_from(F, latest)
    assert np.allclose(pf[:3], F[:3, :3].astype(np.float64) @ latest[:3] + F[:3, 3], atol=1e-6)
    assert np.allclose(synth.quat_to_R(pf[3:]), F[:3, :3].astype(np.float64) @ synth.quat_to_R(latest[3:]), atol=1e-6)


# ---- the whole ICP against an independent implementation ---------------------------------------------------------------
def _kabsch_icp(src, tgt, iters=100):
    from scipy.spatial import cKDTree
    tree = cKDTree(tgt.astype(np.float64))
    cur = src.astype(np.float64)
    F = np.eye(4)
    for _ in range(iters):
        d, j = tree.query(cur)
        keep = d * d <= 900.0
        a = cur[keep]; b = tgt[j[keep]].astype(np.float64)
        ma, mb = a.mean(0), b.mean(0)
        U, _, Vt = np.linalg.svd((b - mb).T @ (a - ma))
        S = np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))])
        R = U @ S @ Vt
        t = mb - R @ ma
        cur = cur @ R.T + t
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t
        F = T @ F
        if np.linalg.norm(t) < 1e-7 and abs(np.trace(R) - 3) < 1e-10:
            break
    return F


def test_icp_against_an_independent_float64_icp(pl):
    """a well-conditioned pair: a volume of points and a moved subset of it; both ICPs must land on the inverse of the motion"""
    rng = np.random.default_rng(40)
    tgt = rng.uniform(-10.0, 10.0, (20000, 3)).astype(np.float32)
    t = np.array([0.4, -0.3, 0.2])
    src, R = _moved(tgt[rng.choice(len(tgt), 4000, replace=False)], 0.06, t, roll=0.02, pitch=-0.03)
    Ti = np.eye(4); Ti[:3, :3] = R.T; Ti[:3, 3] = -R.T @ t
    r = pl.icp(src, tgt)
    F = _kabsch_icp(src, tgt)
    assert r["converged"]
    for M in (r["final"].astype(np.float64), F):
        assert np.max(np.abs(M[:3, :3] - Ti[:3, :3])) <= 1e-5
        assert np.max(np.abs(M[:3, 3] - Ti[:3, 3])) <= 1e-4
    assert r["fitness"] < 1e-9


# ---- the 1-NN against FLANN ---------------------------------------------------------------------------------------
def test_nn_matches_flann_kdtree_single_and_linear(pl):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(50)
    sc = synth.Scene(-30.0, 30.0, rng)
    tgt = sc.sample(40000, rng, -25.0, 25.0).astype(np.float32)
    qry, _ = _moved(sc.sample(5000, rng, -25.0, 25.0), 0.05, [0.3, 0.2, -0.1])
    qry = np.concatenate([qry, (rng.uniform(-1, 1, (200, 3)) + [60.0, 0.0, 0.0]).astype(np.float32)])   # outside the bounding box
    idx, d = pl.nn(tgt, qry)
    for algo, prm in ((4, dict(algorithm=4, leaf_max_size=15)), (0, dict(algorithm=0))):
        index = cv2.flann_Index(tgt, prm)
        fi, fd = index.knnSearch(qry, 1, params=dict(checks=-1, eps=0.0, sorted=True))
        assert np.array_equal(fi[:, 0].astype(np.int32), idx), f"1-NN indices differ from FLANN algorithm {algo}"
        assert np.array_equal(fd[:, 0].astype(np.float32), d), f"1-NN distances differ from FLANN algorithm {algo}"
