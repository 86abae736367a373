"""Seeded synthetic workloads for the LiDAR hot path (SURVEY.md §8(d) "Synthetic inputs").

Street-canyon scene in a world frame with no surface through the origin (avoids the n·x = -1
singularity of the reference plane model, quirk Q2): ground z = -1.8, walls y = ±12,
cross walls every 40 m in x (offset so none passes through x = 0), random boxes.  Points are sampled
uniformly by area + N(0, 0.02 m) along the surface normal + U(-1e-3, 1e-3) jitter (kills kNN distance
ties).  All coordinates are float32, as the reference's pcl::PointXYZI clouds are.

Pure numpy; this is a workload generator, not part of the device path.
"""
import numpy as np

Q_LB = np.array([1.0, 0.0, 0.0, 0.0])          # GLIO/config/config_urban_hk.yaml:90-93
T_LB = np.array([0.0, 0.0, 0.28])              # GLIO/config/config_urban_hk.yaml:94-97
SEED0 = 20260923


def quat_mul(a, b):
    w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3]
    x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2]
    y = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3]
    z = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]
    return np.array([w, x, y, z])


def quat_conj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def quat_to_R(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def quat_from_rpy(roll, pitch, yaw):
    cr, sr = np.cos(roll / 2), np.sin(roll / 2)
    cp, sp = np.cos(pitch / 2), np.sin(pitch / 2)
    cy, sy = np.cos(yaw / 2), np.sin(yaw / 2)
    return np.array([cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy,
                     cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy])


def quat_from_rotvec(v):
    a = np.linalg.norm(v)
    if a < 1e-300:
        return np.array([1.0, 0, 0, 0])
    return np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * v / a])


def lidar_pose_in_world(t, q, q_lb=Q_LB, t_lb=T_LB):
    """Q2 = Q * q_lb^-1 ; T2 = T - Q2 * t_lb     (GLIO/src/Estimator.cpp:2216-2217)."""
    q2 = quat_mul(q, quat_conj(q_lb) / np.dot(q_lb, q_lb))
    t2 = t - quat_to_R(q2) @ t_lb
    return t2, q2


class Scene:
    """A set of rectangles: origin o, edge vectors u, v (so area = |u x v|), unit normal n."""

    def __init__(self, x_min, x_max, rng, n_boxes=30, wall_h=14.0):
        rects = []
        L = x_max - x_min
        zg = -1.8
        rects.append(([x_min, -12, zg], [L, 0, 0], [0, 24, 0]))                      # ground
        rects.append(([x_min, -12, zg], [L, 0, 0], [0, 0, wall_h]))                  # wall y=-12
        rects.append(([x_min, 12, zg], [L, 0, 0], [0, 0, wall_h]))                   # wall y=+12
        x = np.floor(x_min / 40.0) * 40.0 + 17.0
        while x < x_max:                                                             # cross walls (upper part only)
            if x > x_min:
                rects.append(([x, -12, zg + 4.0], [0, 24, 0], [0, 0, wall_h - 4.0]))
            x += 40.0
        nb = max(1, int(round(n_boxes * L / 140.0)))
        for _ in range(nb):
            sx, sy, sz = rng.uniform(1.0, 4.0, 3)
            cx = rng.uniform(x_min, x_max - sx)
            if rng.random() < 0.5:                                                   # keep the driving lane free
                cy = rng.uniform(4.0, 11.0 - sy)
            else:
                cy = rng.uniform(-11.0, -4.0 - sy)
            o = np.array([cx, cy, zg])
            rects.append((o + [0, 0, sz], [sx, 0, 0], [0, sy, 0]))                   # top
            rects.append((o, [sx, 0, 0], [0, 0, sz]))
            rects.append((o + [0, sy, 0], [sx, 0, 0], [0, 0, sz]))
            rects.append((o, [0, sy, 0], [0, 0, sz]))
            rects.append((o + [sx, 0, 0], [0, sy, 0], [0, 0, sz]))
        self.o = np.array([r[0] for r in rects], float)
        self.u = np.array([r[1] for r in rects], float)
        self.v = np.array([r[2] for r in rects], float)
        nrm = np.cross(self.u, self.v)
        self.area = np.linalg.norm(nrm, axis=1)
        self.n = nrm / self.area[:, None]

    def sample(self, n, rng, x_lo=None, x_hi=None, noise=0.02, jitter=1e-3):
        """n points, uniform by area, restricted to x in [x_lo, x_hi] (rectangles are clipped along x)."""
        o, u, v, area = self.o.copy(), self.u.copy(), self.v.copy(), self.area.copy()
        if x_lo is not None:
            # clip the x-extent of rectangles whose u edge is along x; drop others outside
            along = np.abs(u[:, 0]) > 0
            x0 = o[:, 0]; x1 = o[:, 0] + u[:, 0]
            nx0 = np.clip(x0, x_lo, x_hi); nx1 = np.clip(x1, x_lo, x_hi)
            keep = np.where(along, nx1 > nx0, (x0 >= x_lo) & (x0 <= x_hi))
            frac = np.where(along, (nx1 - nx0) / np.where(along, u[:, 0], 1.0), 1.0)
            o[:, 0] = np.where(along, nx0, o[:, 0])
            u[:, 0] = np.where(along, nx1 - nx0, u[:, 0])
            area = area * frac * keep
        p = area / area.sum()
        ridx = rng.choice(len(area), size=n, p=p)
        a = rng.random(n)[:, None]; b = rng.random(n)[:, None]
        pts = o[ridx] + a * u[ridx] + b * v[ridx]
        pts += self.n[ridx] * rng.normal(0.0, noise, n)[:, None]
        pts += rng.uniform(-jitter, jitter, (n, 3))
        return pts


def trajectory(K, rng):
    """KF k at x = 1.0 k, y = 0.5 sin(0.1 k), z = 0, yaw = 0.02 sin(0.05 k), roll/pitch ~ N(0, 0.2 deg)."""
    poses = np.zeros((K, 7))
    for k in range(K):
        poses[k, :3] = [1.0 * k, 0.5 * np.sin(0.1 * k), 0.0]
        r, p = rng.normal(0.0, np.deg2rad(0.2), 2)
        poses[k, 3:] = quat_from_rpy(r, p, 0.02 * np.sin(0.05 * k))
    return poses


def perturb(poses, rng, sig_t=0.05, sig_r_deg=0.5):
    """truth (+) N(0, 0.05 m), N(0, 0.5 deg)."""
    out = poses.copy()
    for k in range(len(poses)):
        out[k, :3] += rng.normal(0.0, sig_t, 3)
        dq = quat_from_rotvec(rng.normal(0.0, np.deg2rad(sig_r_deg), 3))
        q = quat_mul(dq, poses[k, 3:])
        out[k, 3:] = q / np.linalg.norm(q)
    return out


def scan_in_lidar_frame(scene, pose, Q, rng, rng_range=50.0, q_lb=Q_LB, t_lb=T_LB):
    t, q = pose[:3], pose[3:]
    pw = scene.sample(Q, rng, t[0] - rng_range, t[0] + rng_range)
    pb = (pw - t) @ quat_to_R(q)                 # R^T (pw - t)
    pl = pb @ quat_to_R(q_lb).T + t_lb           # p_l = q_lb p_b + t_lb
    return pl.astype(np.float32)


def scan_in_body_frame(scene, pose, Q, rng, rng_range=50.0):
    """Batch path applies body poses directly to the stored scan points (quirk Q7)."""
    t, q = pose[:3], pose[3:]
    pw = scene.sample(Q, rng, t[0] - rng_range, t[0] + rng_range)
    return ((pw - t) @ quat_to_R(q)).astype(np.float32)


def window_problem(W=20, Q=100_000, M=1_000_000, seed=SEED0 + 2, n_boxes=30):
    """cfg 1 / cfg 2 / cfg 5 style sliding-window problem."""
    rng = np.random.default_rng(seed)
    scene = Scene(-60.0, W + 60.0, rng, n_boxes=n_boxes)
    truth = trajectory(W, rng)
    init = perturb(truth, rng)
    map_xyz = scene.sample(M, rng, -55.0, W + 55.0).astype(np.float32)
    scans = [scan_in_lidar_frame(scene, truth[k], Q, rng) for k in range(W)]
    return dict(map_xyz=map_xyz, scans=scans, poses_true=truth, poses_init=init, q_lb=Q_LB.copy(),
                t_lb=T_LB.copy(), W=W, Q=Q, M=M, seed=seed)


def corner_sample(scene, n, rng, x_lo=None, x_hi=None, noise=0.02, jitter=1e-3):
    """n corner points of the scene: uniform by length on the edges of its rectangles (the wall-ground lines, the cross walls'
    and the boxes' edges), restricted to x in [x_lo, x_hi], + N(0, noise) per axis + U(-jitter, jitter) (kills kNN ties)."""
    a = np.concatenate([scene.o, scene.o, scene.o + scene.u, scene.o + scene.v])
    d = np.concatenate([scene.u, scene.v, scene.v, scene.u])
    s0 = np.zeros(len(a)); s1 = np.ones(len(a))
    if x_lo is not None:
        along = d[:, 0] != 0
        dx = np.where(along, d[:, 0], 1.0)
        e0 = (x_lo - a[:, 0]) / dx; e1 = (x_hi - a[:, 0]) / dx
        s0 = np.where(along, np.maximum(0.0, np.minimum(e0, e1)), 0.0)
        s1 = np.where(along, np.minimum(1.0, np.maximum(e0, e1)), 1.0)
        inside = (a[:, 0] >= x_lo) & (a[:, 0] <= x_hi)
        s1 = np.where(along | inside, s1, 0.0)
    length = np.linalg.norm(d, axis=1) * np.maximum(s1 - s0, 0.0)
    idx = rng.choice(len(a), size=n, p=length / length.sum())
    s = s0[idx] + rng.random(n) * (s1[idx] - s0[idx])
    pts = a[idx] + s[:, None] * d[idx]
    pts += rng.normal(0.0, noise, (n, 3))
    pts += rng.uniform(-jitter, jitter, (n, 3))
    return pts


def window_edge_problem(W=20, Q=10_000, M=200_000, seed=SEED0 + 15, n_boxes=30, noise=0.02):
    """The corner counterpart of window_problem: a corner map of M points and W corner scans of Q points each (lidar frame of
    the true poses, range 50 m), e.g. for glio_window_associate_edges."""
    rng = np.random.default_rng(seed)
    scene = Scene(-60.0, W + 60.0, rng, n_boxes=n_boxes)
    truth = trajectory(W, rng)
    init = perturb(truth, rng)
    map_xyz = corner_sample(scene, M, rng, -55.0, W + 55.0, noise=noise).astype(np.float32)
    scans = []
    for k in range(W):
        t, q = truth[k, :3], truth[k, 3:]
        pw = corner_sample(scene, Q, rng, t[0] - 50.0, t[0] + 50.0, noise=noise)
        pb = (pw - t) @ quat_to_R(q)
        scans.append((pb @ quat_to_R(Q_LB).T + T_LB).astype(np.float32))
    return dict(map_xyz=map_xyz, scans=scans, poses_true=truth, poses_init=init, q_lb=Q_LB.copy(), t_lb=T_LB.copy(), W=W, Q=Q, M=M,
                seed=seed)


def batch_problem(K=200, Q=100_000, seed=SEED0 + 3, search_range=6, rng_range=50.0, frames=None):
    """cfg 3 / cfg 4 style batch problem: K keyframes, scans in the body frame.  Every scan has its own RNG stream
    (seed, k), so a rank of a sharded run can generate only the frames it holds (`frames`) and still agree with the
    others; scans[k] is None for frames not requested."""
    rng = np.random.default_rng(seed)
    scene = Scene(-60.0, K + 60.0, rng)
    truth = trajectory(K, rng)
    init = perturb(truth, rng, sig_t=0.03, sig_r_deg=0.2)
    want = set(range(K)) if frames is None else set(int(f) for f in frames)
    scans = [scan_in_body_frame(scene, truth[k], Q, np.random.default_rng([seed, k]), rng_range) if k in want else None for k in range(K)]
    return dict(scans=scans, poses_true=truth, poses_init=init, K=K, Q=Q, search_range=search_range, seed=seed)


def batch_edge_problem(K=200, Q=10_000, seed=SEED0 + 3, search_range=6, frames=None, rng_range=50.0, noise=0.02):
    """The corner counterpart of batch_problem: the same scene and poses for the same (K, seed), and corner scans of Q points in the
    body frame (corner_sample within rng_range of the true pose), e.g. for glio_batch_set_edge_frame.  Every corner scan has its own
    RNG stream (seed, k, 1), so a rank generates only its frames (`frames`; dist.frames_needed gives the halo); corner_scans[k] is
    None for frames not requested."""
    rng = np.random.default_rng(seed)
    scene = Scene(-60.0, K + 60.0, rng)
    truth = trajectory(K, rng)
    init = perturb(truth, rng, sig_t=0.03, sig_r_deg=0.2)
    want = set(range(K)) if frames is None else set(int(f) for f in frames)
    scans = []
    for k in range(K):
        if k not in want:
            scans.append(None)
            continue
        t, q = truth[k, :3], truth[k, 3:]
        pw = corner_sample(scene, Q, np.random.default_rng([seed, k, 1]), t[0] - rng_range, t[0] + rng_range, noise=noise)
        scans.append(((pw - t) @ quat_to_R(q)).astype(np.float32))
    return dict(corner_scans=scans, poses_true=truth, poses_init=init, K=K, Q=Q, search_range=search_range, seed=seed)


def _unify(q):
    """unifyQuaternion: w >= 0."""
    return q if q[0] >= 0 else -q


def _qinv(q):
    return quat_conj(q) / np.dot(q, q)


def attitude_factors(kf, search_range, start_idx=0, end=None):
    """The delta_q_factor_auto list of optimizeBatchWithLandMark (Estimator.cpp:2831-2891, added at both fusion levels) over
    keyframe poses kf (K, 7) = (t, q w x y z), i.e. pose_info_keyframe: per i a backward and then a forward walk, each accepted j a
    factor (i, j, dq = unify(q_i)^-1 q_j).  p_range > 5 / search_range is integer division; p_tmp and factor_count carry over
    from the backward into the forward walk, which a full backward walk resets.  Returns (i, j, dq (n, 4))."""
    end = len(kf) if end is None else end
    thr = 5 // search_range
    I, J, DQ = [], [], []
    for i in range(start_idx, end):
        qi = _unify(kf[i, 3:]); p_tmp = kf[i, :3]
        count = 0
        for walk in (range(i, start_idx - 1, -1), range(i, end)):
            for j in walk:
                if count == search_range:
                    count = 0
                    break
                if j == i:
                    continue
                pj = kf[j, :3]
                if np.linalg.norm(p_tmp - pj) > thr:
                    p_tmp = pj
                    I.append(i); J.append(j); DQ.append(quat_mul(_qinv(qi), kf[j, 3:]))
                    count += 1
    return np.asarray(I, np.int32), np.asarray(J, np.int32), np.asarray(DQ, np.float64).reshape(-1, 4)


def relative_pose_factors(kf, search_range, start_idx=0, end=None):
    """The LidarPoseFactorBatchRelativeAutoDiff list of sms_fusion_level 0 (Estimator.cpp:2897-2954): two loops over
    ms_i = 1 .. search_range - 1, so interior pairs appear twice, always with i < j; dq = q_i^-1 q_j, dp = q_i^-1 (p_j - p_i).
    Returns (i, j, dq (n, 4), dp (n, 3))."""
    end = len(kf) if end is None else end
    pairs = [(idx - m, idx) for idx in range(start_idx + search_range, end) for m in range(1, search_range)]
    pairs += [(idx, idx + m) for idx in range(start_idx, end - search_range) for m in range(1, search_range)]
    I, J, DQ, DP = [], [], [], []
    for i, j in pairs:
        qinv = _qinv(kf[i, 3:])
        I.append(i); J.append(j); DQ.append(quat_mul(qinv, kf[j, 3:]))
        DP.append(quat_to_R(qinv) @ (kf[j, :3] - kf[i, :3]))
    return (np.asarray(I, np.int32), np.asarray(J, np.int32), np.asarray(DQ, np.float64).reshape(-1, 4),
            np.asarray(DP, np.float64).reshape(-1, 3))


def pose_graph_problem(K=200, seed=SEED0 + 16, search_range=6, level=0, sig_t=0.03, sig_r_deg=0.2):
    """The batch refinement's pose factors on a seeded trajectory.  kf: the keyframe poses the factors are measured from
    (pose_info_keyframe: truth + N(0, 0.01 m), N(0, 0.05 deg)); poses_init: the states (truth + N(0, sig_t), N(0, sig_r_deg)).
    level 0: the attitude factors, then the relative factors, in the Estimator's order, as columns i, j, kind, dq, dp (see
    api.pose_factor_records); level 1: the attitude factors alone, and the LiDAR pairs dist.batch_pairs(K, search_range)."""
    rng = np.random.default_rng(seed)
    truth = trajectory(K, rng)
    kf = perturb(truth, rng, sig_t=0.01, sig_r_deg=0.05)
    init = perturb(truth, rng, sig_t=sig_t, sig_r_deg=sig_r_deg)
    ai, aj, adq = attitude_factors(kf, search_range)
    if level == 0:
        ri, rj, rdq, rdp = relative_pose_factors(kf, search_range)
    else:
        ri, rj, rdq, rdp = (np.zeros(0, np.int32),) * 2 + (np.zeros((0, 4)), np.zeros((0, 3)))
    out = dict(K=K, poses_true=truth, kf=kf, poses_init=init, search_range=search_range, seed=seed, level=level,
               i=np.concatenate([ai, ri]), j=np.concatenate([aj, rj]),
               kind=np.concatenate([np.ones(len(ai), np.int32), np.zeros(len(ri), np.int32)]),
               dq=np.concatenate([adq, rdq]), dp=np.concatenate([np.zeros((len(ai), 3)), rdp]))
    if level == 1:
        from .dist import batch_pairs
        out["pairs"] = batch_pairs(K, search_range)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# IMU factors of the batch refinement at sms_fusion_level 1 (ImuFactor between consecutive keyframes, Estimator.cpp:2993-3001)
# ---------------------------------------------------------------------------------------------------------------------------
IMU_GRAVITY = np.array([0.0, 0.0, 9.81])


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _imu_factor_columns(T, kf_times, V, ba, bg, pairs, sig, rng):
    """The per-factor recipe of imu_problem for the keyframe pairs (i, j) of `pairs`, in order, at the true poses T, velocities V
    and biases ba, bg: the factor columns of api.imu_factor_records and the covariances (n x 15 x 15)."""
    n = len(pairs)
    cols = {k: [] for k in ("i", "j", "sum_dt", "delta_p", "delta_q", "delta_v", "linearized_ba", "linearized_bg", "dp_dba", "dp_dbg",
                            "dq_dbg", "dv_dba", "dv_dbg", "sqrt_info")}
    covs = []
    g = IMU_GRAVITY
    for i, j in pairs:
        dt = kf_times[j] - kf_times[i]
        qi, qj = T[i, 3:], T[j, 3:]
        Ri = quat_to_R(qi)
        lin_ba = ba[i] + rng.normal(0.0, 0.005, 3); lin_bg = bg[i] + rng.normal(0.0, 5e-4, 3)
        dp_dba = -0.5 * dt * dt * np.eye(3); dv_dba = -dt * np.eye(3); dq_dbg = -dt * np.eye(3)
        dp_dbg = dt * dt * _skew(rng.normal(0.0, 0.3, 3)); dv_dbg = dt * _skew(rng.normal(0.0, 0.5, 3))
        dba, dbg = ba[i] - lin_ba, bg[i] - lin_bg
        e = rng.normal(0.0, 1.0, 15) * sig
        dp = Ri.T @ (-0.5 * g * dt * dt + T[j, :3] - T[i, :3] - V[i] * dt) - dp_dba @ dba - dp_dbg @ dbg + e[:3]
        dv = Ri.T @ (-g * dt + V[j] - V[i]) - dv_dba @ dba - dv_dbg @ dbg + e[6:9]
        # delta_q deltaQ(dq_dbg dbg) = q_i^-1 q_j (x) exp(e_R / 2) up to normalisation
        dQ = np.concatenate([[1.0], 0.5 * (dq_dbg @ dbg)])
        target = quat_mul(quat_mul(quat_conj(qi), qj), quat_from_rotvec(e[3:6]))
        dq = quat_mul(target, quat_conj(dQ) / np.dot(dQ, dQ))
        dq /= np.linalg.norm(dq)
        C = rng.normal(0.0, 0.1, (15, 15)); C = 0.5 * (C + C.T); np.fill_diagonal(C, 1.0)
        w, U = np.linalg.eigh(C); C = U @ np.diag(np.maximum(w, 0.2)) @ U.T
        d = np.sqrt(np.diag(C)); C = C / np.outer(d, d)
        cov = np.outer(sig, sig) * C
        L = np.linalg.cholesky(np.linalg.inv(cov))
        for name, val in (("i", i), ("j", j), ("sum_dt", dt), ("delta_p", dp), ("delta_q", dq), ("delta_v", dv), ("linearized_ba", lin_ba),
                          ("linearized_bg", lin_bg), ("dp_dba", dp_dba), ("dp_dbg", dp_dbg), ("dq_dbg", dq_dbg), ("dv_dba", dv_dba),
                          ("dv_dbg", dv_dbg), ("sqrt_info", L.T)):
            cols[name].append(val)
        covs.append(cov)
    imu = {k: np.asarray(v, np.int32 if k in ("i", "j") else np.float64) for k, v in cols.items()}
    for k, shape in (("delta_p", (3,)), ("delta_q", (4,)), ("delta_v", (3,)), ("linearized_ba", (3,)), ("linearized_bg", (3,)),
                     ("dp_dba", (3, 3)), ("dp_dbg", (3, 3)), ("dq_dbg", (3, 3)), ("dv_dba", (3, 3)), ("dv_dbg", (3, 3)), ("sqrt_info", (15, 15))):
        imu[k] = imu[k].reshape((n,) + shape)
    imu["g_vec"] = np.broadcast_to(g, (n, 3)).copy()
    return imu, np.asarray(covs).reshape(n, 15, 15)


def imu_problem(K=200, seed=SEED0 + 18, search_range=6, sig_p=0.02, sig_r=0.005, sig_v=0.03, sig_ba=0.02, sig_bg=0.002):
    """A level-1-shaped batch problem with IMU factors.  This is generated data, not a pre-integration: no IMU samples are
    integrated.  pose_graph_problem(level=1)'s trajectory, attitude factors and LiDAR pairs; keyframe times 0.25 .. 0.45 s apart
    (as in dd_psr_problem); true velocities (central differences of the positions over the times) and slowly drifting biases
    (sb_true, K x 9: V, Ba, Bg); perturbed initial speed-bias states (sb_init).  One factor per consecutive pair (k, k+1), in
    order, with T = t_{k+1} - t_k, g = IMU_GRAVITY, linearisation biases off the truth by a little (so Bg_i != linearized_bg),
    first-order jacobian_ blocks (dp_dba = -T^2/2 I, dv_dba = -T I, dq_dbg = -T I, dp_dbg and dv_dbg of the order of T^2 and T
    times a small random rotation term), and deltas chosen so that the raw residual at the truth is N(0, sigma) noise.  The
    covariance is diag(sigma^2) with mild correlations (SPD), and sqrt_info = LLT(covariance^-1).matrixL()^T as ImuFactor forms it.
    Adds kf_times, sb_true, sb_init, cov (n x 15 x 15) and imu (the factor columns of api.imu_factor_records)."""
    P = pose_graph_problem(K=K, seed=seed, search_range=search_range, level=1)
    rng = np.random.default_rng([seed, 2])
    kf_times = 1_600_000_000.0 + np.concatenate([[0.0], np.cumsum(rng.uniform(0.25, 0.45, K - 1))])
    T = P["poses_true"]
    V = np.gradient(T[:, :3], kf_times, axis=0) if K > 1 else np.zeros((K, 3))
    ba = np.array([0.05, -0.03, 0.02]) + np.cumsum(rng.normal(0.0, 1e-4, (K, 3)), axis=0)
    bg = np.array([0.002, -0.001, 0.0015]) + np.cumsum(rng.normal(0.0, 1e-5, (K, 3)), axis=0)
    sb_true = np.concatenate([V, ba, bg], axis=1)
    sb_init = sb_true + np.concatenate([rng.normal(0.0, 0.1, (K, 3)), rng.normal(0.0, 0.01, (K, 3)), rng.normal(0.0, 1e-3, (K, 3))], axis=1)
    sig = np.concatenate([np.full(3, sig_p), np.full(3, sig_r), np.full(3, sig_v), np.full(3, sig_ba), np.full(3, sig_bg)])
    imu, cov = _imu_factor_columns(T, kf_times, V, ba, bg, [(k, k + 1) for k in range(K - 1)], sig, rng)
    P.update(kf_times=kf_times, sb_true=sb_true, sb_init=sb_init, cov=cov, imu=imu)
    return P


def window_imu_problem(W=20, Q=100_000, M=1_000_000, seed=SEED0 + 2, sig_p=0.02, sig_r=0.005, sig_v=0.03, sig_ba=0.02, sig_bg=0.002):
    """window_problem(W, Q, M, seed) plus the window's IMU chain: one factor per consecutive slot pair (k, k+1), in order, by
    imu_problem's per-factor recipe at the window's true poses.  Generated data, not a pre-integration.  Keyframe times 0.25 ..
    0.45 s apart, true velocities (central differences), slowly drifting biases (sb_true, W x 9: V, Ba, Bg) and perturbed initial
    speed-bias states (sb_init).  Adds kf_times, sb_true, sb_init, cov ((W-1) x 15 x 15) and imu (api.imu_factor_records columns)."""
    P = window_problem(W=W, Q=Q, M=M, seed=seed)
    rng = np.random.default_rng([seed, 3])
    kf_times = 1_600_000_000.0 + np.concatenate([[0.0], np.cumsum(rng.uniform(0.25, 0.45, W - 1))])
    T = P["poses_true"]
    V = np.gradient(T[:, :3], kf_times, axis=0) if W > 1 else np.zeros((W, 3))
    ba = np.array([0.05, -0.03, 0.02]) + np.cumsum(rng.normal(0.0, 1e-4, (W, 3)), axis=0)
    bg = np.array([0.002, -0.001, 0.0015]) + np.cumsum(rng.normal(0.0, 1e-5, (W, 3)), axis=0)
    sb_true = np.concatenate([V, ba, bg], axis=1)
    sb_init = sb_true + np.concatenate([rng.normal(0.0, 0.1, (W, 3)), rng.normal(0.0, 0.01, (W, 3)), rng.normal(0.0, 1e-3, (W, 3))], axis=1)
    sig = np.concatenate([np.full(3, sig_p), np.full(3, sig_r), np.full(3, sig_v), np.full(3, sig_ba), np.full(3, sig_bg)])
    imu, cov = _imu_factor_columns(T, kf_times, V, ba, bg, [(k, k + 1) for k in range(W - 1)], sig, rng)
    P.update(kf_times=kf_times, sb_true=sb_true, sb_init=sb_init, cov=cov, imu=imu)
    return P


# ---------------------------------------------------------------------------------------------------------------------------
# GNSS double-differenced pseudorange factors of the batch refinement (dd_psr_factor_20, Estimator.cpp:3086-3272)
# ---------------------------------------------------------------------------------------------------------------------------
WGS84_A, WGS84_E2 = 6378137.0, 6.69437999014e-3            # gnss_constant.hpp: EARTH_SEMI_MAJOR, EARTH_ECCE_2
_PI = 3.1415926535897932
_R2D, _D2R = 180.0 / _PI, _PI / 180.0
DD_PSR_THRESHOLDS = (1e9, 10.0, 8.0, 6.0)                   # DDpsr_threshold of the 4 outer passes (Estimator.cpp:2764-2765)
# one GNSS_Raw of an epoch: the PRN, the satellite's ECEF position, the raw pseudorange and the elevation seen by the receiver
GNSS_RAW_DTYPE = np.dtype([("prn", "<i4"), ("sat_pos", "<f8", (3,)), ("psr", "<f8"), ("elevation", "<f8")])


# the constellation of a PRN (gnss_tools.h:1116-1168, PRN 84 counts as GPS and as Galileo there) in the Estimator's order
def prn_is_gps(prn): return prn <= 32 or prn == 84
def prn_is_bds(prn): return 87 <= prn <= 121
def prn_is_glo(prn): return 32 < prn <= 56
def prn_is_gal(prn): return 56 < prn < 87


# (predicate, the pseudorange > 1000 check): prepareGPS/BDSDDPsrData check it, prepareGLO/GALDDPsrData do not
DD_PSR_SYSTEMS = ((prn_is_gps, True), (prn_is_bds, True), (prn_is_glo, False), (prn_is_gal, False))


def geo_to_ecef(lat_deg, lon_deg, h):
    lat, lon = np.deg2rad(lat_deg), np.deg2rad(lon_deg)
    N = WGS84_A / np.sqrt(1.0 - WGS84_E2 * np.sin(lat) ** 2)
    return np.array([(N + h) * np.cos(lat) * np.cos(lon), (N + h) * np.cos(lat) * np.sin(lon), (N * (1.0 - WGS84_E2) + h) * np.sin(lat)])


def ecef_local_rotation(anchor, yaw):
    """R_ecef_local = ecef2rotation(anchor) * R_enu_local(yaw), gnss_comm's closed form (gnss_utility.cpp:347-388, :738-753): Bowring's
    latitude, atan2 longitude (through degrees, as ecef2geo returns them), the ENU -> ECEF columns, times Rz(yaw)."""
    x, y, z = (float(v) for v in anchor)
    a, e2 = WGS84_A, WGS84_E2
    a2 = a * a; b2 = a2 * (1 - e2); b = np.sqrt(b2); ep2 = (a2 - b2) / b2
    p = np.hypot(x, y)
    s1, s2 = z * a, p * b
    h = np.sqrt(s1 * s1 + s2 * s2)
    sin_t, cos_t = s1 / h, s2 / h
    s1 = z + ep2 * b * sin_t ** 3
    s2 = p - a * e2 * cos_t ** 3
    lat = np.arctan(s1 / s2) * _R2D * _D2R
    lon = np.arctan2(y, x) * _R2D * _D2R
    sl, cl, so, co = np.sin(lat), np.cos(lat), np.sin(lon), np.cos(lon)
    R_ecef_enu = np.array([[-so, -sl * co, cl * co], [co, -sl * so, cl * so], [0.0, cl, sl]])
    cy, sy = np.cos(yaw), np.sin(yaw)
    return R_ecef_enu @ np.array([[cy, -sy, 0.0], [sy, cy, 0.0], [0.0, 0.0, 1.0]])


def gnss_epochs(kf_times, truth_t, R, anchor, station, rng, rate=10.0, outlier_frac=0.03, drop_frac=0.05):
    """Seeded rover and station GNSS epochs at `rate` Hz over the keyframe times.  Satellites of GPS, GLONASS, Galileo and BeiDou
    (MEO, plus two BeiDou IGSO) on orbits of their systems' radii move slowly across the sky; the station's satellite positions differ
    from the rover's by up to a few metres (their own transmit times).  Pseudoranges = range + receiver clock - satellite clock
    (both cancel in the double difference) + noise (rover 1.5 m, station 0.3 m) + on a fraction of rover rows a multipath excess of
    20 .. 60 m; a few rover rows carry a zero pseudorange and a few satellites are missing from one receiver.  The rover's position
    is the true trajectory, linear in time between keyframes, through R and anchor.  Returns a list of (time, user, ref) with
    GNSS_RAW_DTYPE arrays (elevations in degrees, seen from the anchor)."""
    R_enu = ecef_local_rotation(anchor, 0.0)                      # ENU -> ECEF at the anchor
    sats = []                                                   # (prn, radius, azimuth0, elevation0, d az, d el) per satellite
    for prns, radius in ((range(1, 33), 26_560e3), (range(33, 57), 25_510e3), (range(57, 87), 29_600e3), (range(87, 122), 27_900e3)):
        for prn in rng.choice(list(prns), 11, replace=False):
            sats.append((int(prn), radius, rng.uniform(0, 2 * np.pi), rng.uniform(np.deg2rad(12), np.deg2rad(85)),
                         rng.normal(0, 2e-5), rng.normal(0, 1e-5)))
    for prn in (120, 121):                                      # BeiDou IGSO / GEO radius
        if all(s[0] != prn for s in sats):
            sats.append((prn, 42_164e3, rng.uniform(0, 2 * np.pi), rng.uniform(np.deg2rad(30), np.deg2rad(60)), 0.0, 0.0))
    prn, radius, az0, el0, daz, d_el = (np.array(c) for c in zip(*sats))
    ns = len(prn)
    sat_clock = rng.uniform(-3e5, 3e5, ns)
    # zero pseudoranges only where every system's filter drops them: PRN 84 is Galileo too, whose filter keeps it
    zero_ok = np.array([(prn_is_gps(p) or prn_is_bds(p)) and not (prn_is_glo(p) or prn_is_gal(p)) for p in prn])
    t0, t1 = kf_times[0], kf_times[-1]
    times = t0 - 0.05 + np.arange(int(np.ceil((t1 - t0 + 0.1) * rate)) + 1) / rate
    out = []
    for t in times:
        k = int(np.clip(np.searchsorted(kf_times, t) - 1, 0, len(kf_times) - 2))
        u = np.clip((t - kf_times[k]) / (kf_times[k + 1] - kf_times[k]), 0.0, 1.0)
        P = R @ ((1 - u) * truth_t[k] + u * truth_t[k + 1]) + anchor
        clk_u, clk_r = rng.uniform(-3e5, 3e5, 2)
        az, el = az0 + daz * (t - t0), np.clip(el0 + d_el * (t - t0), np.deg2rad(10), np.deg2rad(89))
        d = np.stack([np.sin(az) * np.cos(el), np.cos(az) * np.cos(el), np.sin(el)], axis=1) @ R_enu.T
        bd = d @ anchor                                         # |anchor + rho d| = radius
        rho = -bd + np.sqrt(bd * bd - (anchor @ anchor - radius * radius))
        su = anchor + rho[:, None] * d
        sr = su + rng.uniform(-3.0, 3.0, (ns, 3))
        pu = np.linalg.norm(su - P, axis=1) + clk_u - sat_clock + rng.normal(0, 1.5, ns)
        pu += np.where(rng.random(ns) < outlier_frac, rng.uniform(20.0, 60.0, ns), 0.0)
        pu = np.where((rng.random(ns) < 0.01) & zero_ok, 0.0, pu)
        pr = np.linalg.norm(sr - station, axis=1) + clk_r - sat_clock + rng.normal(0, 0.3, ns)
        user = np.zeros(ns, GNSS_RAW_DTYPE); ref = np.zeros(ns, GNSS_RAW_DTYPE)
        user["prn"], user["sat_pos"], user["psr"], user["elevation"] = prn, su, pu, np.rad2deg(el)
        ref["prn"], ref["sat_pos"], ref["psr"], ref["elevation"] = prn, sr, pr, np.rad2deg(el)
        user = user[rng.random(ns) >= drop_frac]; ref = ref[rng.random(ns) >= drop_frac]
        out.append((float(t), user[rng.permutation(len(user))], ref))   # the rover lists its satellites in its own order
    return out


def _lower_upper(kf_times, t):
    """getGlobalLowerUpperIdx (Estimator.cpp:1635-1662) with keyframe_idx[0] = 1: the keyframes k = 0 .. K-2 closest to t strictly
    before and strictly after it, or -1."""
    cand = np.asarray(kf_times[:-1])
    before, after = np.nonzero(cand < t)[0], np.nonzero(cand > t)[0]
    lo = int(before[np.argmin(t - cand[before])]) if len(before) else -1
    hi = int(after[np.argmin(cand[after] - t)]) if len(after) else -1
    return lo, hi


def dd_psr_factors(epochs, kf_times, trans, station, threshold):
    """The dd_psr_factor_20 list of one outer pass of optimizeBatchWithLandMark (Estimator.cpp:3086-3272) over GNSS epochs
    (gnss_epochs' format): an epoch inside the keyframe times is bracketed by getGlobalLowerUpperIdx (left = i, right = j, ratio =
    (t_j - t) / (t_j - t_i)); it is kept only when the right keyframe's current translation trans[j] is at least 1 m from the
    last kept one (P_add_idx, starting at 0).  Per constellation (GPS, BeiDou, GLONASS, Galileo) the rover's satellites also seen by
    the station (GPS and BeiDou: rover pseudorange > 1000) in the rover's order, the master the first with the largest elevation by
    the reference's |ele| > maxEle test, and a factor when more than 2 satellites remain.  Weight identity.  Returns the columns of
    api.dd_psr_factor_records (sat_offset in order) and the satellites (sat_user, sat_ref, psr_user, psr_ref)."""
    cols = dict(i=[], j=[], n_sat=[], master=[], ratio=[], threshold=[], station=[])
    su, sr, pu, pr = [], [], [], []
    p_add = np.zeros(3)
    for t, user, ref in epochs:
        if t > kf_times[-1] or t < kf_times[0]:
            continue
        lo, hi = _lower_upper(kf_times, t)
        if lo < 0 or hi < 0:
            continue
        ratio = (kf_times[hi] - t) / (kf_times[hi] - kf_times[lo])
        if np.linalg.norm(trans[hi] - p_add) < 1:
            continue
        p_add = np.array(trans[hi], np.float64)
        ref_of = {}
        for b, prn in enumerate(ref["prn"].tolist()):
            ref_of.setdefault(prn, []).append(b)
        for is_sys, psr_check in DD_PSR_SYSTEMS:
            pick = [(a, b) for a, prn in enumerate(user["prn"].tolist()) for b in ref_of.get(prn, ())
                    if is_sys(prn) and (not psr_check or user[a]["psr"] > 1000)]
            if len(pick) <= 2:
                continue
            ele = [float(user[a]["elevation"]) for a, _ in pick]
            master, max_ele = -1, 0.0
            for m, e in enumerate(ele):
                if abs(e) > max_ele:
                    max_ele, master = e, m
            if master < 0 or len(pick) > 20:
                raise ValueError("an epoch the reference cannot evaluate (no master, or more than 20 satellites)")
            cols["i"].append(lo); cols["j"].append(hi); cols["n_sat"].append(len(pick)); cols["master"].append(master)
            cols["ratio"].append(ratio); cols["threshold"].append(threshold); cols["station"].append(np.asarray(station, np.float64))
            for a, b in pick:
                su.append(user[a]["sat_pos"]); sr.append(ref[b]["sat_pos"]); pu.append(user[a]["psr"]); pr.append(ref[b]["psr"])
    cols = {k: np.asarray(v) for k, v in cols.items()}
    cols["station"] = cols["station"].reshape(-1, 3)
    return cols, dict(sat_user=np.asarray(su).reshape(-1, 3), sat_ref=np.asarray(sr).reshape(-1, 3), psr_user=np.asarray(pu, np.float64),
                      psr_ref=np.asarray(pr, np.float64))


def dd_psr_problem(K=200, seed=SEED0 + 17, search_range=6, outer_pass=1, yaw=0.3):
    """The level-0 batch refinement problem with its GNSS factors: pose_graph_problem's pose factors and trajectory, keyframe times
    0.25 .. 0.45 s apart (about 3 Hz), an anchor in Hong Kong with the local frame rotated by `yaw` from ENU, a station 3 km away, the
    epochs of gnss_epochs and the DD list of outer pass `outer_pass` (threshold DD_PSR_THRESHOLDS[outer_pass]) built against
    poses_init.  Adds R (R_ecef_local), anchor, station, kf_times, epochs, dd (the factor columns) and dd_sats."""
    P = pose_graph_problem(K=K, seed=seed, search_range=search_range)
    rng = np.random.default_rng([seed, 1])
    kf_times = 1_600_000_000.0 + np.concatenate([[0.0], np.cumsum(rng.uniform(0.25, 0.45, K - 1))])
    anchor = geo_to_ecef(22.3, 114.18, 5.0)
    station = anchor + ecef_local_rotation(anchor, 0.0) @ np.array([2400.0, -1800.0, 25.0])
    R = ecef_local_rotation(anchor, yaw)
    epochs = gnss_epochs(kf_times, P["poses_true"][:, :3], R, anchor, station, rng)
    dd, sats = dd_psr_factors(epochs, kf_times, P["poses_init"][:, :3], station, DD_PSR_THRESHOLDS[outer_pass])
    P.update(R=R, anchor=anchor, station=station, kf_times=kf_times, epochs=epochs, dd=dd, dd_sats=sats, outer_pass=outer_pass)
    return P


def raw_elevations(n_rings):
    """Elevation table (degrees) of a raw sweep for the ring rules of Preprocessing.cpp:441-483: every line sits inside its ring's
    interval, plus lines each rule treats specially.  16: VLP-16's -15..15 step 2, one line at -16.5 that int() truncates toward
    zero into ring 0, one at +17 (ring 16, skipped).  32: the centres of int((angle + 92/3) * 3/4), one line truncated into ring 0,
    one above (ring 32) and one below (ring -1), both skipped.  64: 33 lines on the upper branch 2 - (k + 0.1)/3 (rings 0..32),
    31 on the lower branch -8.83 - (j + 0.1)/2 (rings 33..63: 51..63 and angle < -24.33 are rejected), and one line above +2
    (int() gives ring 0, rejected by angle > 2)."""
    if n_rings == 16:
        return np.concatenate([np.arange(-15.0, 16.0, 2.0), [-16.5, 17.0]])
    if n_rings == 32:
        return np.concatenate([-92.0 / 3.0 + 4.0 / 3.0 * (np.arange(32) + 0.5), [-92.0 / 3.0 - 0.5, 12.5, -33.0]])
    if n_rings == 64:
        return np.concatenate([2.0 - (np.arange(33) + 0.1) / 3.0, -8.83 - (np.arange(1, 32) + 0.1) / 2.0, [2.3]])
    raise ValueError("n_rings must be 16, 32 or 64")


def _nearest_hit(sc, origin, dw, rects=None):
    """Distance along each world-frame ray dw[i] from origin (one point, or one per ray) to the nearest rectangle of the scene hit
    further than 0.5 m; inf for a miss.  rects: indices of the rectangles to test (default: all)."""
    best = np.full(len(dw), np.inf)
    for i in (range(len(sc.o)) if rects is None else rects):
        o, u, v, nrm = sc.o[i], sc.u[i], sc.v[i], sc.n[i]
        den = dw @ nrm
        with np.errstate(divide="ignore", invalid="ignore"):
            t = ((o - origin) @ nrm) / den
            hit = origin + t[:, None] * dw - o
            a = (hit @ u) / (u @ u); b = (hit @ v) / (v @ v)
        ok = (np.abs(den) > 1e-9) & (t > 0.5) & (a >= 0) & (a <= 1) & (b >= 0) & (b <= 1)
        best = np.where(ok & (t < best), t, best)
    return best


def _cast_firings(sc, origin, e, az, psi, rng, noise, near_frac, nan_frac, n_zaxis, rects=None):
    """Raw returns (n, 4) float32 in the sensor frame for rays of elevation e and azimuth az from a sensor yawed by psi at origin."""
    d = np.stack([np.cos(e) * np.cos(az), np.cos(e) * np.sin(az), np.sin(e)], 1)          # sensor frame
    dw = np.stack([np.cos(psi) * d[:, 0] - np.sin(psi) * d[:, 1], np.sin(psi) * d[:, 0] + np.cos(psi) * d[:, 1], d[:, 2]], 1)
    best = _nearest_hit(sc, origin, dw, rects)
    rg = best + rng.normal(0.0, noise, len(best))
    near = rng.random(len(rg)) < near_frac
    rg[near] = rng.uniform(0.5, 2.9, int(near.sum()))
    rg[~np.isfinite(best) | (best > 80.0) | (rng.random(len(rg)) < nan_frac)] = np.nan
    raw = np.empty((len(d), 4), np.float32)
    raw[:, :3] = rg[:, None] * d
    raw[:, 3] = rng.uniform(0.0, 100.0, len(d))
    if n_zaxis:
        at = rng.choice(len(raw), n_zaxis, replace=False)
        raw[at, 0] = 0.0; raw[at, 1] = 0.0
        raw[at, 2] = rng.choice([-1.0, 1.0], n_zaxis) * rng.uniform(3.5, 20.0, n_zaxis)
    return raw


def raw_sweep(n_rings=32, n_az=1875, start_az=0.3, coverage=2 * np.pi - 0.02, yaw_rate=0.0, seed=SEED0 + 12, t0=100.0,
              sweep_time=0.1, imu_rate=400.0, noise=0.01, nan_frac=0.01, near_frac=0.005, n_zaxis=4):
    """A raw spinning-LiDAR sweep as the driver delivers it (the input of Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:387):
    firing after firing (azimuth-major), the lines of a firing interleaved, x,y,z,intensity float32 (intensity = a reflectivity the
    reference ignores).  The head turns clockwise from azimuth start_az through `coverage` radians (slightly less or more than
    2 pi reaches the endOri corrections of :406-410) in sweep_time seconds while the sensor yaws at yaw_rate rad/s; rays are cast
    against the street-canyon scene in the sensor's pose at the firing's time.  Misses and a fraction nan_frac of the returns are
    NaN, a fraction near_frac are returns closer than 3 m, and n_zaxis points lie on the z axis (x = y = 0).
    Returns dict(raw (n, 4) float32, stamps, gyro (m, 3): IMU samples at imu_rate covering the sweep, t_scan_next = end of sweep,
    elev_deg: the line table)."""
    rng = np.random.default_rng(seed)
    sc = Scene(-60.0, 60.0, rng)
    origin = np.array([0.3, -0.4, 0.2])
    elev = np.deg2rad(raw_elevations(n_rings))
    L = len(elev)
    order = (np.arange(L) * 11) % L                          # interleaved firing order of the lines
    k = np.repeat(np.arange(n_az), L)
    line = np.tile(order, n_az)
    az = start_az - coverage * k / n_az
    psi = yaw_rate * sweep_time * k / n_az                   # sensor yaw at the firing's time
    raw = _cast_firings(sc, origin, elev[line], az, psi, rng, noise, near_frac, nan_frac, n_zaxis)
    stamps = t0 - 0.05 + np.arange(int((sweep_time + 0.1) * imu_rate) + 1) / imu_rate
    gyro = np.zeros((len(stamps), 3)); gyro[:, 2] = yaw_rate
    return dict(raw=raw, stamps=stamps, gyro=gyro, t_scan_next=t0 + sweep_time, elev_deg=np.rad2deg(elev))


def raw_drive(K, n_rings=32, speed=5.0, yaw_rate=0.1, seed=SEED0 + 13, n_az=1875, sweep_time=0.1, t0=100.0, imu_rate=400.0,
              noise=0.01, nan_frac=0.01, weave_period=8.0):
    """K consecutive raw sweeps (raw_sweep's format) of a sensor driving through ONE street-canyon scene at `speed` m/s, its yaw rate
    weaving as yaw_rate * cos(2 pi t / weave_period) rad/s; every firing is cast from the sensor's pose at its own time, so each sweep
    carries the motion that happens during it.  Returns dict(sweeps: list of (n, 4) float32, poses (K, 7): t(x,y,z), q(w,x,y,z) of
    the sensor at the start of each sweep in the frame of the first, stamps / gyro (m, 3): IMU samples at imu_rate over the whole
    drive, t_scan_next (K,): end time of each sweep, t0)."""
    rng = np.random.default_rng(seed)
    path = speed * K * sweep_time
    sc = Scene(-60.0, path + 60.0, rng, n_boxes=int(round(30 * (path + 120.0) / 140.0)))
    origin0 = np.array([0.3, -0.4, 0.2])
    # yaw and position on a 1 ms grid (trapezoidal integration), interpolated at the firing times
    dt = 1e-3
    tg = np.arange(0.0, K * sweep_time + 2 * dt, dt)
    w = 2 * np.pi / weave_period
    yawg = yaw_rate * np.sin(w * tg) / w
    vx, vy = speed * np.cos(yawg), speed * np.sin(yawg)
    xg = np.concatenate([[0.0], np.cumsum(0.5 * (vx[1:] + vx[:-1]) * dt)])
    yg = np.concatenate([[0.0], np.cumsum(0.5 * (vy[1:] + vy[:-1]) * dt)])

    def state(t):
        return np.interp(t, tg, xg), np.interp(t, tg, yg), yaw_rate * np.sin(w * t) / w

    elev = np.deg2rad(raw_elevations(n_rings))
    L = len(elev)
    order = (np.arange(L) * 11) % L
    # rectangles that can give a return within 80 m of some point of the sweep (the others cannot change the nearest hit)
    x_lo_r = np.minimum(sc.o[:, 0], sc.o[:, 0] + sc.u[:, 0] + sc.v[:, 0]); x_hi_r = np.maximum(sc.o[:, 0], sc.o[:, 0] + sc.u[:, 0] + sc.v[:, 0])
    sweeps, poses = [], np.zeros((K, 7))
    for k in range(K):
        kk = np.repeat(np.arange(n_az), L)
        tf = (k + kk / n_az) * sweep_time
        x, y, psi = state(tf)
        origin = np.stack([origin0[0] + x, origin0[1] + y, np.full(len(x), origin0[2])], 1)
        az = 0.3 - (2 * np.pi - 0.02) * kk / n_az
        xs, _, _ = state(np.array([k * sweep_time, (k + 1) * sweep_time]))
        rects = np.nonzero((x_hi_r > xs.min() + origin0[0] - 81.0) & (x_lo_r < xs.max() + origin0[0] + 81.0))[0]
        sweeps.append(_cast_firings(sc, origin, elev[np.tile(order, n_az)], az, psi, rng, noise, 0.0, nan_frac, 0, rects))
        xk, yk, pk = state(k * sweep_time)
        poses[k, :3] = [xk, yk, 0.0]
        poses[k, 3:] = [np.cos(pk / 2), 0.0, 0.0, np.sin(pk / 2)]
    stamps = t0 - 0.05 + np.arange(int((K * sweep_time + 0.1) * imu_rate) + 1) / imu_rate
    gyro = np.zeros((len(stamps), 3)); gyro[:, 2] = yaw_rate * np.cos(w * (stamps - t0))
    return dict(sweeps=sweeps, poses=poses, stamps=stamps, gyro=gyro, t_scan_next=t0 + (np.arange(K) + 1) * sweep_time, t0=t0)


def ring_scan(n_rings=32, n_az=1500, seed=SEED0 + 11, fov=(-25.0, 15.0), noise=0.01, drop=0.02):
    """A spinning-LiDAR sweep of the street-canyon scene, ring by ring, for the front end's feature extraction (SURVEY 8 f-4):
    rays are cast from the sensor against the scene's rectangles (nearest hit), range noise N(0, noise), a fraction `drop` of the
    returns missing.  Returns (cloud (n,4) float32: x,y,z,intensity = ring + 0.1 relTime; scan_start, scan_end int32 arrays) laid
    out as Preprocessing::cloudHandler lays out `laserCloud` (GLIO/src/Preprocessing.cpp:529-534): rings concatenated,
    scanStartInd = first index + 5, scanEndInd = last index - 5."""
    rng = np.random.default_rng(seed)
    sc = Scene(-60.0, 60.0, rng)
    origin = np.array([0.3, -0.4, 0.2])
    elev = np.deg2rad(np.linspace(fov[0], fov[1], n_rings))
    clouds, start, end = [], [], []
    total = 0
    for r in range(n_rings):
        az = np.linspace(0.0, 2 * np.pi, n_az, endpoint=False) + rng.uniform(0, 1e-3)
        d = np.stack([np.cos(elev[r]) * np.cos(az), np.cos(elev[r]) * np.sin(az), np.full(n_az, np.sin(elev[r]))], 1)
        best = np.full(n_az, np.inf)
        for o, u, v, nrm in zip(sc.o, sc.u, sc.v, sc.n):
            den = d @ nrm
            with np.errstate(divide="ignore", invalid="ignore"):
                t = ((o - origin) @ nrm) / den
            hit = origin + t[:, None] * d - o
            a = (hit @ u) / (u @ u); b = (hit @ v) / (v @ v)
            ok = (np.abs(den) > 1e-9) & (t > 0.5) & (a >= 0) & (a <= 1) & (b >= 0) & (b <= 1)
            best = np.where(ok & (t < best), t, best)
        keep = np.isfinite(best) & (best < 80.0) & (rng.random(n_az) > drop)
        rg = best[keep] + rng.normal(0.0, noise, int(keep.sum()))
        pts = origin + rg[:, None] * d[keep]
        rel = az[keep] / (2 * np.pi)
        cl = np.concatenate([pts, (r + 0.1 * rel)[:, None]], 1).astype(np.float32)
        clouds.append(cl)
        start.append(total + 5); total += len(cl); end.append(total - 6)
    return np.concatenate(clouds), np.asarray(start, np.int32), np.asarray(end, np.int32)


def loop_drive(K=240, n_points=2500, dt=0.5, speed=2.0, lane=3.0, drift_t=0.01, drift_yaw_deg=0.01, rng_range=40.0, seed=SEED0 + 14,
               t0=1000.0):
    """Keyframe surf clouds of one street-canyon scene along a closed path, for the loop closure (GLIO/src/Estimator.cpp:5090-5273).

    The sensor drives out along the lane y = -lane for K/2 keyframes, turns round and drives back along y = +lane to where it
    started: keyframe k and keyframe K-1-k see the same stretch of street, (K-1-2k)*dt seconds apart, so the path revisits its
    beginning after more than lc_time_thres seconds once K*dt is large enough.  clouds[k] is n_points points of the scene within
    rng_range of the sensor in the lidar frame of the TRUE pose (float32, packed x,y,z); poses[k] (t, q) carries a drift that grows
    with k: a yaw of drift_yaw_deg*k degrees about the origin and a shift of (drift_t*k, drift_t*k/2, 0) metres, so a registration
    of the returning keyframes against the outbound ones has a real correction to find.  times[k] = t0 + k*dt."""
    rng = np.random.default_rng(seed)
    half = K // 2
    x_max = speed * dt * max(half - 1, 1)
    scene = Scene(-rng_range - 10.0, x_max + rng_range + 10.0, rng)
    truth = np.zeros((K, 7)); poses = np.zeros((K, 7))
    for k in range(K):
        out = k < half
        x = speed * dt * (k if out else K - 1 - k)
        truth[k, :3] = [x, -lane if out else lane, 0.0]
        truth[k, 3:] = quat_from_rpy(0.0, 0.0, 0.0 if out else np.pi)
        psi = np.deg2rad(drift_yaw_deg * k)
        qd = quat_from_rpy(0.0, 0.0, psi)
        poses[k, :3] = quat_to_R(qd) @ truth[k, :3] + [drift_t * k, 0.5 * drift_t * k, 0.0]
        q = quat_mul(qd, truth[k, 3:])
        poses[k, 3:] = q / np.linalg.norm(q)
    clouds = [scan_in_lidar_frame(scene, truth[k], n_points, rng, rng_range) for k in range(K)]
    return dict(clouds=clouds, poses=poses, poses_true=truth, times=t0 + dt * np.arange(K), K=K, dt=dt, seed=seed)
