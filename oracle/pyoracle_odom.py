"""Sequential restatement of the front end's LidarOdometry node (GLIO/src/LidarOdometry.cpp:661-695, run() and what it calls), written
literally on top of the CPU oracle's primitives: pyoracle.voxel_filter (stable), transform_points, assoc_scan_to_map with the front
end's gates and the kd-tree, and WindowProblem.solve with Levenberg-Marquardt over DENSE_QR (reserved = 2) and no time limit.

TEST INFRASTRUCTURE ONLY - imported by tests/ and scripts/.  The pose bookkeeping is scalar double arithmetic in Eigen's generic
operation order (Quaternion product, _transformVector, inverse() = conjugate / squaredNorm with coeffs() summed x, y, z, w).
PARITY UNPINNED: Eigen's SSE2 quaternion product and reduction order, which a vectorised build of the reference uses instead.

Poses inside follow the reference (abs_pose / rel_pose: q(w,x,y,z), t(x,y,z)); what step() returns is in the library's t, q order.
"""
import math

import numpy as np

from oracle import pyoracle as po

MAX_ROUNDS = 8
NO_BLOCKS = "Function tolerance reached. No non-constant parameter blocks found."


# ---- Eigen arithmetic, scalar
def quat_mul(a, b):
    return (a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
            a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1])


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def quat_rot(q, v):
    """QuaternionBase::_transformVector: uv = 2 (vec x v); v + w uv + vec x uv."""
    u = (q[1], q[2], q[3])
    uv = _cross(u, v)
    uv = (uv[0] + uv[0], uv[1] + uv[1], uv[2] + uv[2])
    c = _cross(u, uv)
    return (v[0] + q[0] * uv[0] + c[0], v[1] + q[0] * uv[1] + c[1], v[2] + q[0] * uv[2] + c[2])


def quat_inverse(q):
    """Quaternion::inverse(): the conjugate divided by squaredNorm() (NOT just the conjugate); zero for a zero quaternion."""
    n2 = ((q[1] * q[1] + q[2] * q[2]) + q[3] * q[3]) + q[0] * q[0]
    if n2 > 0.0:
        return (q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2)
    return (0.0, 0.0, 0.0, 0.0)


def unify_quaternion(q):
    """unifyQuaternion (GLIO/include/utils/math_tools.h:166-173)."""
    return tuple(q) if q[0] >= 0 else (-q[0], -q[1], -q[2], -q[3])


def predict(abs_pose, rel_pose):
    """poseInitialization (:406-433): t0 = q0*dt + t0, q0 = q0*dq.  Poses q, t."""
    q0, t0, dq, dt = abs_pose[:4], abs_pose[4:], rel_pose[:4], rel_pose[4:]
    v = quat_rot(q0, dt)
    t = (v[0] + t0[0], v[1] + t0[1], v[2] + t0[2])
    return tuple(quat_mul(q0, dq)) + t


def relative(p1, p2):
    """computeRelative (:435-471): q1^-1 q2, q1^-1 (t2 - t1).  Poses q, t."""
    qi = quat_inverse(p1[:4])
    q = quat_mul(qi, p2[:4])
    t = quat_rot(qi, (p2[4] - p1[4], p2[5] - p1[5], p2[6] - p1[6]))
    return tuple(q) + tuple(t)


def keyframe_rule(t_cur, q_cur, t_kf, q_kf, size, kf_num):
    """:566-578 with C++'s precedence; size = pose count before this sweep's savePoses.  acos of a w above 1 is NaN -> False."""
    d = (t_cur[0] - t_kf[0], t_cur[1] - t_kf[1], t_cur[2] - t_kf[2])
    dis = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    w = quat_mul(quat_inverse(q_kf), q_cur)[0]
    ang = 2 * math.acos(w) if -1.0 <= w <= 1.0 else float("nan")
    return (((dis > 0.2 or ang > 0.1) and size - kf_num > 1) or size - kf_num > 2) or size <= 1


def deskew(cloud, trans):
    """undistortion (:176-200) with the identity quaternion of publishCloudLast: float(double(p) + r*trans),
    r = min(double(float(i - int(i))) / 0.1, 1)."""
    c = np.array(cloud, np.float32, copy=True).reshape(-1, 4)
    i = c[:, 3]
    line = np.trunc(i).astype(np.int64)
    dt_f = (i - line.astype(np.float32)).astype(np.float32)
    r = dt_f.astype(np.float64) / 0.1
    r = np.where(r > 1, 1.0, r)
    for k in range(3):
        c[:, k] = (c[:, k].astype(np.float64) + r * float(trans[k])).astype(np.float32)
    return c


def voxel(xyz):
    """VoxelGrid(0.2) with PCL's pass-through on voxel-index overflow."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    if len(xyz) == 0:
        return xyz
    r = po.voxel_filter(xyz, 0.2, stable=True)
    return xyz.copy() if r is None else r[0]


def front_end_params():
    """findCorrespondingSurfFeatures (:343-404): squared radius 1.0, plane 0.06, weight 0.4."""
    prm = po.default_params()
    prm.kd_max_radius = 1.0; prm.surf_dist_thres = 0.06; prm.weight_min = 0.4; prm.lidar_const = 1.0
    return prm


def _tq(p):
    return np.array([p[4], p[5], p[6], p[0], p[1], p[2], p[3]])


class OdometryOracle:
    def __init__(self, max_num_iter=12, scan_match_cnt=1, deskew=0, nthreads=0):
        self.max_num_iter, self.scan_match_cnt, self.deskew = max_num_iter, scan_match_cnt, deskew
        self.nthreads = nthreads            # association threads (0: the oracle's default); the solve runs on one
        self.reset()

    def reset(self):
        self.initialized = False
        self.abs_pose = (1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
        self.rel_pose = (1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
        self.pose_info = []            # pose_info_cloud_frame
        self.surf_frames = []          # surf_last_ds of every saved sweep (scan frame); only the last one is read
        self.recent = []               # recent_surf_frames (world frame)
        self.latest_frame_idx = 0
        self.kf, self.kf_num = True, 0
        self.trans_last_kf, self.quat_last_kf = (0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0)

    def step(self, surf, full=None, forced=None):
        """One sweep.  surf / full: (n, 4) float32.  forced: optional list of poses (t, q) that replace the pose after each round
        (so the oracle can be driven along another implementation's trajectory).  Returns a dict like Odometry.step, plus map / scan
        (the filtered clouds), per-round status / steps, and the published clouds."""
        surf = np.asarray(surf, np.float32).reshape(-1, 4)
        full = None if full is None else np.asarray(full, np.float32).reshape(-1, 4)
        out = dict(initialised=False, keyframe=False, skipped=False, n_map=0, n_scan=0, rounds=[], map=np.zeros((0, 3), np.float32),
                   scan=np.zeros((0, 3), np.float32), surf=None, full=None, summary=None)
        if not self.initialized:
            # savePoses before surf_last_ds was ever filled: identity pose, EMPTY frame; then checkInitialization
            self.pose_info.append(self.abs_pose)
            self.surf_frames.append(np.zeros((0, 3), np.float32))
            self.initialized = True
            out.update(initialised=True, surf=surf.copy(), full=None if full is None else full.copy())
        else:
            self.abs_pose = predict(self.abs_pose, self.rel_pose)
            # buildLocalMap (:267-288)
            size = len(self.pose_info)
            if size <= 1:
                surf_from_map = surf[:, :3].copy()
            else:
                i = size - 1
                p = self.pose_info[i]
                if len(self.recent) < 20:
                    self.recent.append(po.transform_points(self.surf_frames[-1], p[4:], p[:4]) if len(self.surf_frames[-1]) else
                                       np.zeros((0, 3), np.float32))
                elif self.latest_frame_idx != size - 1:
                    self.recent.pop(0)
                    self.latest_frame_idx = size - 1
                    p = self.pose_info[self.latest_frame_idx]
                    self.recent.append(po.transform_points(self.surf_frames[-1], p[4:], p[:4]) if len(self.surf_frames[-1]) else
                                       np.zeros((0, 3), np.float32))
                surf_from_map = np.concatenate(self.recent) if self.recent else np.zeros((0, 3), np.float32)
            # downSampleCloud (:305-313)
            map_ds = voxel(surf_from_map)
            scan = voxel(surf[:, :3])
            out.update(map=map_ds, scan=scan, n_map=len(map_ds), n_scan=len(scan))
            # updateTransformationWithCeres (:474-579)
            if len(map_ds) < 10:
                out["skipped"] = True
            else:
                tree = po.KdTree(map_ds)
                rounds = 8 if len(self.pose_info) < 2 else self.scan_match_cnt
                prm = front_end_params()
                for r in range(rounds):
                    x = _tq(self.abs_pose)
                    rd = dict(n_match=0, status=None, iterations=0, successful=0, termination=0, steps=np.zeros((0, 6)), message=NO_BLOCKS)
                    if len(scan):
                        a = po.assoc_scan_to_map(map_ds, scan, x[:3], x[3:], prm=prm, tree=tree, nthreads=self.nthreads)
                        rd["status"] = a["status"]; rd["n_match"] = a["nvalid"]
                        v = a["status"] == po.GO_VALID
                    if rd["n_match"] > 0:
                        prob = po.WindowProblem(x[None, :], None, [1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0], huber_delta=0.1)
                        prob.add_unary(np.zeros(int(v.sum()), np.int32), scan[v], a["nsd"][v], np.ones(int(v.sum())))
                        ro = prob.solve(po.solver_options(reserved=2, max_num_iterations=self.max_num_iter), mode=0)
                        s = ro["summary"]
                        x = ro["poses"][0]
                        rd.update(iterations=s.num_iterations, successful=s.num_successful_steps, termination=s.termination,
                                  steps=ro["steps"], message=s.message.decode(), iteration_log=ro["iterations"])
                    q = unify_quaternion((float(x[3]), float(x[4]), float(x[5]), float(x[6])))
                    self.abs_pose = q + (float(x[0]), float(x[1]), float(x[2]))
                    rd["solved_pose"] = _tq(self.abs_pose)
                    if forced is not None:
                        f = np.asarray(forced[r], np.float64)
                        self.abs_pose = (f[3], f[4], f[5], f[6], f[0], f[1], f[2])
                    rd["pose"] = _tq(self.abs_pose)
                    out["rounds"].append(rd)
                t_cur, q_cur = self.abs_pose[4:], self.abs_pose[:4]
                if keyframe_rule(t_cur, q_cur, self.trans_last_kf, self.quat_last_kf, len(self.pose_info), self.kf_num):
                    self.kf = True
                    self.trans_last_kf, self.quat_last_kf = tuple(t_cur), tuple(q_cur)
                else:
                    self.kf = False
            # savePoses, computeRelative
            self.pose_info.append(self.abs_pose)
            self.surf_frames.append(scan)
            del self.surf_frames[:-21]                 # clearCloud keeps at most 20 (+ the one just saved); only the last is read
            self.rel_pose = relative(self.pose_info[-2], self.pose_info[-1])
            if self.kf:
                self.kf_num = len(self.pose_info)
                trans = self.rel_pose[4:]
                out.update(surf=deskew(surf, trans) if self.deskew else surf.copy(),
                           full=None if full is None else (deskew(full, trans) if self.deskew else full.copy()))
            out["keyframe"] = self.kf
        out["pose"] = _tq(self.abs_pose)
        out["rel_pose"] = _tq(self.rel_pose)
        return out
