"""ctypes binding of the loop-closure oracle (oracle/loop/libgo_loop.so) and a sequential restatement of the Estimator's loop
closure up to the GTSAM factor (detectLoopClosure + performLoopClosure, GLIO/src/Estimator.cpp:5101-5273).

TEST INFRASTRUCTURE ONLY - imported by tests/ and scripts/.  Nothing under glio_b200/ may import this module.
The clouds are assembled on the existing oracle primitives (pyoracle.transform_points = transformCloud, pyoracle.voxel_filter with
the stable order = ds_filter_his_frames); the pose arithmetic is scalar double code in Eigen's generic operation order
(pyoracle_odom's quaternion helpers).  PARITY UNPINNED: see the header of oracle/loop/go_loop.cpp.
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np

from oracle import pyoracle as po
from oracle import pyoracle_odom as pod

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "loop")
_SO = os.path.join(_DIR, "libgo_loop.so")
_LIB = None

NOT_CONVERGED, ITERATIONS, TRANSFORM, ABS_MSE, REL_MSE, NO_CORRESPONDENCES = range(6)
STATE_NAMES = {0: "NOT_CONVERGED", 1: "ITERATIONS", 2: "TRANSFORM", 3: "ABS_MSE", 4: "REL_MSE", 5: "NO_CORRESPONDENCES"}


class IcpResult(C.Structure):
    _fields_ = [("converged", C.c_int32), ("state", C.c_int32), ("iterations", C.c_int32), ("pad", C.c_int32), ("n_corr", C.c_int64),
                ("final_T", C.c_float * 16), ("fitness", C.c_double)]


class IcpIteration(C.Structure):
    _fields_ = [("transformation", C.c_float * 16), ("n_corr", C.c_int64), ("mse", C.c_double)]


def build(force=False):
    src = os.path.join(_DIR, "go_loop.cpp")
    if force or not os.path.exists(_SO) or os.path.getmtime(src) > os.path.getmtime(_SO):
        subprocess.check_call(["make", "-C", _DIR, "-s"], stdout=subprocess.DEVNULL)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        L.go_lc_hsum_f.restype = C.c_float
        L.go_lc_hsum_d.restype = C.c_double
        L.go_lc_detect.restype = C.c_int
        _LIB = L
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _xyz(a):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, 3))


def svd3(a):
    """Eigen 3.3 JacobiSVD<Matrix3f>(a, ComputeFullU | ComputeFullV): (U, singular values, V), float32."""
    a = np.ascontiguousarray(a, np.float32).reshape(3, 3)
    U = np.empty((3, 3), np.float32); S = np.empty(3, np.float32); V = np.empty((3, 3), np.float32)
    lib().go_lc_svd3(_p(a), _p(U), _p(S), _p(V))
    return U, S, V


def umeyama(src, dst):
    """pcl::umeyama(src, dst, false) with the documented summation order; row-major 4x4 float32."""
    s = _xyz(src); d = _xyz(dst)
    T = np.empty((4, 4), np.float32)
    lib().go_lc_umeyama(_p(s), _p(d), C.c_int64(len(s)), _p(T))
    return T


def nn(tgt, qry):
    """exact 1-NN (float L2_Simple, ties by index): (idx int32, squared distance float32)."""
    t = _xyz(tgt); q = _xyz(qry)
    idx = np.empty(len(q), np.int32); d = np.empty(len(q), np.float32)
    lib().go_lc_nn(_p(t), C.c_int64(len(t)), _p(q), C.c_int64(len(q)), _p(idx), _p(d))
    return idx, d


def hsum(v):
    v = np.ascontiguousarray(v)
    if v.dtype == np.float32:
        return np.float32(lib().go_lc_hsum_f(_p(v), C.c_int64(len(v))))
    v = v.astype(np.float64)
    return float(lib().go_lc_hsum_d(_p(v), C.c_int64(len(v))))


def icp(src, tgt, max_iterations=100, max_correspondence_distance=30.0, transformation_epsilon=1e-6, euclidean_fitness_epsilon=1e-6,
        log_cap=None):
    """IterativeClosestPoint::align with an identity guess + getFitnessScore.  Returns dict(converged, state, iterations, n_corr,
    final (4x4 float32), fitness, aligned (n, 3), log: list of (transformation, n_corr, mse), corr: (query, match, dist))."""
    s = _xyz(src); t = _xyz(tgt)
    n = len(s)
    cap = max_iterations if log_cap is None else log_cap
    res = IcpResult()
    aligned = np.empty((n, 3), np.float32)
    log = (IcpIteration * max(cap, 1))()
    cq = np.empty(max(n, 1), np.int32); cm = np.empty(max(n, 1), np.int32); cd = np.empty(max(n, 1), np.float32)
    lib().go_lc_icp(_p(s), C.c_int64(n), _p(t), C.c_int64(len(t)), C.c_int(max_iterations), C.c_double(max_correspondence_distance),
                    C.c_double(transformation_epsilon), C.c_double(euclidean_fitness_epsilon), C.byref(res), _p(aligned), log, C.c_int(cap),
                    _p(cq), _p(cm), _p(cd), C.c_int64(n))
    k = min(res.iterations, cap)
    nc = int(res.n_corr)
    return dict(converged=bool(res.converged), state=int(res.state), iterations=int(res.iterations), n_corr=nc,
                final=np.array(res.final_T[:], np.float32).reshape(4, 4), fitness=float(res.fitness), aligned=aligned,
                log=[(np.array(log[i].transformation[:], np.float32).reshape(4, 4), int(log[i].n_corr), float(log[i].mse)) for i in range(k)],
                corr=(cq[:nc].copy(), cm[:nc].copy(), cd[:nc].copy()))


def detect(pos, times, sel, time_new_odom, radius, time_thres):
    """radius search of the keyframe positions + the time test: (closest_his_idx, radius-search order)."""
    p = _xyz(pos); tm = np.ascontiguousarray(times, np.float64); s = np.ascontiguousarray(sel, np.float32)
    order = np.empty(max(len(p), 1), np.int32); nf = C.c_int32(0)
    c = lib().go_lc_detect(_p(p), _p(tm), C.c_int(len(p)), _p(s), C.c_double(time_new_odom), C.c_double(radius), C.c_double(time_thres),
                           _p(order), C.byref(nf))
    return int(c), order[:nf.value].copy()


# ---- host pose arithmetic (poses t, q; scalar double in Eigen's order)
def extrinsic_bl(q_lb, t_lb):
    """q_bl = q_lb.inverse(), t_bl = -(q_bl * t_lb) (Estimator.cpp:873-877)."""
    q_bl = pod.quat_inverse(tuple(float(x) for x in q_lb))
    r = pod.quat_rot(q_bl, tuple(float(x) for x in t_lb))
    return q_bl, (-r[0], -r[1], -r[2])


def world_of_cloud(pose, q_bl, t_bl):
    """q_tmp = q_po * q_bl, t_tmp = q_po * t_bl + t_po (:5140-5141)."""
    t_po = tuple(float(x) for x in pose[:3]); q_po = tuple(float(x) for x in pose[3:])
    q = pod.quat_mul(q_po, q_bl)
    r = pod.quat_rot(q_po, t_bl)
    return (r[0] + t_po[0], r[1] + t_po[1], r[2] + t_po[2]), q


def quat_from_R(R):
    """Eigen quaternion_assign_impl<Other, 3, 3> (w, x, y, z)."""
    m = [[float(R[i][j]) for j in range(3)] for i in range(3)]
    t = (m[0][0] + m[1][1]) + m[2][2]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        return (w, (m[2][1] - m[1][2]) * t, (m[0][2] - m[2][0]) * t, (m[1][0] - m[0][1]) * t)
    i = 0
    if m[1][1] > m[0][0]:
        i = 1
    if m[2][2] > m[i][i]:
        i = 2
    j = (i + 1) % 3; k = (j + 1) % 3
    t = math.sqrt(((m[i][i] - m[j][j]) - m[k][k]) + 1.0)
    c = [0.0, 0.0, 0.0]
    c[i] = 0.5 * t
    t = 0.5 / t
    w = (m[k][j] - m[j][k]) * t
    c[j] = (m[j][i] + m[i][j]) * t
    c[k] = (m[k][i] + m[i][k]) * t
    return (w, c[0], c[1], c[2])


def pose_from(final, latest):
    """quaternionIncre from final's rotation, (qIncre * q_latest, qIncre * t_latest + t) (:5228-5242); t then q."""
    F = np.asarray(final, np.float32).astype(np.float64)
    qi = quat_from_R(F[:3, :3])
    q = pod.quat_mul(qi, tuple(float(x) for x in latest[3:]))
    r = pod.quat_rot(qi, tuple(float(x) for x in latest[:3]))
    return np.array([r[0] + F[0, 3], r[1] + F[1, 3], r[2] + F[2, 3], q[0], q[1], q[2], q[3]])


def loop_default_options(**kw):
    o = dict(lc_search_radius=25.0, lc_time_thres=30.0, lc_map_width=25, lc_icp_thres=0.2, slide_window_width=5, leaf=0.4,
             q_lb=(1.0, 0.0, 0.0, 0.0), t_lb=(0.0, 0.0, 0.28), max_iterations=100, max_correspondence_distance=30.0,
             transformation_epsilon=1e-6, euclidean_fitness_epsilon=1e-6)
    o.update(kw)
    return o


class LoopOracle:
    """The keyframe store and one loop-closure step, sequentially (see glio_loop_step in include/glio_b200.h)."""

    def __init__(self, **options):
        self.o = loop_default_options(**options)
        self.q_bl, self.t_bl = extrinsic_bl(self.o["q_lb"], self.o["t_lb"])
        self.clouds, self.poses, self.times = [], [], []
        self.time_last_loop = 0.0

    def add_keyframe(self, cloud, pose, time):
        self.clouds.append(_xyz(cloud).copy()); self.poses.append(np.array(pose, np.float64)); self.times.append(float(time))
        return len(self.clouds) - 1

    def set_poses(self, first, poses):
        for i, p in enumerate(np.asarray(poses, np.float64).reshape(-1, 7)):
            self.poses[first + i] = p.copy()

    def _cloud(self, ids):
        parts = []
        for k in ids:
            t, q = world_of_cloud(self.poses[k], self.q_bl, self.t_bl)
            parts.append(po.transform_points(self.clouds[k], np.array(t), np.array(q)) if len(self.clouds[k]) else np.zeros((0, 3), np.float32))
        cat = np.concatenate(parts) if parts else np.zeros((0, 3), np.float32)
        if len(cat) == 0:
            return cat, cat
        f = po.voxel_filter(cat, self.o["leaf"], stable=True)
        return cat, (cat if f is None else f[0])

    def step(self, sel, time_new_odom):
        o = self.o
        rep = dict(detected=False, closest_his_idx=-1, latest_frame_idx=-1, accepted=False, n_candidates=0, icp=None, latest=None, his=None,
                   pose_from=None, pose_to=None, noise_score=None)
        K = len(self.clouds)
        if K:
            pos = np.array([p[:3] for p in self.poses], np.float64).astype(np.float32)
            c, order = detect(pos, np.array(self.times), sel, time_new_odom, o["lc_search_radius"], o["lc_time_thres"])
            rep["closest_his_idx"] = c; rep["n_candidates"] = len(order)
            if c >= 0 and not (abs(self.time_last_loop - time_new_odom) < 0.2):
                rep["detected"] = True
                latest = K - o["slide_window_width"]
                rep["latest_frame_idx"] = latest
                lat_ids = [latest - j for j in range(6) if latest - j >= 0]
                his_ids = [c + j for j in range(-o["lc_map_width"], o["lc_map_width"] + 1) if 0 <= c + j <= latest]
                lat_raw, lat = self._cloud(lat_ids)
                his_raw, his = self._cloud(his_ids)
                rep.update(latest=lat, his=his, n_latest=len(lat_raw), n_his=len(his_raw))
                r = icp(lat, his, o["max_iterations"], o["max_correspondence_distance"], o["transformation_epsilon"], o["euclidean_fitness_epsilon"])
                rep["icp"] = r
                if r["converged"] and not (r["fitness"] > float(np.float32(o["lc_icp_thres"]))):
                    rep["accepted"] = True
                    rep["pose_from"] = pose_from(r["final"], self.poses[latest])
                    rep["pose_to"] = self.poses[c].copy()
                    rep["noise_score"] = r["fitness"]
                    self.time_last_loop = self.times[latest]
        rep["time_last_loop"] = self.time_last_loop
        return rep
