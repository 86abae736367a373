"""Python mirror of the C ABI (include/glio_b200.h) — a thin ctypes layer over glio_b200/libglio_b200.so.

The method names follow the reference's own vocabulary (GLIO/src/Estimator.cpp): set_map ~ kd_tree->setInputCloud,
assoc_scan_to_map ~ findCorrespondingSurfFeatures, select ~ featureSelection (as an input index list),
eval_unary ~ ResidualBlock::Evaluate over LidarPlaneNormFactor + normal-equation accumulation.

There is no CPU fallback: if the CUDA library is missing or no GPU is visible, construction raises.
torch is used only for device buffers/streams by callers (bench.py); this module needs numpy + ctypes only.
"""
import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libglio_b200.so")
_LIB = None
_LIB_LOCK = threading.Lock()

HOST, DEVICE = 0, 1
MATCH_VALID, MATCH_FAIL_RADIUS, MATCH_FAIL_PLANE, MATCH_FAIL_WEIGHT = 0, 1, 2, 3


class GlioError(RuntimeError):
    pass


class Params(C.Structure):
    _fields_ = [("kd_max_radius", C.c_double), ("surf_dist_thres", C.c_double), ("lidar_const", C.c_double),
                ("weight_min", C.c_double), ("huber_delta", C.c_double), ("q_lb", C.c_double * 4),
                ("t_lb", C.c_double * 3), ("batch_max_radius", C.c_double), ("batch_dist_thres", C.c_double),
                ("batch_score", C.c_double), ("cell_size", C.c_float), ("keep_debug", C.c_int32), ("unit_score", C.c_int32)]


def lib():
    """Load the CUDA library; raise loudly when it is not built (no fallback path exists).  Threads that ask first at the same
    time get the one handle, with its prototypes set before anyone sees it."""
    global _LIB
    if _LIB is not None:
        return _LIB
    with _LIB_LOCK:
        if _LIB is not None:
            return _LIB
        if not os.path.exists(_LIB_PATH):
            raise GlioError(f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(glio_b200 has no CPU fallback)")
        L = C.CDLL(_LIB_PATH)
        L.glio_last_error.restype = C.c_char_p
        L.glio_last_error.argtypes = [C.c_void_p]
        L.glio_stream.restype = C.c_void_p
        L.glio_stream.argtypes = [C.c_void_p]
        L.glio_launch_count.restype = C.c_int64
        L.glio_launch_count.argtypes = [C.c_void_p]
        L.glio_destroy.argtypes = [C.c_void_p]
        L.glio_destroy.restype = None
        L.glio_marg_prior_destroy.argtypes = [C.c_void_p]
        L.glio_marg_prior_destroy.restype = None
        L.glio_marg_prior_create.restype = C.c_void_p
        _LIB = L
    return _LIB


def default_params(**kw):
    p = Params()
    lib().glio_default_params(C.byref(p))
    for k, v in kw.items():
        if k in ("q_lb", "t_lb"):
            arr = getattr(p, k)
            for i, x in enumerate(v):
                arr[i] = float(x)
        else:
            setattr(p, k, v)
    return p


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if isinstance(a, int):
        return C.c_void_p(a)
    raise TypeError(type(a))


def _points_arg(xyz):
    """numpy float32 (n,3|stride) host array, or (device_ptr:int, n, stride) tuple / torch tensor."""
    if isinstance(xyz, np.ndarray):
        a = np.ascontiguousarray(xyz, dtype=np.float32)
        if a.ndim == 1:
            a = a.reshape(-1, 3)
        return a, _ptr(a), a.shape[0], a.shape[1], HOST
    if hasattr(xyz, "data_ptr"):          # torch tensor on the GPU
        assert xyz.is_cuda and xyz.is_contiguous() and xyz.dtype.itemsize == 4
        return xyz, C.c_void_p(xyz.data_ptr()), xyz.shape[0], xyz.shape[1], DEVICE
    raise TypeError("points must be a numpy array or a CUDA torch tensor")


class Context:
    def __init__(self, device=0, params=None, **kw):
        self._lib = lib()
        self.params = params if params is not None else default_params(**kw)
        self._h = C.c_void_p()
        rc = self._lib.glio_create(C.c_int(device), C.byref(self.params), C.byref(self._h))
        if rc != 0:
            msg = self._lib.glio_last_error(None)
            raise GlioError(f"glio_create failed ({rc}): {msg.decode() if msg else ''}")
        self._keep = []
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._lib.glio_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc != 0:
            msg = self._lib.glio_last_error(self._h)
            raise GlioError(f"glio error {rc}: {msg.decode() if msg else ''}")

    @property
    def stream(self):
        return self._lib.glio_stream(self._h)

    @property
    def launch_count(self):
        return int(self._lib.glio_launch_count(self._h))

    def synchronize(self):
        self._chk(self._lib.glio_synchronize(self._h))

    def lidar_pose(self, pose_body):
        pb = np.ascontiguousarray(pose_body, np.float64)
        t2 = np.zeros(3); q2 = np.zeros(4)
        self._lib.glio_lidar_pose(C.byref(self.params), _ptr(pb), _ptr(t2), _ptr(q2))
        return t2, q2

    # every kernel name the library hands its launch counter (tests/test_profile_names.py keeps this list complete)
    KERNELS = ["k_sp_bounds", "k_sp_consts", "k_sp_classify", "k_sp_ranges", "k_sp_emit",
               "k_feat_curvature", "k_feat_select", "k_feat_voxel", "k_feat_offsets", "k_feat_gather", "k_knn_box", "k_plane_fit", "k_plane_fit_pair",
               "k_eval_unary", "k_eval_unary_cost", "k_unary_residuals", "k_eval_edge", "k_eval_edge_cost", "k_transform_hist", "k_order_scatter",
               "k_compact", "k_flags", "k_cell_hist", "k_cell_scatter", "k_load_bounds", "k_scan_block", "k_scan_add",
               "k_eval_binary", "k_eval_binary_cost", "k_bin_assemble", "k_bin_pair_sums", "k_gather_sel", "k_sel_sample",
               "k_lm_transform", "k_vox_hist", "k_vox_scatter", "k_vox_sort", "k_vox_flags", "k_vox_centroid", "k_init_bounds",
               "k_line_fit", "k_compact_edge", "k_seg_counts", "k_line_fit_pair", "k_eval_binary_edge", "k_eval_binary_edge_cost",
               "k_bin_pair_add", "k_odom_publish",
               "k_lc_load", "k_lc_qhist", "k_lc_qscatter", "k_lc_init", "k_lc_nn", "k_lc_compact", "k_lc_sum0",
               "k_lc_sum1", "k_lc_means", "k_lc_solve", "k_lc_transform", "k_lc_final", "k_lc_fitness",
               "k_vs_key", "k_vs_hist", "k_vs_scatter", "k_vs_heads", "k_vs_centroid", "k_vs_pack", "k_gm_transform",
               "k_pose_pair_sums", "k_pose_pair_sums_cost", "k_pose_assemble",
               "k_psr_pair_sums", "k_psr_pair_sums_cost", "k_psr_assemble",
               "k_imu_pair_sums", "k_imu_pair_sums_cost", "k_imu_pair_sums_ambient", "k_imu_assemble",
               "k_band_chol_solve", "k_band_assemble", "k_band_assemble_g", "k_band_scale", "k_band_shift", "k_band_symv",
               "k_bcr_gather", "k_bcr_potrf", "k_bcr_trsm", "k_bcr_update", "k_bcr_back", "k_bcr_finish"]

    def lib_profile(self, on):
        self._chk(self._lib.glio_profile_enable(self._h, C.c_int(1 if on else 0)))

    def lib_profile_read(self):
        out = {}
        for k in self.KERNELS:
            ms = C.c_double(0); n = C.c_int64(0)
            self._chk(self._lib.glio_profile_get(self._h, k.encode(), C.byref(ms), C.byref(n)))
            if n.value:
                out[k] = (ms.value, int(n.value))
        return out

    def knn_fallback_queries(self, reset=False):
        """Queries the kNN search handed to a second pass: always 0, the box search has none (glio_get_stats)."""
        n = C.c_int64(0)
        self._chk(self._lib.glio_get_stats(self._h, C.byref(n), C.c_int(1 if reset else 0)))
        return int(n.value)

    def get_match_counts(self, W, active=True):
        nm = np.zeros(W, np.int64); na = np.zeros(W, np.int64)
        self._chk(self._lib.glio_get_match_counts(self._h, C.c_int(W), _ptr(nm), _ptr(na)))
        return na if active else nm

    # ---- K0
    def set_map(self, xyz):
        keep, p, n, stride, mem = _points_arg(xyz)
        self._map_keep = keep
        self._chk(self._lib.glio_set_map(self._h, p, C.c_int64(n), C.c_int(stride), C.c_int(mem)))

    def map_prefetch(self, xyz):
        keep, p, n, stride, mem = _points_arg(xyz)
        assert mem == HOST
        self._map_pf_keep = keep
        self._chk(self._lib.glio_map_prefetch(self._h, p, C.c_int64(n), C.c_int(stride)))

    # ---- K1
    # ---- local map maintenance on the device
    def localmap_clear(self):
        self._chk(self._lib.glio_localmap_clear(self._h))

    def localmap_push(self, cloud_xyz, t, q, at_front=False):
        keep, p, n, stride, mem = _points_arg(cloud_xyz)
        t = np.ascontiguousarray(t, np.float64); q = np.ascontiguousarray(q, np.float64)
        self._chk(self._lib.glio_localmap_push(self._h, C.c_int(1 if at_front else 0), p, C.c_int64(n), C.c_int(stride), C.c_int(mem), _ptr(t), _ptr(q)))

    def localmap_pop_front(self):
        self._chk(self._lib.glio_localmap_pop_front(self._h))

    def localmap_size(self):
        nf = C.c_int(0); npnt = C.c_int64(0)
        self._chk(self._lib.glio_localmap_size(self._h, C.byref(nf), C.byref(npnt)))
        return nf.value, int(npnt.value)

    def localmap_build(self, leaf=0.4):
        n = C.c_int64(0)
        self._chk(self._lib.glio_localmap_build(self._h, C.c_float(leaf), C.byref(n)))
        return int(n.value)

    def get_map(self):
        n = C.c_int64(0)
        self._chk(self._lib.glio_get_map(self._h, C.c_int64(0), None, C.byref(n)))
        out = np.empty((int(n.value), 3), np.float32)
        self._chk(self._lib.glio_get_map(self._h, C.c_int64(len(out)), _ptr(out), C.byref(n)))
        return out

    def voxel_filter(self, xyz, leaf, out="host"):
        """pcl::VoxelGrid(leaf) of any cloud on the device (glio_voxel_filter; downSampleCloud's ds_filter_surf, Estimator.cpp:3628-3630).
        xyz: (n, stride) float32 numpy array or CUDA tensor with x, y, z in columns 0..2.  Returns (points (m, 3) float32, filtered):
        filtered is False when PCL's leaf-size check passed the input through.  With out="device" the points are a CUDA tensor that
        window_set_scan and LoopClosure.add_keyframe take as they are."""
        if out not in ("host", "device"):
            raise ValueError("out must be 'host' or 'device'")
        if _npts(xyz):
            keep, p, n, stride, mem = _points_arg(xyz)
        else:
            p, n, stride, mem = None, 0, 3, HOST
        buf, optr, omem = _vs_output(self, n, out)
        m = C.c_int64(0); f = C.c_int32(0)
        self._chk(self._lib.glio_voxel_filter(self._h, p, C.c_int64(n), C.c_int(stride), C.c_int(mem), C.c_float(leaf), C.c_int64(n), optr,
                                              C.c_int(omem), C.byref(m), C.byref(f)))
        return buf[:m.value], bool(f.value)

    def assoc_scan_to_map(self, slot, scan_xyz, t, q):
        keep, p, n, stride, mem = _points_arg(scan_xyz)
        self._keep.append(keep); self._keep = self._keep[-64:]
        t = np.ascontiguousarray(t, np.float64); q = np.ascontiguousarray(q, np.float64)
        nm = C.c_int64(0)
        self._chk(self._lib.glio_assoc_scan_to_map(self._h, C.c_int(slot), p, C.c_int64(n), C.c_int(stride), C.c_int(mem),
                                                   _ptr(t), _ptr(q), C.byref(nm)))
        return int(nm.value)

    def window_set_scans(self, scans):
        args = [_points_arg(s) for s in scans]
        self._scan_keep = [a[0] for a in args]
        W = len(args)
        ptrs = (C.c_void_p * W)(*[a[1] for a in args])
        Q = (C.c_int64 * W)(*[a[2] for a in args])
        strides = {a[3] for a in args}; mems = {a[4] for a in args}
        assert len(strides) == 1 and len(mems) == 1
        self._chk(self._lib.glio_window_set_scans(self._h, C.c_int(W), ptrs, Q, C.c_int(strides.pop()), C.c_int(mems.pop())))

    def window_set_scan(self, slot, scan):
        keep, p, n, stride, mem = _points_arg(scan)
        if not hasattr(self, "_slot_keep"):
            self._slot_keep = {}
        self._slot_keep[slot] = keep
        self._chk(self._lib.glio_window_set_scan(self._h, C.c_int(slot), p, C.c_int64(n), C.c_int(stride), C.c_int(mem)))

    def window_slide(self, W):
        self._chk(self._lib.glio_window_slide(self._h, C.c_int(W)))

    def window_associate(self, poses_body):
        pb = np.ascontiguousarray(poses_body, np.float64).reshape(-1, 7)
        W = len(pb)
        nm = np.zeros(W, np.int64)
        self._chk(self._lib.glio_window_associate(self._h, C.c_int(W), _ptr(pb), _ptr(nm)))
        return nm

    def get_matches(self, slot, capacity):
        cp = np.empty((capacity, 3), np.float32); nsd = np.empty((capacity, 4), np.float32)
        w = np.empty(capacity, np.float32); src = np.empty(capacity, np.int32)
        n = C.c_int64(0)
        self._chk(self._lib.glio_get_matches(self._h, C.c_int(slot), C.c_int64(capacity), _ptr(cp), _ptr(nsd), _ptr(w), _ptr(src), C.byref(n)))
        n = int(n.value)
        return dict(cp=cp[:n], nsd=nsd[:n], weight=w[:n], src=src[:n], n=n)

    def get_assoc_debug(self, slot, Q):
        out = dict(status=np.empty(Q, np.uint8), idx5=np.empty((Q, 5), np.int32), sqd5=np.empty((Q, 5), np.float32),
                   pm=np.empty((Q, 3), np.float32), plane=np.empty((Q, 4), np.float64))
        self._chk(self._lib.glio_get_assoc_debug(self._h, C.c_int(slot), C.c_int64(Q), _ptr(out["status"]), _ptr(out["idx5"]),
                                                 _ptr(out["sqd5"]), _ptr(out["pm"]), _ptr(out["plane"])))
        return out

    def select(self, slot, keep):
        if keep is None:
            self._chk(self._lib.glio_select(self._h, C.c_int(slot), None, C.c_int64(-1)))
            return
        k = np.ascontiguousarray(keep, np.int32)
        self._chk(self._lib.glio_select(self._h, C.c_int(slot), _ptr(k), C.c_int64(len(k))))

    # ---- K2
    def set_matches(self, slot, cp, nsd, weight):
        """glio_set_matches: upload a slot's plane correspondences as they are (cp (n, 3), nsd (n, 4) = (n, d), weight (n,),
        all float32) instead of associating them; score = lidar_const * weight."""
        cp = np.ascontiguousarray(cp, np.float32).reshape(-1, 3); nsd = np.ascontiguousarray(nsd, np.float32).reshape(-1, 4)
        w = np.ascontiguousarray(weight, np.float32).ravel()
        if not (len(cp) == len(nsd) == len(w)):
            raise ValueError("cp, nsd and weight must have the same length")
        self._chk(self._lib.glio_set_matches(self._h, C.c_int(slot), _ptr(cp), _ptr(nsd), _ptr(w), C.c_int64(len(w))))

    def eval_unary(self, poses_body, jac_kind=0, want_jac=True):
        pb = np.ascontiguousarray(poses_body, np.float64).reshape(-1, 7)
        W = len(pb)
        H = np.zeros((W, 6, 6)) if want_jac else None
        g = np.zeros((W, 6)) if want_jac else None
        cost = np.zeros(W)
        self._chk(self._lib.glio_eval_unary(self._h, C.c_int(W), _ptr(pb), C.c_int(jac_kind), _ptr(H), _ptr(g), _ptr(cost)))
        return dict(H=H, g=g, cost=cost)

    def eval_unary_residuals(self, slot, pose_body, capacity, jac_kind=0):
        pb = np.ascontiguousarray(pose_body, np.float64)
        r = np.empty(capacity); J = np.empty((capacity, 6)); n = C.c_int64(0)
        self._chk(self._lib.glio_eval_unary_residuals(self._h, C.c_int(slot), _ptr(pb), C.c_int(jac_kind), C.c_int64(capacity),
                                                      _ptr(r), _ptr(J), C.byref(n)))
        n = int(n.value)
        return r[:n], J[:n]


# ---------------------------------------------------------------------------------------------------
# minimizer iteration (ceres::Solve replacement for the window problem) and stand-in host factors
# ---------------------------------------------------------------------------------------------------
class SolverOptions(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int32), ("dogleg_type", C.c_int32), ("use_nonmonotonic_steps", C.c_int32),
                ("max_consecutive_nonmonotonic_steps", C.c_int32), ("initial_trust_region_radius", C.c_double),
                ("max_trust_region_radius", C.c_double), ("min_trust_region_radius", C.c_double),
                ("min_relative_decrease", C.c_double), ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double),
                ("max_num_consecutive_invalid_steps", C.c_int32), ("jacobi_scaling", C.c_int32),
                ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double),
                ("fuse_candidate_jacobian", C.c_int32), ("trust_region_strategy", C.c_int32)]


class Iteration(C.Structure):
    _fields_ = [("iteration", C.c_int32), ("step_is_valid", C.c_int32), ("step_is_successful", C.c_int32), ("reserved", C.c_int32),
                ("cost", C.c_double), ("cost_change", C.c_double), ("gradient_max_norm", C.c_double), ("gradient_norm", C.c_double),
                ("step_norm", C.c_double), ("relative_decrease", C.c_double), ("trust_region_radius", C.c_double), ("mu", C.c_double)]


class SolverSummary(C.Structure):
    _fields_ = [("termination", C.c_int32), ("num_iterations", C.c_int32), ("num_successful_steps", C.c_int32),
                ("num_unsuccessful_steps", C.c_int32), ("num_evaluations", C.c_int32), ("num_jacobian_evaluations", C.c_int32),
                ("num_linear_solves", C.c_int32), ("num_valid_steps", C.c_int32), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("eval_seconds", C.c_double), ("linear_solver_seconds", C.c_double),
                ("total_seconds", C.c_double), ("message", C.c_char * 128)]


HOST_FACTORS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int,
                              C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))


def default_solver_options(**kw):
    o = SolverOptions()
    lib().glio_default_solver_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def iterations_to_dicts(log, n):
    names = [f[0] for f in Iteration._fields_ if f[0] != "reserved"]
    return [{k: getattr(log[i], k) for k in names} for i in range(n)]


class HostFactorSet:
    """Stand-in host factors (prior / between / range) evaluated analytically on the CPU by the library."""

    def __init__(self):
        L = lib()
        L.glio_hf_create.restype = C.c_void_p
        L.glio_hf_destroy.argtypes = [C.c_void_p]
        self._lib = L
        self._h = C.c_void_p(L.glio_hf_create())

    def add_prior(self, kf, t0, q0, sb0, sqrt_w):
        a = [np.ascontiguousarray(v, np.float64) if v is not None else None for v in (t0, q0, sb0, sqrt_w)]
        self._lib.glio_hf_add_prior(self._h, C.c_int(kf), _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]))

    def add_between(self, i, j, dp, dq, dv, dt, sqrt_w):
        a = [np.ascontiguousarray(v, np.float64) for v in (dp, dq, dv, sqrt_w)]
        self._lib.glio_hf_add_between(self._h, C.c_int(i), C.c_int(j), _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), C.c_double(dt), _ptr(a[3]))

    def add_range(self, kf, lever, sat, rho, w):
        a = [np.ascontiguousarray(v, np.float64) for v in (lever, sat)]
        self._lib.glio_hf_add_range(self._h, C.c_int(kf), _ptr(a[0]), _ptr(a[1]), C.c_double(rho), C.c_double(w))

    def set_marg_prior(self, prior):
        """Attach a MargPrior (or None) to this factor set: it then acts as the MarginalizationFactor of the window."""
        self._prior_keep = prior
        rc = self._lib.glio_hf_set_marg_prior(self._h, prior._h if prior is not None else None)
        assert rc == 0

    def marg_half_bandwidth(self):
        return int(self._lib.glio_hf_marg_half_bandwidth(self._h))

    def marg_evaluate(self, poses, speed_bias):
        """The non-LiDAR part of MarginalizationInfo's A, b (marginalisation ordering, N = 6W + 18)."""
        pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); W = len(pb)
        sb = np.ascontiguousarray(speed_bias, np.float64).reshape(W, 9)
        N = 6 * W + 18
        A = np.zeros((N, N)); b = np.zeros(N)
        rc = self._lib.glio_hf_marg_evaluate(self._h, C.c_int(W), _ptr(pb), _ptr(sb), _ptr(A), _ptr(b))
        assert rc == 0
        return A, b

    def evaluate(self, poses, speed_bias=None, want_jac=True):
        pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); W = len(pb)
        sb = None if speed_bias is None else np.ascontiguousarray(speed_bias, np.float64).reshape(W, 9)
        n = W * (15 if sb is not None else 6)
        H = np.zeros((n, n)); g = np.zeros(n); c = np.zeros(1)
        rc = self._lib.glio_hf_evaluate(self._h, C.c_int(W), _ptr(pb), _ptr(sb), C.c_int(1 if want_jac else 0), _ptr(H), _ptr(g), _ptr(c))
        assert rc == 0
        return H, g, float(c[0])

    @property
    def callback(self):
        return C.cast(self._lib.glio_hf_evaluate, HOST_FACTORS_FN), self._h

    def __del__(self):
        try:
            if self._h:
                self._lib.glio_hf_destroy(self._h); self._h = None
        except Exception:
            pass


def _extract_features(self, cloud_xyzi, scan_start, scan_end, ds_rate=1, edge_thres=1.0, surf_thres=0.1, ds_v=0.4, intensity_offset=None):
    """Preprocessing::cloudHandler's feature extraction (GLIO/src/Preprocessing.cpp:529-655) on the device."""
    keep, p, n, stride, mem = _points_arg(cloud_xyzi)
    ioff = intensity_offset if intensity_offset is not None else (4 if stride == 8 else 3)
    ss = np.ascontiguousarray(scan_start, np.int32); se = np.ascontiguousarray(scan_end, np.int32); S = len(ss)
    out = dict(curvature=np.empty(n, np.float32), label=np.empty(n, np.int8), sharp=np.empty(12 * S, np.int32), less_sharp=np.empty(60 * S, np.int32),
               flat=np.empty(24 * S, np.int32), less_flat=np.empty(n, np.int32), less_flat_ds=np.empty((n, 4), np.float32))
    cnt = [C.c_int64(0) for _ in range(5)]
    self._chk(self._lib.glio_extract_features(self._h, p, C.c_int64(n), C.c_int(stride), C.c_int(ioff), C.c_int(mem), C.c_int(S), _ptr(ss), _ptr(se), C.c_int(ds_rate),
                                              C.c_double(edge_thres), C.c_double(surf_thres), C.c_float(ds_v), _ptr(out["curvature"]), _ptr(out["label"]),
                                              _ptr(out["sharp"]), C.byref(cnt[0]), _ptr(out["less_sharp"]), C.byref(cnt[1]), _ptr(out["flat"]), C.byref(cnt[2]),
                                              _ptr(out["less_flat"]), C.byref(cnt[3]), _ptr(out["less_flat_ds"]), C.byref(cnt[4])))
    for k, c in zip(("sharp", "less_sharp", "flat", "less_flat", "less_flat_ds"), cnt):
        out[k] = out[k][:c.value]
    return out


Context.extract_features = _extract_features


class ImuState(C.Structure):
    """glio_imu_state: idx_imu, current_time_imu, gyr_0, first_imu of Preprocessing (GLIO/src/Preprocessing.cpp:33-39).
    A fresh (zero) state has seen no IMU sample yet."""
    _fields_ = [("idx_imu", C.c_int64), ("current_time_imu", C.c_double), ("gyr_0", C.c_double * 3), ("first_imu", C.c_int32),
                ("reserved", C.c_int32)]


def imu_sweep_rotation(state, stamps, gyro, t_scan_next):
    """The sweep's IMU rotation qIMU (w, x, y, z): processIMU + solveRotation (Preprocessing.cpp:202-259) over the IMU buffer
    received so far (stamps[n] seconds, gyro[n, 3] rad/s) up to t_scan_next.  `state` (ImuState) carries over between sweeps."""
    st = np.ascontiguousarray(stamps, np.float64).ravel(); g = np.ascontiguousarray(gyro, np.float64).reshape(-1, 3)
    if len(g) != len(st):
        raise ValueError("stamps and gyro must have the same number of samples")
    q = np.zeros(4)
    L = lib()
    rc = L.glio_imu_sweep_rotation(C.byref(state), _ptr(st), _ptr(g), C.c_int64(len(st)), C.c_double(t_scan_next), _ptr(q))
    if rc != 0:
        msg = L.glio_last_error(None)
        raise GlioError(f"glio_imu_sweep_rotation failed ({rc}): {msg.decode() if msg else ''}")
    return q


def _prepare_scan(self, raw, n_scans, q_imu=None, q_lb=None, out="host"):
    """Preprocessing::cloudHandler's sweep preparation (GLIO/src/Preprocessing.cpp:387-526) on the device: NaN / 3 m filters, ring
    assignment, relative time and IMU de-skew, rings concatenated.  raw: (n, stride) float32 numpy array or CUDA tensor with x, y, z
    in columns 0..2 (pcl::PointXYZI: stride 8).  q_imu: the sweep's rotation (imu_sweep_rotation), None = identity; q_lb: the
    extrinsic, default synth.Q_LB.  Returns (cloud (m, 4) x,y,z,intensity, scan_start, scan_end); with out="device" the cloud
    is a CUDA tensor that extract_features takes as it is."""
    if out not in ("host", "device"):
        raise ValueError("out must be 'host' or 'device'")
    if q_lb is None:
        from . import synth
        q_lb = synth.Q_LB
    keep, p, n, stride, mem = _points_arg(raw)
    qi = None if q_imu is None else np.ascontiguousarray(q_imu, np.float64)
    ql = np.ascontiguousarray(q_lb, np.float64)
    ss = np.empty(n_scans, np.int32); se = np.empty(n_scans, np.int32)
    m = C.c_int64(0)
    if out == "device":
        import torch
        dev = torch.device("cuda", self.device)           # the context's GPU: the library rejects memory of any other
        buf = torch.empty((max(n, 1), 4), dtype=torch.float32, device=dev)
        # the buffer comes from torch's caching allocator on torch's stream, the library writes it on the context's stream:
        # let torch's pending work on that memory finish first (the library call itself returns only when its writes are done)
        torch.cuda.current_stream(dev).synchronize()
        optr, omem = C.c_void_p(buf.data_ptr()), DEVICE
    else:
        buf = np.empty((n, 4), np.float32)
        optr, omem = _ptr(buf), HOST
    self._chk(self._lib.glio_prepare_scan(self._h, p, C.c_int64(n), C.c_int(stride), C.c_int(mem), C.c_int(n_scans), _ptr(qi), _ptr(ql),
                                          optr, C.c_int(omem), C.c_int64(n), C.byref(m), _ptr(ss), _ptr(se)))
    return buf[:m.value], ss, se


def _scanprep_guard_hits(self, reset=False):
    """glio_scanprep_stats: atanf / atan2f evaluations of prepare_scan decided in double-double since the last reset."""
    h = C.c_int64(0)
    self._chk(self._lib.glio_scanprep_stats(self._h, C.byref(h), C.c_int(1 if reset else 0)))
    return int(h.value)


Context.prepare_scan = _prepare_scan
Context.scanprep_guard_hits = _scanprep_guard_hits


HOST_MARG_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))


class MargPrior:
    """glio_marg_prior: linearized_jacobians / residuals + keep_block_data of MarginalizationInfo (next window's numbering)."""

    def __init__(self, handle, lib_):
        self._h = handle; self._lib = lib_
        n = C.c_int(0); W = C.c_int(0)
        self._lib.glio_marg_prior_size(self._h, C.byref(n), C.byref(W))
        self.n, self.W = n.value, W.value

    @classmethod
    def from_arrays(cls, W, lin_jac, lin_res, x0_pose, x0_sb):
        L = lib()
        a = [np.ascontiguousarray(v, np.float64) for v in (lin_jac, lin_res, x0_pose, x0_sb)]
        h = L.glio_marg_prior_create(C.c_int(W), _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]))
        assert h
        return cls(C.c_void_p(h), L)

    def arrays(self):
        n, W = self.n, self.W
        out = dict(W=W, lin_jac=np.zeros((n, n)), lin_res=np.zeros(n), x0_pose=np.zeros((W - 1, 7)), x0_sb=np.zeros(9), A_info=np.zeros((n, n)), b_info=np.zeros(n))
        self._lib.glio_marg_prior_get(self._h, _ptr(out["lin_jac"]), _ptr(out["lin_res"]), _ptr(out["x0_pose"]), _ptr(out["x0_sb"]), _ptr(out["A_info"]), _ptr(out["b_info"]))
        return out

    def __del__(self):
        try:
            if self._h:
                self._lib.glio_marg_prior_destroy(self._h); self._h = None
        except Exception:
            pass


def _window_marginalize(self, poses, speed_bias, host_factors=None, eps=1e-8):
    """MarginalizationInfo::PreMarginalize + Marginalize of KF0 (Estimator.cpp:2462-2608): LiDAR blocks from the device, the
    other factors from `host_factors` (a HostFactorSet).  Returns a MargPrior for the next window."""
    pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); W = len(pb)
    sb = np.ascontiguousarray(speed_bias, np.float64).reshape(W, 9)
    if host_factors is None:
        fn, user = C.cast(None, HOST_MARG_FN), None
    else:
        fn, user = C.cast(self._lib.glio_hf_marg_evaluate, HOST_MARG_FN), host_factors._h
    out = C.c_void_p()
    self._chk(self._lib.glio_window_marginalize(self._h, C.c_int(W), _ptr(pb), _ptr(sb), fn, user, C.c_double(eps), C.byref(out)))
    return MargPrior(out, self._lib)


Context.window_marginalize = _window_marginalize


class MargJob:
    """glio_marg_job: a marginalisation whose host half runs on the context's worker thread; wait() joins it -> MargPrior."""

    def __init__(self, ctx, handle, keep):
        self._ctx = ctx; self._h = handle; self._keep = keep          # keep: the arrays / factor set the job may still read

    def wait(self):
        assert self._h is not None, "job already waited for"
        out = C.c_void_p()
        h, self._h = self._h, None
        self._ctx._chk(self._ctx._lib.glio_marg_job_wait(h, C.byref(out)))
        self._keep = None
        return MargPrior(out, self._ctx._lib)


def _window_marginalize_async(self, poses, speed_bias, host_factors=None, eps=1e-8):
    """glio_window_marginalize_async: queues the device half, runs the host callback, returns a MargJob at once."""
    pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); W = len(pb)
    sb = np.ascontiguousarray(speed_bias, np.float64).reshape(W, 9)
    if host_factors is None:
        fn, user = C.cast(None, HOST_MARG_FN), None
    else:
        fn, user = C.cast(self._lib.glio_hf_marg_evaluate, HOST_MARG_FN), host_factors._h
    job = C.c_void_p()
    self._chk(self._lib.glio_window_marginalize_async(self._h, C.c_int(W), _ptr(pb), _ptr(sb), fn, user, C.c_double(eps), C.byref(job)))
    return MargJob(self, job, (pb, sb, host_factors))


Context.window_marginalize_async = _window_marginalize_async


def _window_solve(self, poses, speed_bias=None, host_factors=None, options=None, max_log=64, band=None):
    """ceres::Solve for the window problem (Estimator.cpp:2424-2433).  Returns dict(poses, speed_bias, summary, iterations, steps)."""
    pb = np.array(poses, np.float64).reshape(-1, 7).copy(); W = len(pb)
    sb = None if speed_bias is None else np.array(speed_bias, np.float64).reshape(W, 9).copy()
    n = W * (15 if sb is not None else 6)
    opt = options if options is not None else default_solver_options()
    summ = SolverSummary(); log = (Iteration * max_log)(); steps = np.zeros((max_log, n))
    if host_factors is None:
        fn, user = C.cast(None, HOST_FACTORS_FN), None
    elif isinstance(host_factors, HostFactorSet):
        fn, user = host_factors.callback
    else:
        fn, user = host_factors, None          # a HOST_FACTORS_FN instance
    if band is not None and isinstance(host_factors, HostFactorSet):
        # host factors straight into band storage (band = half bandwidth, e.g. 29 for prior + chain with speed-bias)
        bfn = C.cast(self._lib.glio_hf_evaluate_band, HOST_FACTORS_BAND_FN)
        self._chk(self._lib.glio_window_solve_band(self._h, C.c_int(W), _ptr(pb), _ptr(sb), bfn, C.c_int(band), host_factors._h, C.byref(opt),
                                                   C.byref(summ), log, C.c_int(max_log), _ptr(steps), C.c_int64(steps.size)))
    else:
        self._chk(self._lib.glio_window_solve(self._h, C.c_int(W), _ptr(pb), _ptr(sb), fn, user, C.byref(opt), C.byref(summ), log,
                                              C.c_int(max_log), _ptr(steps), C.c_int64(steps.size)))
    return dict(poses=pb, speed_bias=sb, summary=summ, iterations=iterations_to_dicts(log, min(summ.num_iterations, max_log)),
                steps=steps[:summ.num_valid_steps])


Context.window_solve = _window_solve


# ---------------------------------------------------------------------------------------------------
# batch (scan-to-multiscan) path
# ---------------------------------------------------------------------------------------------------
def _batch_set_frame(self, frame, scan_xyz, pose):
    keep, p, n, stride, mem = _points_arg(scan_xyz)
    if not hasattr(self, "_frame_keep"):
        self._frame_keep = {}
    self._frame_keep[frame] = keep
    ps = np.ascontiguousarray(pose, np.float64)
    self._chk(self._lib.glio_batch_set_frame(self._h, C.c_int(frame), p, C.c_int64(n), C.c_int(stride), C.c_int(mem), _ptr(ps)))


def _batch_set_pose(self, frame, pose):
    ps = np.ascontiguousarray(pose, np.float64)
    self._chk(self._lib.glio_batch_set_pose(self._h, C.c_int(frame), _ptr(ps)))


def _batch_associate_pairs(self, cur, oth):
    cur = np.ascontiguousarray(cur, np.int32); oth = np.ascontiguousarray(oth, np.int32)
    nm = np.zeros(len(cur), np.int64)
    self._chk(self._lib.glio_batch_associate_pairs(self._h, _ptr(cur), _ptr(oth), C.c_int64(len(cur)), _ptr(nm)))
    return nm


def _batch_get_matches(self, cur, oth, capacity):
    cp = np.empty((capacity, 3), np.float32); w = np.empty(capacity, np.float32); nc = np.empty((capacity, 6), np.float64)
    src = np.empty(capacity, np.int32); n = C.c_int64(0)
    self._chk(self._lib.glio_batch_get_matches(self._h, C.c_int(cur), C.c_int(oth), C.c_int64(capacity), _ptr(cp), _ptr(w), _ptr(nc), _ptr(src), C.byref(n)))
    n = int(n.value)
    return dict(cp=cp[:n], weight=w[:n], normal_cent=nc[:n], src=src[:n], n=n)


def _batch_select(self, cur, oth, keep):
    if keep is None:
        self._chk(self._lib.glio_batch_select(self._h, C.c_int(cur), C.c_int(oth), None, C.c_int64(-1)))
        return
    k = np.ascontiguousarray(keep, np.int32)
    self._chk(self._lib.glio_batch_select(self._h, C.c_int(cur), C.c_int(oth), _ptr(k), C.c_int64(len(k))))


def _pair_table(self, pair_list):
    """The two int32 columns of a pair table read through a glio_*pair_list entry point: the count, then the table."""
    n = C.c_int64(0)
    self._chk(pair_list(self._h, C.c_int64(0), None, None, C.byref(n)))
    a = np.zeros(n.value, np.int32); b = np.zeros(n.value, np.int32)
    self._chk(pair_list(self._h, C.c_int64(n.value), _ptr(a), _ptr(b), C.byref(n)))
    return a, b


def _eval_blocks(self, eval_fn, pair_list, poses, want_jac):
    """The blocks of a glio_eval_* entry point, Hoff sized by the pair table of pair_list: Hdiag (K,6,6), Hoff (P,6,6) and g (K,6)
    (None without want_jac), and the cost."""
    pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); K = len(pb)
    n = C.c_int64(0)
    self._chk(pair_list(self._h, C.c_int64(0), None, None, C.byref(n)))
    P = int(n.value)
    Hd = np.zeros((K, 6, 6)) if want_jac else None; Ho = np.zeros((P, 6, 6)) if want_jac else None
    g = np.zeros((K, 6)) if want_jac else None; cost = np.zeros(1)
    self._chk(eval_fn(self._h, C.c_int(K), _ptr(pb), _ptr(Hd), _ptr(Ho), _ptr(g), _ptr(cost)))
    return dict(Hdiag=Hd, Hoff=Ho, g=g, cost=float(cost[0]))


def _batch_pair_list(self):
    return _pair_table(self, self._lib.glio_batch_pair_list)


def _batch_clear(self):
    self._chk(self._lib.glio_batch_clear(self._h))


def _eval_binary(self, poses, want_jac=True):
    return _eval_blocks(self, self._lib.glio_eval_binary, self._lib.glio_batch_pair_list, poses, want_jac)


HOST_FACTORS_BAND_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int,
                                   C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double))
ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p)


def batch_solver_options(**kw):
    """Estimator.cpp:3275-3281: SUBSPACE_DOGLEG, nonmonotonic steps, max_num_iter (100 in the shipped yaml)."""
    base = dict(dogleg_type=1, use_nonmonotonic_steps=1, max_num_iterations=100)
    base.update(kw)
    return default_solver_options(**base)


def _batch_declare_pairs(self, cur, oth):
    cur = np.ascontiguousarray(cur, np.int32); oth = np.ascontiguousarray(oth, np.int32)
    self._chk(self._lib.glio_batch_declare_pairs(self._h, _ptr(cur), _ptr(oth), C.c_int64(len(cur))))


def _batch_solve(self, poses, speed_bias=None, host_factors=None, options=None, max_log=256):
    pb = np.array(poses, np.float64).reshape(-1, 7).copy(); K = len(pb)
    sb = None if speed_bias is None else np.array(speed_bias, np.float64).reshape(K, 9).copy()
    n = K * (15 if sb is not None else 6)
    opt = options if options is not None else batch_solver_options()
    summ = SolverSummary(); log = (Iteration * max_log)(); steps = np.zeros((max_log, n))
    if host_factors is None:
        fn, user = C.cast(None, HOST_FACTORS_BAND_FN), None
    else:
        fn, user = C.cast(self._lib.glio_hf_evaluate_band, HOST_FACTORS_BAND_FN), host_factors._h
    self._chk(self._lib.glio_batch_solve(self._h, C.c_int(K), _ptr(pb), _ptr(sb), fn, user, C.byref(opt), C.byref(summ), log,
                                         C.c_int(max_log), _ptr(steps), C.c_int64(steps.size)))
    return dict(poses=pb, speed_bias=sb, summary=summ, iterations=iterations_to_dicts(log, min(summ.num_iterations, max_log)),
                steps=steps[:summ.num_valid_steps])


def _set_allreduce(self, fn, user=None):
    """fn: an ALLREDUCE_FN instance (or a raw function pointer from libglio_nccl.so); keeps a reference alive."""
    self._allreduce_keep = (fn, user)
    self._chk(self._lib.glio_set_allreduce(self._h, fn, user))


def _set_edges(self, slot, cp, pa, pb, s):
    cp = np.ascontiguousarray(cp, np.float32).reshape(-1, 3); pa = np.ascontiguousarray(pa, np.float32).reshape(-1, 3)
    pb = np.ascontiguousarray(pb, np.float32).reshape(-1, 3); s = np.ascontiguousarray(s, np.float64)
    self._chk(self._lib.glio_set_edges(self._h, C.c_int(slot), _ptr(cp), _ptr(pa), _ptr(pb), _ptr(s), C.c_int64(len(s))))


def _eval_edge(self, poses_body, want_jac=True):
    pb = np.ascontiguousarray(poses_body, np.float64).reshape(-1, 7); W = len(pb)
    H = np.zeros((W, 6, 6)) if want_jac else None; g = np.zeros((W, 6)) if want_jac else None; cost = np.zeros(W)
    self._chk(self._lib.glio_eval_edge(self._h, C.c_int(W), _ptr(pb), _ptr(H), _ptr(g), _ptr(cost)))
    return dict(H=H, g=g, cost=cost)


Context.set_edges = _set_edges
Context.eval_edge = _eval_edge

EDGE_VALID, EDGE_FAIL_RADIUS, EDGE_FAIL_LINE = 0, 1, 2


class EdgeOptions(C.Structure):
    _fields_ = [("max_sqdist", C.c_double), ("min_ratio", C.c_double), ("half_length", C.c_double), ("score", C.c_double)]


def edge_default_options(**kw):
    """glio_edge_default_options (max_sqdist 1.0, min_ratio 3.0, half_length 0.1, score 1.0), fields overridden by keyword."""
    o = EdgeOptions()
    lib().glio_edge_default_options(C.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise AttributeError(k)
        setattr(o, k, float(v))
    return o


def _set_edge_map(self, xyz):
    """glio_set_edge_map: the corner map (its own grid; the surf map is untouched)."""
    keep, p, n, stride, mem = _points_arg(xyz)
    self._edge_map_keep = keep
    self._chk(self._lib.glio_set_edge_map(self._h, p, C.c_int64(n), C.c_int(stride), C.c_int(mem)))


def _edge_localmap_clear(self):
    self._chk(self._lib.glio_edge_localmap_clear(self._h))


def _edge_localmap_push(self, cloud_xyz, t, q, at_front=False):
    keep, p, n, stride, mem = _points_arg(cloud_xyz)
    t = np.ascontiguousarray(t, np.float64); q = np.ascontiguousarray(q, np.float64)
    self._chk(self._lib.glio_edge_localmap_push(self._h, C.c_int(1 if at_front else 0), p, C.c_int64(n), C.c_int(stride), C.c_int(mem),
                                                _ptr(t), _ptr(q)))


def _edge_localmap_pop_front(self):
    self._chk(self._lib.glio_edge_localmap_pop_front(self._h))


def _edge_localmap_build(self, leaf=0.2):
    """Concatenate the corner local map, VoxelGrid(leaf) (leaf <= 0: none) and make it the corner map; returns its size."""
    n = C.c_int64(0)
    self._chk(self._lib.glio_edge_localmap_build(self._h, C.c_float(leaf), C.byref(n)))
    return int(n.value)


def _window_set_edge_scan(self, slot, xyz):
    """glio_window_set_edge_scan: one keyframe's corner points (host buffers stay referenced until the next association)."""
    keep, p, n, stride, mem = _points_arg(xyz)
    if not hasattr(self, "_edge_slot_keep"):
        self._edge_slot_keep = {}
    self._edge_slot_keep[slot] = keep
    self._chk(self._lib.glio_window_set_edge_scan(self._h, C.c_int(slot), p, C.c_int64(n), C.c_int(stride), C.c_int(mem)))


def _window_associate_edges(self, poses_body, options=None, **kw):
    """Edge association of slots 0..W-1 against the corner map; returns the edge count per slot."""
    pb = np.ascontiguousarray(poses_body, np.float64).reshape(-1, 7)
    W = len(pb)
    opt = options if options is not None else edge_default_options(**kw)
    ne = np.zeros(W, np.int64)
    self._chk(self._lib.glio_window_associate_edges(self._h, C.c_int(W), _ptr(pb), C.byref(opt), _ptr(ne)))
    return ne


def _get_edges(self, slot):
    """A slot's edge list: cp, pa, pb (n, 3) float32, s (n,) float64, src (n,) int32 (-1 for uploaded edges), n."""
    n = C.c_int64(0)
    self._chk(self._lib.glio_get_edges(self._h, C.c_int(slot), C.c_int64(0), None, None, None, None, None, C.byref(n)))
    m = int(n.value)
    out = dict(cp=np.empty((m, 3), np.float32), pa=np.empty((m, 3), np.float32), pb=np.empty((m, 3), np.float32), s=np.empty(m),
               src=np.empty(m, np.int32))
    self._chk(self._lib.glio_get_edges(self._h, C.c_int(slot), C.c_int64(m), _ptr(out["cp"]), _ptr(out["pa"]), _ptr(out["pb"]),
                                       _ptr(out["s"]), _ptr(out["src"]), C.byref(n)))
    out["n"] = m
    return out


def _get_edge_debug(self, slot, Q):
    """Per-query view of the slot's last edge association (keep_debug): status, idx5, sqd5, pm, eig (ascending)."""
    out = dict(status=np.empty(Q, np.uint8), idx5=np.empty((Q, 5), np.int32), sqd5=np.empty((Q, 5), np.float32),
               pm=np.empty((Q, 3), np.float32), eig=np.empty((Q, 3), np.float64))
    self._chk(self._lib.glio_get_edge_debug(self._h, C.c_int(slot), C.c_int64(Q), _ptr(out["status"]), _ptr(out["idx5"]),
                                            _ptr(out["sqd5"]), _ptr(out["pm"]), _ptr(out["eig"])))
    return out


def _eval_edge_kind(self, poses_body, jac_kind=0, want_jac=True):
    """glio_eval_edge_kind: the edge blocks with tangent (0, = eval_edge) or ambient x,y,z quaternion columns (1, marginalisation)."""
    pb = np.ascontiguousarray(poses_body, np.float64).reshape(-1, 7); W = len(pb)
    H = np.zeros((W, 6, 6)) if want_jac else None; g = np.zeros((W, 6)) if want_jac else None; cost = np.zeros(W)
    self._chk(self._lib.glio_eval_edge_kind(self._h, C.c_int(W), _ptr(pb), C.c_int(jac_kind), _ptr(H), _ptr(g), _ptr(cost)))
    return dict(H=H, g=g, cost=cost)


def _window_use_edges(self, on):
    """glio_window_use_edges: window solves and marginalisations add the slots' edge blocks (default off)."""
    self._chk(self._lib.glio_window_use_edges(self._h, C.c_int(1 if on else 0)))


Context.eval_edge_kind = _eval_edge_kind
Context.window_use_edges = _window_use_edges
Context.set_edge_map = _set_edge_map
Context.edge_localmap_clear = _edge_localmap_clear
Context.edge_localmap_push = _edge_localmap_push
Context.edge_localmap_pop_front = _edge_localmap_pop_front
Context.edge_localmap_build = _edge_localmap_build
Context.window_set_edge_scan = _window_set_edge_scan
Context.window_associate_edges = _window_associate_edges
Context.get_edges = _get_edges
Context.get_edge_debug = _get_edge_debug

def _batch_set_pair_matches(self, cur, oth, cp, normal_cent, weight):
    """Upload the matches of pair (cur, oth) instead of associating them (score = batch_score * weight)."""
    cp = np.ascontiguousarray(cp, np.float32).reshape(-1, 3); nc = np.ascontiguousarray(normal_cent, np.float64).reshape(-1, 6)
    w = np.ascontiguousarray(weight, np.float32)
    self._chk(self._lib.glio_batch_set_pair_matches(self._h, C.c_int(cur), C.c_int(oth), _ptr(cp), _ptr(nc), _ptr(w), C.c_int64(len(w))))


Context.batch_set_pair_matches = _batch_set_pair_matches


# ---------------------------------------------------------------------------------------------------
# batch edges: scan-to-multiscan edge association (K1be) and binary point-to-edge factors (K2be)
# ---------------------------------------------------------------------------------------------------
def _batch_set_edge_frame(self, frame, xyz):
    """glio_batch_set_edge_frame: the corner scan (body frame, 0 points allowed) of a frame set with batch_set_frame."""
    if isinstance(xyz, np.ndarray) and xyz.size == 0:
        stride = xyz.shape[1] if xyz.ndim == 2 else 3
        keep, p, n, mem = None, None, 0, HOST
    else:
        keep, p, n, stride, mem = _points_arg(xyz)
    if not hasattr(self, "_edge_frame_keep"):
        self._edge_frame_keep = {}
    self._edge_frame_keep[frame] = keep
    self._chk(self._lib.glio_batch_set_edge_frame(self._h, C.c_int(frame), p, C.c_int64(n), C.c_int(stride), C.c_int(mem)))


def _batch_associate_edges_pairs(self, cur, oth, options=None, **kw):
    """K1be over pairs (cur[i], oth[i]); returns the edge count per pair."""
    cur = np.ascontiguousarray(cur, np.int32); oth = np.ascontiguousarray(oth, np.int32)
    if len(cur) != len(oth):
        raise ValueError("cur and oth must have the same length")
    opt = options if options is not None else edge_default_options(**kw)
    ne = np.zeros(len(cur), np.int64)
    self._chk(self._lib.glio_batch_associate_edges_pairs(self._h, _ptr(cur), _ptr(oth), C.c_int64(len(cur)), C.byref(opt), _ptr(ne)))
    return ne


def _batch_get_edges(self, cur, oth):
    """The edge list of pair (cur, oth): cp (cur's frame), pa, pb (oth's frame) (n, 3) float32, s (n,), src (n,) int32, n."""
    n = C.c_int64(0)
    self._chk(self._lib.glio_batch_get_edges(self._h, C.c_int(cur), C.c_int(oth), C.c_int64(0), None, None, None, None, None, C.byref(n)))
    m = int(n.value)
    out = dict(cp=np.empty((m, 3), np.float32), pa=np.empty((m, 3), np.float32), pb=np.empty((m, 3), np.float32), s=np.empty(m),
               src=np.empty(m, np.int32))
    self._chk(self._lib.glio_batch_get_edges(self._h, C.c_int(cur), C.c_int(oth), C.c_int64(m), _ptr(out["cp"]), _ptr(out["pa"]),
                                             _ptr(out["pb"]), _ptr(out["s"]), _ptr(out["src"]), C.byref(n)))
    out["n"] = m
    return out


def _batch_set_pair_edges(self, cur, oth, cp, pa, pb, s):
    """Upload the edge list of pair (cur, oth) instead of associating it (src reads back as -1)."""
    cp = np.ascontiguousarray(cp, np.float32).reshape(-1, 3); pa = np.ascontiguousarray(pa, np.float32).reshape(-1, 3)
    pb = np.ascontiguousarray(pb, np.float32).reshape(-1, 3); s = np.ascontiguousarray(s, np.float64)
    self._chk(self._lib.glio_batch_set_pair_edges(self._h, C.c_int(cur), C.c_int(oth), _ptr(cp), _ptr(pa), _ptr(pb), _ptr(s),
                                                  C.c_int64(len(s))))


def _eval_binary_edge(self, poses, want_jac=True):
    """glio_eval_binary_edge: the binary edge blocks alone, in eval_binary's layout and pair order."""
    return _eval_blocks(self, self._lib.glio_eval_binary_edge, self._lib.glio_batch_pair_list, poses, want_jac)


def _batch_use_edges(self, on):
    """glio_batch_use_edges: batch solves add the pairs' edge blocks (default off)."""
    self._chk(self._lib.glio_batch_use_edges(self._h, C.c_int(1 if on else 0)))


Context.batch_set_edge_frame = _batch_set_edge_frame
Context.batch_associate_edges_pairs = _batch_associate_edges_pairs
Context.batch_get_edges = _batch_get_edges
Context.batch_set_pair_edges = _batch_set_pair_edges
Context.eval_binary_edge = _eval_binary_edge
Context.batch_use_edges = _batch_use_edges


# ---------------------------------------------------------------------------------------------------
# the batch refinement's pose factors (K2p): LidarPoseFactorBatchRelativeAutoDiff and delta_q_factor_auto
# ---------------------------------------------------------------------------------------------------
POSE_RELATIVE, POSE_DELTA_Q = 0, 1
POSE_MAX_KF = 1 << 22                     # keyframe indices of a pose factor are below this (GLIO_POSE_MAX_KF)
# glio_pose_factor: i, j, kind, active (int32), dq (w, x, y, z), dp (float64)
POSE_FACTOR_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("kind", "<i4"), ("active", "<i4"), ("dq", "<f8", (4,)), ("dp", "<f8", (3,))])
assert POSE_FACTOR_DTYPE.itemsize == 72


def pose_factor_records(i, j, kind, dq, dp=None, active=None):
    """A glio_pose_factor array from per-factor columns (dp defaults to 0, active to 1)."""
    n = len(i)
    f = np.zeros(n, POSE_FACTOR_DTYPE)
    f["i"], f["j"], f["kind"] = i, j, kind
    f["dq"] = np.asarray(dq, np.float64).reshape(n, 4)
    if dp is not None:
        f["dp"] = np.asarray(dp, np.float64).reshape(n, 3)
    f["active"] = 1 if active is None else np.asarray(active, np.int32)
    return f


def _batch_set_pose_factors(self, factors):
    """glio_batch_set_pose_factors: replace the pose-factor list (a POSE_FACTOR_DTYPE array; empty empties it)."""
    f = np.ascontiguousarray(factors, POSE_FACTOR_DTYPE)
    self._chk(self._lib.glio_batch_set_pose_factors(self._h, _ptr(f) if len(f) else None, C.c_int64(len(f))))


def _batch_pose_pair_list(self):
    """The pose-pair table (a, b), a < b, in order of first appearance."""
    return _pair_table(self, self._lib.glio_batch_pose_pair_list)


def _eval_pose_factors(self, poses, want_jac=True):
    """glio_eval_pose_factors: the pose blocks alone; Hoff in pose-pair order (d2 cost / d x_a d x_b, rows for a)."""
    return _eval_blocks(self, self._lib.glio_eval_pose_factors, self._lib.glio_batch_pose_pair_list, poses, want_jac)


def _batch_use_pose_factors(self, on):
    """glio_batch_use_pose_factors: batch solves add the pose blocks (default off)."""
    self._chk(self._lib.glio_batch_use_pose_factors(self._h, C.c_int(1 if on else 0)))


Context.batch_set_pose_factors = _batch_set_pose_factors
Context.batch_pose_pair_list = _batch_pose_pair_list
Context.eval_pose_factors = _eval_pose_factors
Context.batch_use_pose_factors = _batch_use_pose_factors


# ---------------------------------------------------------------------------------------------------
# the batch refinement's double-differenced pseudorange factors (K2g): dd_psr_factor_20
# ---------------------------------------------------------------------------------------------------
DD_PSR_MAX_SAT = 20                       # GLIO_DD_PSR_MAX_SAT: the reference's 19-row buffer
DD_PSR_MAX_KF = 1 << 22                   # GLIO_DD_PSR_MAX_KF
# glio_dd_psr_factor: i, j, n_sat, master, active, reserved (int32), sat_offset, w_offset (int64; -1 = identity), ratio,
# threshold, station (float64)
DD_PSR_FACTOR_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("n_sat", "<i4"), ("master", "<i4"), ("active", "<i4"), ("reserved", "<i4"),
                                ("sat_offset", "<i8"), ("w_offset", "<i8"), ("ratio", "<f8"), ("threshold", "<f8"), ("station", "<f8", (3,))])
assert DD_PSR_FACTOR_DTYPE.itemsize == 80
# glio_dd_psr_sat: sat_user, sat_ref (ECEF, m), psr_user, psr_ref (m)
DD_PSR_SAT_DTYPE = np.dtype([("sat_user", "<f8", (3,)), ("sat_ref", "<f8", (3,)), ("psr_user", "<f8"), ("psr_ref", "<f8")])
assert DD_PSR_SAT_DTYPE.itemsize == 64


def dd_psr_factor_records(i, j, n_sat, master, ratio, threshold, station, sat_offset=None, w_offset=None, active=None):
    """A glio_dd_psr_factor array from per-factor columns.  sat_offset defaults to the running sum of n_sat (each factor's
    satellites follow the previous factor's), w_offset to -1 (identity), active to 1; threshold and station may be scalars /
    one 3-vector for all factors."""
    n = len(i)
    f = np.zeros(n, DD_PSR_FACTOR_DTYPE)
    f["i"], f["j"], f["n_sat"], f["master"] = i, j, n_sat, master
    f["ratio"], f["threshold"] = ratio, threshold
    f["station"] = np.broadcast_to(np.asarray(station, np.float64), (n, 3))
    if sat_offset is None:
        sat_offset = np.cumsum(f["n_sat"].astype(np.int64)) - f["n_sat"]
    f["sat_offset"] = sat_offset
    f["w_offset"] = -1 if w_offset is None else w_offset
    f["active"] = 1 if active is None else np.asarray(active, np.int32)
    return f


def dd_psr_sat_records(sat_user, sat_ref, psr_user, psr_ref):
    """A glio_dd_psr_sat array from columns (n, 3), (n, 3), (n,), (n,)."""
    s = np.zeros(len(psr_user), DD_PSR_SAT_DTYPE)
    s["sat_user"], s["sat_ref"], s["psr_user"], s["psr_ref"] = sat_user, sat_ref, psr_user, psr_ref
    return s


def _batch_set_dd_psr_factors(self, factors, sats, R_ecef_local, anchor_ecef, W=None):
    """glio_batch_set_dd_psr_factors: replace the DD-pseudorange list (an empty factor array empties it)."""
    f = np.ascontiguousarray(factors, DD_PSR_FACTOR_DTYPE)
    s = np.ascontiguousarray(sats, DD_PSR_SAT_DTYPE)
    w = np.zeros(0) if W is None else np.ascontiguousarray(W, np.float64).ravel()
    R = np.ascontiguousarray(R_ecef_local, np.float64).reshape(9)
    a = np.ascontiguousarray(anchor_ecef, np.float64).reshape(3)
    self._chk(self._lib.glio_batch_set_dd_psr_factors(self._h, _ptr(f) if len(f) else None, C.c_int64(len(f)), _ptr(s) if len(s) else None,
                                                      C.c_int64(len(s)), _ptr(w) if len(w) else None, C.c_int64(len(w)), _ptr(R), _ptr(a)))


def _batch_dd_psr_pair_list(self):
    """The DD pair table (a, b), a < b, in order of first appearance."""
    return _pair_table(self, self._lib.glio_batch_dd_psr_pair_list)


def _eval_dd_psr_factors(self, poses, want_jac=True):
    """glio_eval_dd_psr_factors: the DD blocks alone; Hoff in DD-pair order (d2 cost / d x_a d x_b, rows for a)."""
    return _eval_blocks(self, self._lib.glio_eval_dd_psr_factors, self._lib.glio_batch_dd_psr_pair_list, poses, want_jac)


def _batch_use_dd_psr_factors(self, on):
    """glio_batch_use_dd_psr_factors: batch solves add the DD blocks (default off)."""
    self._chk(self._lib.glio_batch_use_dd_psr_factors(self._h, C.c_int(1 if on else 0)))


Context.batch_set_dd_psr_factors = _batch_set_dd_psr_factors
Context.batch_dd_psr_pair_list = _batch_dd_psr_pair_list
Context.eval_dd_psr_factors = _eval_dd_psr_factors
Context.batch_use_dd_psr_factors = _batch_use_dd_psr_factors


# ---------------------------------------------------------------------------------------------------
# the batch refinement's IMU factors (K2i): ImuFactor from the caller's pre-integration
# ---------------------------------------------------------------------------------------------------
IMU_MAX_KF = 1 << 22                      # keyframe indices of an IMU factor are below this (GLIO_IMU_MAX_KF)
# glio_imu_factor: i, j, active, reserved (int32), then float64: sum_dt, g_vec, delta_p, delta_q (w, x, y, z), delta_v,
# linearized_ba, linearized_bg, the jacobian_ blocks dp_dba, dp_dbg, dq_dbg, dv_dba, dv_dbg (3 x 3) and sqrt_info (15 x 15), row-major
IMU_FACTOR_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("active", "<i4"), ("reserved", "<i4"), ("sum_dt", "<f8"), ("g_vec", "<f8", (3,)),
                             ("delta_p", "<f8", (3,)), ("delta_q", "<f8", (4,)), ("delta_v", "<f8", (3,)),
                             ("linearized_ba", "<f8", (3,)), ("linearized_bg", "<f8", (3,)),
                             ("dp_dba", "<f8", (3, 3)), ("dp_dbg", "<f8", (3, 3)), ("dq_dbg", "<f8", (3, 3)), ("dv_dba", "<f8", (3, 3)),
                             ("dv_dbg", "<f8", (3, 3)), ("sqrt_info", "<f8", (15, 15))])
assert IMU_FACTOR_DTYPE.itemsize == 2336


def imu_factor_records(i, j, sum_dt, g_vec, delta_p, delta_q, delta_v, linearized_ba, linearized_bg, dp_dba, dp_dbg, dq_dbg, dv_dba,
                       dv_dbg, sqrt_info, active=None):
    """A glio_imu_factor array from per-factor columns (g_vec may be one vector for all; active defaults to 1)."""
    n = len(i)
    f = np.zeros(n, IMU_FACTOR_DTYPE)
    f["i"], f["j"], f["sum_dt"] = i, j, sum_dt
    f["g_vec"] = np.broadcast_to(np.asarray(g_vec, np.float64), (n, 3))
    for name, val, shape in (("delta_p", delta_p, (3,)), ("delta_q", delta_q, (4,)), ("delta_v", delta_v, (3,)),
                             ("linearized_ba", linearized_ba, (3,)), ("linearized_bg", linearized_bg, (3,)), ("dp_dba", dp_dba, (3, 3)),
                             ("dp_dbg", dp_dbg, (3, 3)), ("dq_dbg", dq_dbg, (3, 3)), ("dv_dba", dv_dba, (3, 3)), ("dv_dbg", dv_dbg, (3, 3)),
                             ("sqrt_info", sqrt_info, (15, 15))):
        f[name] = np.asarray(val, np.float64).reshape((n,) + shape)
    f["active"] = 1 if active is None else np.asarray(active, np.int32)
    return f


def _batch_set_imu_factors(self, factors):
    """glio_batch_set_imu_factors: replace the IMU list (an IMU_FACTOR_DTYPE array; empty empties it)."""
    f = np.ascontiguousarray(factors, IMU_FACTOR_DTYPE)
    self._chk(self._lib.glio_batch_set_imu_factors(self._h, _ptr(f) if len(f) else None, C.c_int64(len(f))))


def _batch_imu_pair_list(self):
    """The IMU pair table (a, b), a < b, in order of first appearance."""
    return _pair_table(self, self._lib.glio_batch_imu_pair_list)


def _eval_imu_factors(self, poses, speed_bias, want_jac=True):
    """glio_eval_imu_factors: the IMU blocks alone at poses (K, 7) and speed_bias (K, 9): Hdiag (K,15,15), Hoff (P,15,15) in
    IMU-pair order (d2 cost / d x_a d x_b, rows for a) and g (K,15) (None without want_jac), and the cost."""
    pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); K = len(pb)
    sb = np.ascontiguousarray(speed_bias, np.float64).reshape(K, 9)
    P = len(_pair_table(self, self._lib.glio_batch_imu_pair_list)[0])
    Hd = np.zeros((K, 15, 15)) if want_jac else None; Ho = np.zeros((P, 15, 15)) if want_jac else None
    g = np.zeros((K, 15)) if want_jac else None; cost = np.zeros(1)
    self._chk(self._lib.glio_eval_imu_factors(self._h, C.c_int(K), _ptr(pb), _ptr(sb), _ptr(Hd), _ptr(Ho), _ptr(g), _ptr(cost)))
    return dict(Hdiag=Hd, Hoff=Ho, g=g, cost=float(cost[0]))


def _batch_use_imu_factors(self, on):
    """glio_batch_use_imu_factors: batch solves add the IMU blocks (default off; they need speed_bias)."""
    self._chk(self._lib.glio_batch_use_imu_factors(self._h, C.c_int(1 if on else 0)))


Context.batch_set_imu_factors = _batch_set_imu_factors
Context.batch_imu_pair_list = _batch_imu_pair_list
Context.eval_imu_factors = _eval_imu_factors
Context.batch_use_imu_factors = _batch_use_imu_factors


# the window's IMU chain (K2i in the sliding window): its own list of IMU_FACTOR_DTYPE records, i and j window slots
WINDOW_MAX_SLOTS = 4096                   # window slots of an IMU factor are below this


def _window_set_imu_factors(self, factors):
    """glio_window_set_imu_factors: replace the window IMU list (an IMU_FACTOR_DTYPE array; empty empties it).  The batch list
    is left alone."""
    f = np.ascontiguousarray(factors, IMU_FACTOR_DTYPE)
    self._chk(self._lib.glio_window_set_imu_factors(self._h, _ptr(f) if len(f) else None, C.c_int64(len(f))))


def _window_imu_pair_list(self):
    """The window IMU pair table (a, b), a < b, in order of first appearance."""
    return _pair_table(self, self._lib.glio_window_imu_pair_list)


def _eval_window_imu_factors(self, poses, speed_bias, jac_kind=0, want_jac=True):
    """glio_eval_window_imu_factors: the window IMU blocks alone at poses (W, 7) and speed_bias (W, 9), eval_imu_factors' layout.
    jac_kind 0: tangent quaternion columns; 1: the ambient x, y, z columns the marginalisation reads."""
    pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); W = len(pb)
    sb = np.ascontiguousarray(speed_bias, np.float64).reshape(W, 9)
    P = len(_pair_table(self, self._lib.glio_window_imu_pair_list)[0])
    Hd = np.zeros((W, 15, 15)) if want_jac else None; Ho = np.zeros((P, 15, 15)) if want_jac else None
    g = np.zeros((W, 15)) if want_jac else None; cost = np.zeros(1)
    self._chk(self._lib.glio_eval_window_imu_factors(self._h, C.c_int(W), _ptr(pb), _ptr(sb), C.c_int(jac_kind), _ptr(Hd), _ptr(Ho),
                                                     _ptr(g), _ptr(cost)))
    return dict(Hdiag=Hd, Hoff=Ho, g=g, cost=float(cost[0]))


def _window_use_imu_factors(self, on):
    """glio_window_use_imu_factors: window solves and marginalisations take the IMU chain from the device (default off; they
    need speed_bias)."""
    self._chk(self._lib.glio_window_use_imu_factors(self._h, C.c_int(1 if on else 0)))


Context.window_set_imu_factors = _window_set_imu_factors
Context.window_imu_pair_list = _window_imu_pair_list
Context.eval_window_imu_factors = _eval_window_imu_factors
Context.window_use_imu_factors = _window_use_imu_factors


# K4: the band Cholesky factor-and-solve on the device
BAND_MAX_HB = 160                         # GLIO_BAND_MAX_HB: the largest half bandwidth glio_band_solve takes


def _band_solve(self, band, b):
    """glio_band_solve: factor the symmetric band (n, hb+1) (lower band, glio_batch_solve's layout) and solve A x = b on the
    device.  Returns (L, x, ok): L the factored band in the same layout, x the solution, ok False when a pivot was not positive
    and finite or x is not finite (then L and x hold partial results)."""
    L = np.array(band, np.float64, order="C", copy=True)
    n, w = L.shape
    rhs = np.ascontiguousarray(b, np.float64).reshape(n)
    x = np.zeros(n); ok = C.c_int(0)
    self._chk(self._lib.glio_band_solve(self._h, C.c_int(n), C.c_int(w - 1), _ptr(L), _ptr(rhs), _ptr(x), C.byref(ok)))
    return L, x, bool(ok.value)


Context.band_solve = _band_solve


def _band_ops(self, H, s, v, x):
    """glio_band_ops: the device minimizer's scale, shift and product on the band H (n, hb+1) and the n-vectors s, v and x.
    Returns (Hs, hs_diag, A, y): Hs = S H S, hs_diag its diagonal, A = Hs + diag(v*v) and y = Hs x.  The slots of Hs and A with
    j < 0 are unspecified.  Takes hb up to BAND_BCR_MAX_HB, the widest band the device minimizer takes."""
    Hb = np.ascontiguousarray(H, np.float64)
    n, w = Hb.shape
    s, v, x = (np.ascontiguousarray(a, np.float64).reshape(n) for a in (s, v, x))
    Hs = np.zeros((n, w)); A = np.zeros((n, w)); hs_diag = np.zeros(n); y = np.zeros(n)
    self._chk(self._lib.glio_band_ops(self._h, C.c_int(n), C.c_int(w - 1), _ptr(Hb), _ptr(s), _ptr(v), _ptr(x), _ptr(Hs),
                                      _ptr(hs_diag), _ptr(A), _ptr(y)))
    return Hs, hs_diag, A, y


Context.band_ops = _band_ops


# the band solve by block cyclic reduction on the device
BAND_BCR_MAX_HB = 256                     # GLIO_BAND_BCR_MAX_HB: the largest half bandwidth glio_band_solve_bcr takes
FACTOR_SEQUENTIAL = 0                     # GLIO_FACTOR_SEQUENTIAL: the device minimizer factors with K4 (the default)
FACTOR_BCR = 1                            # GLIO_FACTOR_BCR: the device minimizer solves by block cyclic reduction


def _band_solve_bcr(self, band, b):
    """glio_band_solve_bcr: solve A x = b for the symmetric band (n, hb+1) (lower band, glio_batch_solve's layout) by block cyclic
    reduction on the device; the band is not changed.  Returns (x, ok): ok False when a block pivot was not positive and finite
    or x is not finite (then x is unspecified)."""
    A = np.ascontiguousarray(band, np.float64)
    n, w = A.shape
    rhs = np.ascontiguousarray(b, np.float64).reshape(n)
    x = np.zeros(n); ok = C.c_int(0)
    self._chk(self._lib.glio_band_solve_bcr(self._h, C.c_int(n), C.c_int(w - 1), _ptr(A), _ptr(rhs), _ptr(x), C.byref(ok)))
    return x, bool(ok.value)


def _batch_device_factorization(self, kind):
    """glio_batch_device_factorization: FACTOR_SEQUENTIAL (K4, the default) or FACTOR_BCR for the device minimizer's solves."""
    self._chk(self._lib.glio_batch_device_factorization(self._h, C.c_int(kind)))


Context.band_solve_bcr = _band_solve_bcr
Context.batch_device_factorization = _batch_device_factorization


def _batch_use_device_solver(self, on):
    """glio_batch_use_device_solver: batch solves run the minimizer's band algebra on the device (default off)."""
    self._chk(self._lib.glio_batch_use_device_solver(self._h, C.c_int(1 if on else 0)))


def _batch_normal_equations(self, poses, speed_bias=None, host_factors=None, on_device=False):
    """glio_batch_normal_equations: (band (n, hb+1), g (n), cost) at one state, by the host path or on the device (hb up to
    BAND_BCR_MAX_HB)."""
    pb = np.ascontiguousarray(poses, np.float64).reshape(-1, 7); K = len(pb)
    sb = None if speed_bias is None else np.ascontiguousarray(speed_bias, np.float64).reshape(K, 9)
    n = K * (15 if sb is not None else 6)
    cap = n * n if n < 4096 else n * 256
    H = np.zeros(cap); g = np.zeros(n); cost = np.zeros(1); hb = C.c_int(0)
    if host_factors is None:
        fn, user = C.cast(None, HOST_FACTORS_BAND_FN), None
    else:
        fn, user = C.cast(self._lib.glio_hf_evaluate_band, HOST_FACTORS_BAND_FN), host_factors._h
    self._chk(self._lib.glio_batch_normal_equations(self._h, C.c_int(K), _ptr(pb), _ptr(sb), fn, user, C.c_int(1 if on_device else 0),
                                                    C.c_int64(cap), _ptr(H), C.byref(hb), _ptr(g), _ptr(cost)))
    w = hb.value + 1
    return H[:n * w].reshape(n, w).copy(), g, float(cost[0])


Context.batch_use_device_solver = _batch_use_device_solver
Context.batch_normal_equations = _batch_normal_equations


# ---------------------------------------------------------------------------------------------------
# feature selection on the device (featureSelection / globalFeatureSelection[Add]_Batch, Estimator.cpp:3894-4116, seeded)
# ---------------------------------------------------------------------------------------------------
class SelectOptions(C.Structure):
    _fields_ = [("feature_res_num", C.c_int32), ("rand_set_num", C.c_int32), ("batch_feature_res_num", C.c_int32),
                ("batch_rand_set_num", C.c_int32), ("random_select", C.c_int32), ("reserved", C.c_int32), ("seed", C.c_uint64),
                ("nonce", C.c_uint64)]


def select_default_options(**kw):
    """glio_select_default_options (the shipped configuration: F 100, R 300, B 25, BR 400, random_select, seed 0, nonce 0)."""
    o = SelectOptions()
    lib().glio_select_default_options(C.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise AttributeError(k)
        setattr(o, k, int(v))
    return o


def _select_random(self, stream_ids, options=None, **kw):
    """glio_select_random for slots 0..len(stream_ids)-1 (stream id = the slot's keyframe index); returns the active counts."""
    ids = np.ascontiguousarray(stream_ids, np.int64)
    opt = options if options is not None else select_default_options(**kw)
    na = np.zeros(len(ids), np.int64)
    self._chk(self._lib.glio_select_random(self._h, C.c_int(len(ids)), _ptr(ids), C.byref(opt), _ptr(na)))
    return na


def _batch_select_random(self, cur, oth, mode, options=None, **kw):
    """glio_batch_select_random over pairs (cur[i], oth[i]) grouped by cur; mode 0 start/end, 1 incremental; returns the active counts."""
    cur = np.ascontiguousarray(cur, np.int32); oth = np.ascontiguousarray(oth, np.int32)
    if len(cur) != len(oth):
        raise ValueError("cur and oth must have the same length")
    opt = options if options is not None else select_default_options(**kw)
    na = np.zeros(len(cur), np.int64)
    self._chk(self._lib.glio_batch_select_random(self._h, _ptr(cur), _ptr(oth), C.c_int64(len(cur)), C.c_int(mode), C.byref(opt), _ptr(na)))
    return na


def _selection_out(call):
    n = C.c_int64(0)
    call(C.c_int64(0), None, C.byref(n))
    if n.value < 0:
        return None
    keep = np.empty(n.value, np.int32)
    call(C.c_int64(n.value), _ptr(keep), C.byref(n))
    return keep


def _get_selection(self, slot):
    """The active match indices of a slot (int32 array), or None when all its matches are active."""
    return _selection_out(lambda cap, p, n: self._chk(self._lib.glio_get_selection(self._h, C.c_int(slot), cap, p, n)))


def _batch_get_selection(self, cur, oth):
    """The active match indices of pair (cur, oth), or None when all its matches are active."""
    return _selection_out(lambda cap, p, n: self._chk(self._lib.glio_batch_get_selection(self._h, C.c_int(cur), C.c_int(oth), cap, p, n)))


def _select_random_edges(self, stream_ids, options=None, **kw):
    """glio_select_random_edges: featureSelection's rule and sampler on the edge lists of slots 0..len(stream_ids)-1 (domain 3);
    returns the active edge counts."""
    ids = np.ascontiguousarray(stream_ids, np.int64)
    opt = options if options is not None else select_default_options(**kw)
    na = np.zeros(len(ids), np.int64)
    self._chk(self._lib.glio_select_random_edges(self._h, C.c_int(len(ids)), _ptr(ids), C.byref(opt), _ptr(na)))
    return na


def _batch_select_random_edges(self, cur, oth, mode, options=None, **kw):
    """glio_batch_select_random_edges: the batch rules and sampler on the edge lists of pairs (cur[i], oth[i]) (domains 4 / 5);
    returns the active edge counts."""
    cur = np.ascontiguousarray(cur, np.int32); oth = np.ascontiguousarray(oth, np.int32)
    if len(cur) != len(oth):
        raise ValueError("cur and oth must have the same length")
    opt = options if options is not None else select_default_options(**kw)
    na = np.zeros(len(cur), np.int64)
    self._chk(self._lib.glio_batch_select_random_edges(self._h, _ptr(cur), _ptr(oth), C.c_int64(len(cur)), C.c_int(mode), C.byref(opt),
                                                       _ptr(na)))
    return na


def _get_edge_selection(self, slot):
    """The selected edge indices of a slot in draw order (int32 array), or None when all its edges are active."""
    return _selection_out(lambda cap, p, n: self._chk(self._lib.glio_get_edge_selection(self._h, C.c_int(slot), cap, p, n)))


def _batch_get_edge_selection(self, cur, oth):
    """The selected edge indices of pair (cur, oth) in draw order, or None when all its edges are active."""
    return _selection_out(lambda cap, p, n: self._chk(self._lib.glio_batch_get_edge_selection(self._h, C.c_int(cur), C.c_int(oth), cap, p, n)))


Context.select_random = _select_random
Context.batch_select_random = _batch_select_random
Context.get_selection = _get_selection
Context.batch_get_selection = _batch_get_selection
Context.select_random_edges = _select_random_edges
Context.batch_select_random_edges = _batch_select_random_edges
Context.get_edge_selection = _get_edge_selection
Context.batch_get_edge_selection = _batch_get_edge_selection
Context.batch_declare_pairs = _batch_declare_pairs
Context.batch_solve = _batch_solve
Context.set_allreduce = _set_allreduce
Context.batch_set_frame = _batch_set_frame
Context.batch_set_pose = _batch_set_pose
Context.batch_associate_pairs = _batch_associate_pairs
Context.batch_get_matches = _batch_get_matches
Context.batch_select = _batch_select
Context.batch_pair_list = _batch_pair_list
Context.batch_clear = _batch_clear
Context.eval_binary = _eval_binary


# ---------------------------------------------------------------------------------------------------
# front-end LiDAR odometry (LidarOdometry::run, GLIO/src/LidarOdometry.cpp:661-695)
# ---------------------------------------------------------------------------------------------------
class OdomOptions(C.Structure):
    _fields_ = [("max_num_iter", C.c_int32), ("scan_match_cnt", C.c_int32), ("deskew", C.c_int32), ("reserved", C.c_int32),
                ("max_solver_time_s", C.c_double)]


ODOM_MAX_ROUNDS = 8


class OdomReport(C.Structure):
    _fields_ = [("pose", C.c_double * 7), ("rel_pose", C.c_double * 7), ("initialised", C.c_int32), ("keyframe", C.c_int32),
                ("skipped", C.c_int32), ("n_rounds", C.c_int32), ("n_map", C.c_int64), ("n_scan", C.c_int64),
                ("round_n_match", C.c_int64 * ODOM_MAX_ROUNDS), ("round_iterations", C.c_int32 * ODOM_MAX_ROUNDS),
                ("round_successful", C.c_int32 * ODOM_MAX_ROUNDS), ("round_termination", C.c_int32 * ODOM_MAX_ROUNDS),
                ("reserved", C.c_int32), ("round_pose", (C.c_double * 7) * ODOM_MAX_ROUNDS), ("summary", SolverSummary)]


def default_odom_options(**kw):
    o = OdomOptions()
    lib().glio_odom_default_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _cloud4_arg(a):
    """(n, 4) float32 x,y,z,intensity: numpy array (host) or contiguous CUDA tensor (device)."""
    if a is None:
        return None, None, 0, HOST
    if isinstance(a, np.ndarray):
        h = np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 4)
        return h, _ptr(h), h.shape[0], HOST
    if hasattr(a, "data_ptr"):
        if not (a.is_cuda and a.is_contiguous() and a.dtype.itemsize == 4 and a.dim() == 2 and a.shape[1] == 4):
            raise ValueError("a device cloud must be a contiguous (n, 4) float32 CUDA tensor")
        return a, C.c_void_p(a.data_ptr()), a.shape[0], DEVICE
    raise TypeError("clouds must be numpy arrays or CUDA torch tensors")


class Odometry:
    """The front end's LidarOdometry node on the device: one step() per sweep with its surf features (extract_features'
    less_flat_ds) and optionally its full cloud (prepare_scan's output), both (n, 4) x,y,z,intensity, numpy or CUDA tensors.
    Runs on the context's GPU and stream; its state is its own (see glio_odom_step in include/glio_b200.h)."""

    def __init__(self, ctx, **options):
        self.ctx = ctx
        self._lib = ctx._lib
        self.options = default_odom_options(**options)
        self._h = C.c_void_p()
        ctx._chk(self._lib.glio_odom_create(ctx._h, C.byref(self.options), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self.ctx._h:      # a closed context has already freed its odometries
            self._lib.glio_odom_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self.ctx._chk(self._lib.glio_odom_reset(self._h))

    def step(self, surf, full=None, out="host"):
        """Returns dict(pose (7,) t,q; rel_pose (7,) t,q; initialised, keyframe, skipped: bool; n_map, n_scan; rounds: list of
        dict(n_match, iterations, successful, termination, pose); summary: the last round's SolverSummary; surf / full: the
        published clouds (None when this sweep publishes nothing or the input was not given)."""
        if out not in ("host", "device"):
            raise ValueError("out must be 'host' or 'device'")
        ks, ps, ns, ms = _cloud4_arg(surf)
        kf, pf, nf, mf = _cloud4_arg(full)
        if out == "device":
            import torch
            dev = torch.device("cuda", self.ctx.device)
            so = torch.empty((max(ns, 1), 4), dtype=torch.float32, device=dev)
            fo = torch.empty((max(nf, 1), 4), dtype=torch.float32, device=dev) if full is not None else None
            # torch's allocator hands the memory out on torch's stream, the library writes it on the context's: let torch finish first
            torch.cuda.current_stream(dev).synchronize()
            pso, pfo, om = C.c_void_p(so.data_ptr()), (C.c_void_p(fo.data_ptr()) if fo is not None else None), DEVICE
        else:
            so = np.empty((ns, 4), np.float32)
            fo = np.empty((nf, 4), np.float32) if full is not None else None
            pso, pfo, om = _ptr(so), _ptr(fo), HOST
        rep = OdomReport()
        self.ctx._chk(self._lib.glio_odom_step(self._h, ps, C.c_int64(ns), C.c_int(ms), pf, C.c_int64(nf), C.c_int(mf), pso, pfo,
                                               C.c_int(om), C.byref(rep)))
        published = bool(rep.initialised or rep.keyframe)
        rounds = [dict(n_match=int(rep.round_n_match[r]), iterations=int(rep.round_iterations[r]), successful=int(rep.round_successful[r]),
                       termination=int(rep.round_termination[r]), pose=np.array(rep.round_pose[r][:])) for r in range(rep.n_rounds)]
        return dict(pose=np.array(rep.pose[:]), rel_pose=np.array(rep.rel_pose[:]), initialised=bool(rep.initialised),
                    keyframe=bool(rep.keyframe), skipped=bool(rep.skipped), n_map=int(rep.n_map), n_scan=int(rep.n_scan), rounds=rounds,
                    summary=rep.summary, surf=so[:ns] if published else None,
                    full=(fo[:nf] if published and fo is not None else None))

    def clouds(self):
        """The last step's filtered map and filtered scan, (n, 3) float32 each (debug copy-out)."""
        nm = C.c_int64(0); nsc = C.c_int64(0)
        self.ctx._chk(self._lib.glio_odom_get_clouds(self._h, C.c_int64(0), None, C.byref(nm), C.c_int64(0), None, C.byref(nsc)))
        m = np.empty((nm.value, 3), np.float32); s = np.empty((nsc.value, 3), np.float32)
        self.ctx._chk(self._lib.glio_odom_get_clouds(self._h, C.c_int64(nm.value), _ptr(m), C.byref(nm), C.c_int64(nsc.value), _ptr(s),
                                                     C.byref(nsc)))
        return m, s


# ---------------------------------------------------------------------------------------------------------------------------
# loop-closure registration (detectLoopClosure / performLoopClosure, GLIO/src/Estimator.cpp:5101-5273, without the GTSAM half)
# ---------------------------------------------------------------------------------------------------------------------------
ICP_NOT_CONVERGED, ICP_ITERATIONS, ICP_TRANSFORM, ICP_ABS_MSE, ICP_REL_MSE, ICP_NO_CORRESPONDENCES = range(6)


class IcpOptions(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("reserved", C.c_int32), ("max_correspondence_distance", C.c_double),
                ("transformation_epsilon", C.c_double), ("euclidean_fitness_epsilon", C.c_double)]


class IcpIteration(C.Structure):
    _fields_ = [("transformation", C.c_float * 16), ("n_corr", C.c_int64), ("mse", C.c_double)]


class IcpResult(C.Structure):
    _fields_ = [("converged", C.c_int32), ("state", C.c_int32), ("iterations", C.c_int32), ("host_syncs", C.c_int32),
                ("n_source", C.c_int64), ("n_target", C.c_int64), ("n_corr", C.c_int64), ("launches", C.c_int64),
                ("final_transformation", C.c_float * 16), ("fitness", C.c_double)]


class LoopOptions(C.Structure):
    _fields_ = [("lc_search_radius", C.c_double), ("lc_time_thres", C.c_double), ("lc_map_width", C.c_int32), ("lc_icp_thres", C.c_float),
                ("slide_window_width", C.c_int32), ("leaf", C.c_float), ("q_lb", C.c_double * 4), ("t_lb", C.c_double * 3),
                ("icp", IcpOptions)]


class LoopReport(C.Structure):
    _fields_ = [("detected", C.c_int32), ("closest_his_idx", C.c_int32), ("latest_frame_idx", C.c_int32), ("accepted", C.c_int32),
                ("n_latest", C.c_int64), ("n_latest_ds", C.c_int64), ("n_his", C.c_int64), ("n_his_ds", C.c_int64),
                ("n_candidates", C.c_int64), ("icp", IcpResult), ("pose_from", C.c_double * 7), ("pose_to", C.c_double * 7),
                ("noise_score", C.c_double), ("time_last_loop", C.c_double)]


_ICP_KEYS = ("max_iterations", "max_correspondence_distance", "transformation_epsilon", "euclidean_fitness_epsilon")


def default_icp_options(**kw):
    o = IcpOptions()
    lib().glio_icp_default_options(C.byref(o))
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def default_loop_options(**kw):
    """glio_loop_default_options (the shipped configuration); the ICP settings may be given by name as well."""
    o = LoopOptions()
    lib().glio_loop_default_options(C.byref(o))
    for k, v in kw.items():
        if k in ("q_lb", "t_lb"):
            arr = getattr(o, k)
            for i, x in enumerate(v):
                arr[i] = float(x)
        elif k in _ICP_KEYS:
            setattr(o.icp, k, v)
        else:
            setattr(o, k, v)
    return o


def _icp_dict(r):
    return dict(converged=bool(r.converged), state=int(r.state), iterations=int(r.iterations), host_syncs=int(r.host_syncs),
                n_source=int(r.n_source), n_target=int(r.n_target), n_corr=int(r.n_corr), launches=int(r.launches),
                final=np.array(r.final_transformation[:], np.float32).reshape(4, 4), fitness=float(r.fitness))


def _icp_align(self, src, tgt, iter_log=True, correspondences=False, aligned=True, **options):
    """pcl::IterativeClosestPoint::align (identity guess) + getFitnessScore on the device.  src / tgt: (n, stride) float32 numpy arrays or
    CUDA tensors with x, y, z in columns 0..2.  options: the glio_icp_options fields (default: the Estimator's settings).  Returns
    the result dict (converged, state, iterations, host_syncs, n_corr, launches, final (4x4), fitness) plus aligned (n, 3), log (list of
    (transformation, n_corr, mse)) and corr ((query, match, dist) of the last correspondence estimation) when asked for."""
    opt = default_icp_options(**options)
    ks, ps, ns, ss, ms = _points_arg(src) if _npts(src) else (None, None, 0, 3, HOST)
    kt, pt, nt, st, mt = _points_arg(tgt) if _npts(tgt) else (None, None, 0, 3, HOST)
    al = np.empty((ns, 3), np.float32) if aligned else None
    cap = opt.max_iterations if iter_log else 0
    log = (IcpIteration * max(cap, 1))()
    cq = cm = cd = None
    if correspondences:
        cq = np.empty(max(ns, 1), np.int32); cm = np.empty(max(ns, 1), np.int32); cd = np.empty(max(ns, 1), np.float32)
    res = IcpResult()
    self._chk(self._lib.glio_icp_align(self._h, ps, C.c_int64(ns), C.c_int(ss), C.c_int(ms), pt, C.c_int64(nt), C.c_int(st), C.c_int(mt),
                                       C.byref(opt), _ptr(al), C.byref(res), log if cap else None, C.c_int(cap), _ptr(cq), _ptr(cm), _ptr(cd),
                                       C.c_int64(ns if correspondences else 0)))
    out = _icp_dict(res)
    if aligned:
        out["aligned"] = al
    if iter_log:
        k = min(res.iterations, cap)
        out["log"] = [(np.array(log[i].transformation[:], np.float32).reshape(4, 4), int(log[i].n_corr), float(log[i].mse)) for i in range(k)]
    if correspondences:
        nc = int(res.n_corr)
        out["corr"] = (cq[:nc].copy(), cm[:nc].copy(), cd[:nc].copy())
    return out


def _npts(a):
    return a is not None and (a.shape[0] if hasattr(a, "shape") else len(a)) > 0


def _vs_output(ctx, n, out):
    """room for n packed x,y,z points: a numpy array, or a CUDA tensor on the context's GPU"""
    if out == "device":
        import torch
        dev = torch.device("cuda", ctx.device)
        buf = torch.empty((max(n, 1), 3), dtype=torch.float32, device=dev)
        # torch's allocator hands the memory out on torch's stream, the library writes it on the context's: let torch finish first
        torch.cuda.current_stream(dev).synchronize()
        return buf, C.c_void_p(buf.data_ptr()), DEVICE
    buf = np.empty((n, 3), np.float32)
    return buf, _ptr(buf), HOST


Context.icp_align = _icp_align


class LoopClosure:
    """The Estimator's loop-closure keyframe store and its detection + registration step on the device (see glio_loop_step in
    include/glio_b200.h).  Keyframe clouds stay resident on the context's GPU; the state is the object's own."""

    def __init__(self, ctx, **options):
        self.ctx = ctx
        self._lib = ctx._lib
        self.options = default_loop_options(**options)
        self._h = C.c_void_p()
        self._sizes = []                                   # keyframe cloud sizes: the global map's capacity
        ctx._chk(self._lib.glio_loop_create(ctx._h, C.byref(self.options), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self.ctx._h:      # a closed context has already freed its loop objects
            self._lib.glio_loop_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self.ctx._chk(self._lib.glio_loop_reset(self._h))
        self._sizes = []

    def __len__(self):
        n = C.c_int(0)
        self.ctx._chk(self._lib.glio_loop_size(self._h, C.byref(n)))
        return int(n.value)

    def add_keyframe(self, cloud, pose, time):
        """cloud: (n, stride) float32 numpy array or CUDA tensor, lidar frame (surf_last_ds); pose: body pose t, q; returns its index."""
        if _npts(cloud):
            keep, p, n, stride, mem = _points_arg(cloud)
        else:
            p, n, stride, mem = None, 0, 3, HOST
        ps = np.ascontiguousarray(pose, np.float64)
        idx = C.c_int32(0)
        self.ctx._chk(self._lib.glio_loop_add_keyframe(self._h, p, C.c_int64(n), C.c_int(stride), C.c_int(mem), _ptr(ps), C.c_double(time),
                                                       C.byref(idx)))
        self._sizes.append(int(n))
        return int(idx.value)

    def global_map(self, interval=3, leaf=0.2, out="host"):
        """save_pcd's global map (glio_loop_global_map, Estimator.cpp:5324-5349): keyframes 0, interval, ... moved by Tbl then by their
        current pose, concatenated, VoxelGrid(leaf).  Returns (points (m, 3) float32, filtered, n_raw): filtered is False when PCL's
        leaf-size check passed the concatenation (n_raw points) through.  out="device" returns a CUDA tensor."""
        if out not in ("host", "device"):
            raise ValueError("out must be 'host' or 'device'")
        cap = sum(self._sizes[::interval]) if interval >= 1 else 0
        buf, optr, omem = _vs_output(self.ctx, cap, out)
        m = C.c_int64(0); raw = C.c_int64(0); f = C.c_int32(0)
        self.ctx._chk(self._lib.glio_loop_global_map(self._h, C.c_int(interval), C.c_float(leaf), C.c_int64(cap), optr, C.c_int(omem), C.byref(m),
                                                     C.byref(raw), C.byref(f)))
        return buf[:m.value], bool(f.value), int(raw.value)

    def set_poses(self, first, poses):
        ps = np.ascontiguousarray(poses, np.float64).reshape(-1, 7)
        self.ctx._chk(self._lib.glio_loop_set_poses(self._h, C.c_int(first), C.c_int(len(ps)), _ptr(ps)))

    def step(self, select_xyz, time_new_odom):
        """Returns dict(detected, closest_his_idx, latest_frame_idx, accepted, n_latest, n_latest_ds, n_his, n_his_ds, n_candidates,
        icp (result dict, None when nothing ran), pose_from / pose_to (t, q; None unless accepted), noise_score, time_last_loop)."""
        s = np.ascontiguousarray(select_xyz, np.float32)
        rep = LoopReport()
        self.ctx._chk(self._lib.glio_loop_step(self._h, _ptr(s), C.c_double(time_new_odom), C.byref(rep)))
        acc = bool(rep.accepted)
        return dict(detected=bool(rep.detected), closest_his_idx=int(rep.closest_his_idx), latest_frame_idx=int(rep.latest_frame_idx),
                    accepted=acc, n_latest=int(rep.n_latest), n_latest_ds=int(rep.n_latest_ds), n_his=int(rep.n_his), n_his_ds=int(rep.n_his_ds),
                    n_candidates=int(rep.n_candidates), icp=_icp_dict(rep.icp) if rep.detected else None,
                    pose_from=np.array(rep.pose_from[:]) if acc else None, pose_to=np.array(rep.pose_to[:]) if acc else None,
                    noise_score=float(rep.noise_score) if acc else None, time_last_loop=float(rep.time_last_loop))

    def clouds(self):
        """The last registration's filtered latest and history clouds, (n, 3) float32 each (debug copy-out)."""
        nl = C.c_int64(0); nh = C.c_int64(0)
        self.ctx._chk(self._lib.glio_loop_get_clouds(self._h, C.c_int64(0), None, C.byref(nl), C.c_int64(0), None, C.byref(nh)))
        a = np.empty((nl.value, 3), np.float32); b = np.empty((nh.value, 3), np.float32)
        self.ctx._chk(self._lib.glio_loop_get_clouds(self._h, C.c_int64(nl.value), _ptr(a), C.byref(nl), C.c_int64(nh.value), _ptr(b), C.byref(nh)))
        return a, b
