"""ctypes binding of the sweep-preparation oracle (oracle/scanprep/libgo_scanprep.so).

TEST INFRASTRUCTURE ONLY — imported by tests/ and scripts/bench_frontend.py.  Nothing under glio_b200/ may import this module.
PARITY UNPINNED: see the header of oracle/scanprep/go_scanprep.cpp.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scanprep")
_SO = os.path.join(_DIR, "libgo_scanprep.so")
_LIB = None


class ImuState(C.Structure):
    """idx_imu, current_time_imu, gyr_0 and first_imu of Preprocessing (GLIO/src/Preprocessing.cpp:33-39); zero = no sample yet."""
    _fields_ = [("idx_imu", C.c_int64), ("current_time_imu", C.c_double), ("gyr_0", C.c_double * 3), ("first_imu", C.c_int32),
                ("reserved", C.c_int32)]


def build(force=False):
    src = os.path.join(_DIR, "go_scanprep.cpp")
    if force or not os.path.exists(_SO) or os.path.getmtime(src) > os.path.getmtime(_SO):
        subprocess.check_call(["make", "-C", _DIR, "-s"], stdout=subprocess.DEVNULL)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        L.go_cr_atan2f.restype = C.c_float
        L.go_cr_atan2f.argtypes = [C.c_float, C.c_float]
        L.go_cr_atanf.restype = C.c_float
        L.go_cr_atanf.argtypes = [C.c_float]
        L.go_cr_guard_hits.restype = C.c_longlong
        L.go_prepare_scan.restype = C.c_int
        _LIB = L
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def cr_atan2f(y, x):
    """Correctly rounded float atan2 of float arrays (double libm, long double inside the guard band)."""
    y = np.ascontiguousarray(y, np.float32).ravel(); x = np.ascontiguousarray(x, np.float32).ravel()
    out = np.empty_like(y)
    lib().go_cr_atan2f_n(_p(y), _p(x), C.c_int64(len(y)), _p(out))
    return out


def cr_atanf(a):
    a = np.ascontiguousarray(a, np.float32).ravel()
    out = np.empty_like(a)
    lib().go_cr_atanf_n(_p(a), C.c_int64(len(a)), _p(out))
    return out


def libm_atan2f(y, x):
    y = np.ascontiguousarray(y, np.float32).ravel(); x = np.ascontiguousarray(x, np.float32).ravel()
    out = np.empty_like(y)
    lib().go_libm_atan2f_n(_p(y), _p(x), C.c_int64(len(y)), _p(out))
    return out


def libm_atanf(a):
    a = np.ascontiguousarray(a, np.float32).ravel()
    out = np.empty_like(a)
    lib().go_libm_atanf_n(_p(a), C.c_int64(len(a)), _p(out))
    return out


def guard_hits(reset=False):
    return int(lib().go_cr_guard_hits(C.c_int(1 if reset else 0)))


def prepare_scan(raw, n_scans, q_imu=None, q_lb=None):
    """Preprocessing::cloudHandler, :387-526.  raw: (n, stride) float32 with x, y, z in columns 0..2.
    Returns dict(cloud (m, 4) float32, scan_start, scan_end int32, half_index) or raises ValueError where the device call fails."""
    r = np.ascontiguousarray(raw, np.float32)
    n, stride = r.shape
    out = np.empty((n, 4), np.float32)
    ss = np.empty(n_scans, np.int32); se = np.empty(n_scans, np.int32)
    m = C.c_int64(0); h = C.c_int64(0)
    qi = None if q_imu is None else np.ascontiguousarray(q_imu, np.float64)
    ql = None if q_lb is None else np.ascontiguousarray(q_lb, np.float64)
    rc = lib().go_prepare_scan(_p(r), C.c_int64(n), C.c_int(stride), C.c_int(n_scans), _p(qi), _p(ql), _p(out), C.byref(m),
                               _p(ss), _p(se), C.byref(h))
    if rc != 0:
        raise ValueError(f"go_prepare_scan: {rc}")
    return dict(cloud=out[:m.value].copy(), scan_start=ss, scan_end=se, half_index=int(h.value))


def imu_sweep_rotation(state, stamps, gyro, t_scan_next):
    """processIMU (:222-259) for one sweep; `state` (ImuState) is updated in place.  Returns q (w, x, y, z)."""
    st = np.ascontiguousarray(stamps, np.float64); g = np.ascontiguousarray(gyro, np.float64).reshape(-1, 3)
    q = np.zeros(4)
    lib().go_imu_sweep_rotation(C.byref(state), _p(st), _p(g), C.c_int64(len(st)), C.c_double(t_scan_next), _p(q))
    return q
