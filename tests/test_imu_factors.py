"""K2i on the CPU: the longdouble restatement of ImuFactor::Evaluate (tests/imu_factor_reference.py) against 50-digit mpmath for
the residual and for central differences of the columns where the analytic Jacobian is the exact derivative (t, v, ba: r is linear
in them), every Jacobian block against a separate block-wise float64 transliteration of ImuFactor.h, the generator's covariance
and sqrt_info, and the glio_imu_factor record layout."""
import ctypes as C

import mpmath as mp
import numpy as np
import pytest

from glio_b200 import api, synth
from tests import eval_reference as er
from tests import imu_factor_reference as ir

mp.mp.dps = 50


def _case(kind, K=8, seed=3):
    """poses, speed-bias states and an IMU list over K keyframes; kind picks the quirks"""
    P = synth.imu_problem(K=K, seed=seed)
    poses = P["poses_init"].copy(); sb = P["sb_init"].copy()
    cols = dict(P["imu"])
    rng = np.random.default_rng(seed)
    if kind == "quirks":
        poses[:, 3:] *= rng.uniform(0.7, 1.4, (K, 1))                         # non-unit quaternions
        poses[1::2, 3:] *= -1.0                                                # w < 0
        poses[:, :3] += np.array([20_000.0, -15_000.0, 300.0])                 # 20 km offsets
        sb[:, 6:] += rng.normal(0.0, 0.01, (K, 3))                             # Bg_i far from linearized_bg
        cols["i"], cols["j"] = cols["j"].copy(), cols["i"].copy()              # i > j
    return poses, sb, api.imu_factor_records(**cols)


# ---------------------------------------------------------------------------------------------------------------------------
# 50-digit restatement of the residual
# ---------------------------------------------------------------------------------------------------------------------------
def _mq(a, b):
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]]


def _minv(q):
    n2 = sum(x * x for x in q)
    return [q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2]


def _mnorm(q):
    n = mp.sqrt(sum(x * x for x in q))
    return [x / n for x in q]


def _mrot(q, v):
    return _mq(_mq(q, [mp.mpf(0)] + list(v)), _minv(q))[1:]       # exact rotation by q, |q| = 1 in exact arithmetic


def _ld(x):
    """a longdouble as an exact mpf"""
    return mp.mpf(np.format_float_scientific(x, unique=True))


def _mp_residual(pi, si, pj, sj, F):
    m = lambda x: [mp.mpf(float(y)) for y in np.ravel(x)]
    return _mp_residual_states(m(pi), m(si), m(pj), m(sj), F)


@pytest.mark.parametrize("kind", ["plain", "quirks"])
def test_residual_matches_50_digits(kind):
    poses, sb, f = _case(kind)
    ref = ir.factor_residuals(poses, sb, f)
    for n in range(len(f)):
        F = f[n]
        r = _mp_residual(poses[F["i"]], sb[F["i"]], poses[F["j"]], sb[F["j"]], F)
        err = np.array([abs(float(r[a] - _ld(ref["r"][n, a]))) for a in range(15)])
        assert np.all(err <= er.U * np.asarray(ref["Mr"][n], np.float64)), (n, err)


# ---------------------------------------------------------------------------------------------------------------------------
# central differences where the analytic Jacobian is exact: r is linear in t_i, t_j, v_i, v_j, ba_i, ba_j
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["plain", "quirks"])
def test_exact_columns_match_central_differences(kind):
    poses, sb, f = _case(kind, K=5)
    ref = ir.factor_residuals(poses, sb, f)
    h = mp.mpf("1e-20")
    for n in range(len(f)):
        F = f[n]
        a = min(int(F["i"]), int(F["j"]))
        for col in list(range(0, 3)) + list(range(6, 12)) + list(range(15, 18)) + list(range(21, 27)):
            k = a if col < 15 else max(int(F["i"]), int(F["j"]))
            c = col % 15
            outs = []
            for s in (1, -1):
                P_ = [[mp.mpf(float(x)) for x in poses[q]] for q in range(len(poses))]
                S_ = [[mp.mpf(float(x)) for x in sb[q]] for q in range(len(sb))]
                if c < 3:
                    P_[k][c] += s * h
                else:
                    S_[k][c - 6] += s * h
                outs.append(_mp_residual_states(P_[F["i"]], S_[F["i"]], P_[F["j"]], S_[F["j"]], F))
            d = [(outs[0][r] - outs[1][r]) / (2 * h) for r in range(15)]
            err = np.array([abs(float(d[r] - _ld(ref["J"][n, r, col]))) for r in range(15)])
            assert np.all(err <= er.U * np.asarray(ref["MJ"][n, :, col], np.float64) + 1e-25), (n, col, err)


def _mp_residual_states(pi, si, pj, sj, F):
    """ImuFactor's residual at 50 digits from mpf states (t, q) and (V, Ba, Bg)"""
    m = lambda x: [mp.mpf(float(y)) for y in np.ravel(x)]
    Pi, Qi, Pj, Qj = list(pi[:3]), _mnorm(list(pi[3:])), list(pj[:3]), _mnorm(list(pj[3:]))
    Vi, Bai, Bgi, Vj, Baj, Bgj = list(si[:3]), list(si[3:6]), list(si[6:]), list(sj[:3]), list(sj[3:6]), list(sj[6:])
    M = lambda A, v: [sum(mp.mpf(float(A[r, k])) * v[k] for k in range(3)) for r in range(3)]
    T, g = mp.mpf(float(F["sum_dt"])), m(F["g_vec"])
    dba = [Bai[k] - mp.mpf(float(F["linearized_ba"][k])) for k in range(3)]
    dbg = [Bgi[k] - mp.mpf(float(F["linearized_bg"][k])) for k in range(3)]
    th = M(F["dq_dbg"], dbg)
    cdq = _mq(m(F["delta_q"]), [mp.mpf(1)] + [x / 2 for x in th])
    cdp = [mp.mpf(float(F["delta_p"][k])) + M(F["dp_dba"], dba)[k] + M(F["dp_dbg"], dbg)[k] for k in range(3)]
    cdv = [mp.mpf(float(F["delta_v"][k])) + M(F["dv_dba"], dba)[k] + M(F["dv_dbg"], dbg)[k] for k in range(3)]
    Qii = _minv(Qi)
    rp = _mrot(Qii, [-g[k] * T * T / 2 + Pj[k] - Pi[k] - Vi[k] * T for k in range(3)])
    rv = _mrot(Qii, [-g[k] * T + Vj[k] - Vi[k] for k in range(3)])
    E = _mnorm(_mq(_minv(cdq), _mq(Qii, Qj)))
    raw = [rp[k] - cdp[k] for k in range(3)] + [2 * E[1 + k] for k in range(3)] + [rv[k] - cdv[k] for k in range(3)] \
        + [Baj[k] - Bai[k] for k in range(3)] + [Bgj[k] - Bgi[k] for k in range(3)]
    S = F["sqrt_info"]
    return [sum(mp.mpf(float(S[a, b])) * raw[b] for b in range(15)) for a in range(15)]


# ---------------------------------------------------------------------------------------------------------------------------
# an independent block-wise transliteration of ImuFactor::Evaluate's Jacobians (float64, Eigen's matrix forms)
# ---------------------------------------------------------------------------------------------------------------------------
def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _Qleft(q):
    m = np.zeros((4, 4)); m[0, 0] = q[0]; m[0, 1:] = -q[1:]; m[1:, 0] = q[1:]; m[1:, 1:] = q[0] * np.eye(3) + _skew(q[1:])
    return m


def _Qright(p):
    m = np.zeros((4, 4)); m[0, 0] = p[0]; m[0, 1:] = -p[1:]; m[1:, 0] = p[1:]; m[1:, 1:] = p[0] * np.eye(3) - _skew(p[1:])
    return m


def _qm(a, b):
    return _Qleft(a) @ b


def _qi(q):
    return np.array([q[0], -q[1], -q[2], -q[3]]) / np.dot(q, q)


def _R(q):
    w, x, y, z = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    return np.array([[1 - (ty * y + tz * z), ty * x - tz * w, tz * x + ty * w], [ty * x + tz * w, 1 - (tx * x + tz * z), tz * y - tx * w],
                     [tz * x - ty * w, tz * y + tx * w, 1 - (tx * x + ty * y)]])


def _plus_jac(q):
    w, x, y, z = q
    return np.array([[-x, -y, -z], [w, z, -y], [-z, w, x], [y, -x, w]])


def _blockwise_jacobians(pi, si, pj, sj, F):
    """the six blocks of ImuFactor::Evaluate, as written, then the local Jacobian and sqrt_info: (15, 30) over (x_i, x_j)"""
    Qi = pi[3:] / np.linalg.norm(pi[3:]); Qj = pj[3:] / np.linalg.norm(pj[3:])
    T, g = F["sum_dt"], F["g_vec"]
    dq_dbg = F["dq_dbg"]
    cdq = _qm(F["delta_q"], np.concatenate([[1.0], dq_dbg @ (si[6:] - F["linearized_bg"]) / 2.0]))
    RiT = _R(_qi(Qi))
    tmp = -0.5 * g * T * T + pj[:3] - pi[:3] - si[:3] * T
    tmp1 = -g * T + sj[:3] - si[:3]

    def qrows(t):
        b = np.zeros((3, 4))
        b[:, 0] = 2 * (Qi[0] * t + _skew(Qi[1:]) @ t)
        b[:, 1:] = 2 * (np.dot(Qi[1:], t) * np.eye(3) + np.outer(Qi[1:], t) - np.outer(t, Qi[1:]) - Qi[0] * _skew(t))
        return b
    J0 = np.zeros((15, 3)); J0[0:3] = -RiT
    J1 = np.zeros((15, 4)); J1[0:3] = qrows(tmp); J1[3:6] = -2 * (_Qleft(_qi(Qj)) @ _Qright(cdq))[1:, :]; J1[6:9] = qrows(tmp1)
    J2 = np.zeros((15, 9))
    J2[0:3, 0:3] = -RiT * T; J2[0:3, 3:6] = -F["dp_dba"]; J2[0:3, 6:9] = -F["dp_dbg"]
    J2[3:6, 6:9] = -(_Qleft(_qm(_qm(_qi(Qj), Qi), cdq))[1:, 1:]) @ dq_dbg     # LeftQuatMatrix(q).topLeft = w I + [v]x = Qleft's lower block
    J2[6:9, 0:3] = -RiT; J2[6:9, 3:6] = -F["dv_dba"]; J2[6:9, 6:9] = -F["dv_dbg"]
    J2[9:12, 3:6] = -np.eye(3); J2[12:15, 6:9] = -np.eye(3)
    J3 = np.zeros((15, 3)); J3[0:3] = RiT
    J4 = np.zeros((15, 4)); J4[3:6] = 2 * _Qleft(_qm(_qi(cdq), _qi(Qi)))[1:, :]
    J5 = np.zeros((15, 9)); J5[6:9, 0:3] = RiT; J5[9:12, 3:6] = np.eye(3); J5[12:15, 6:9] = np.eye(3)
    S = F["sqrt_info"]
    return S @ np.concatenate([J0, J1 @ _plus_jac(pi[3:]), J2, J3, J4 @ _plus_jac(pj[3:]), J5], axis=1)


@pytest.mark.parametrize("kind", ["plain", "quirks"])
def test_jacobian_blocks_match_a_blockwise_transliteration(kind):
    poses, sb, f = _case(kind, K=12)
    ref = ir.factor_residuals(poses, sb, f)
    for n in range(len(f)):
        F = f[n]
        i, j = int(F["i"]), int(F["j"])
        J = _blockwise_jacobians(poses[i], sb[i], poses[j], sb[j], F)
        if i > j:
            J = np.concatenate([J[:, 15:], J[:, :15]], axis=1)
        er.assert_within(J, ref["J"][n], ref["MJ"][n], f"factor {n}")


# ---------------------------------------------------------------------------------------------------------------------------
# the generator and the record
# ---------------------------------------------------------------------------------------------------------------------------
def test_generator_sqrt_info_and_shape():
    P = synth.imu_problem(K=30)
    imu = P["imu"]
    assert list(imu["i"]) == list(range(29)) and list(imu["j"]) == list(range(1, 30))
    dt = np.diff(P["kf_times"])
    assert np.all((dt >= 0.25) & (dt <= 0.45)) and np.array_equal(imu["sum_dt"], dt)
    for S, cov in zip(imu["sqrt_info"], P["cov"]):
        assert np.all(np.tril(S, -1) == 0.0) and np.all(np.diag(S) > 0)
        assert np.all(np.linalg.eigvalsh(cov) > 0)
        # |S^T S cov - I| is bounded by a few n u cond(cov) (the inverse and the Cholesky factor are backward stable)
        bound = 64 * 15 * er.U * np.linalg.cond(cov)
        assert np.max(np.abs(S.T @ S @ cov - np.eye(15))) <= bound
    # the deltas were generated from the truth: the raw residual there is the injected noise, a few sigma at most
    f = api.imu_factor_records(**imu)
    R = ir.factor_residuals(P["poses_true"], P["sb_true"], f)
    assert np.max(np.abs(np.asarray(R["r"], np.float64))) < 6.0
    assert np.any(P["sb_init"] != P["sb_true"]) and np.any(imu["linearized_bg"] != P["sb_true"][:-1, 6:])


class _GlioImuFactor(C.Structure):
    """glio_imu_factor as include/glio_b200.h declares it"""
    _fields_ = [("i", C.c_int32), ("j", C.c_int32), ("active", C.c_int32), ("reserved", C.c_int32), ("sum_dt", C.c_double),
                ("g_vec", C.c_double * 3), ("delta_p", C.c_double * 3), ("delta_q", C.c_double * 4), ("delta_v", C.c_double * 3),
                ("linearized_ba", C.c_double * 3), ("linearized_bg", C.c_double * 3), ("dp_dba", C.c_double * 9),
                ("dp_dbg", C.c_double * 9), ("dq_dbg", C.c_double * 9), ("dv_dba", C.c_double * 9), ("dv_dbg", C.c_double * 9),
                ("sqrt_info", C.c_double * 225)]


def test_record_layout():
    assert C.sizeof(_GlioImuFactor) == api.IMU_FACTOR_DTYPE.itemsize == 2336
    for name, _ in _GlioImuFactor._fields_:
        assert getattr(_GlioImuFactor, name).offset == api.IMU_FACTOR_DTYPE.fields[name][1], name
