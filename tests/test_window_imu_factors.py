"""CPU checks of the window IMU chain's references and data: the ambient-column ImuFactor Jacobian of tests/window_imu_reference.py
against a separate block-wise float64 transliteration of ImuFactor::Evaluate (ImuFactor.h:63-165), the identity
ambient x local Jacobian = tangent Jacobian against tests/imu_factor_reference.py, the marginalisation-ordering scatter of pair
{0, 1}, and synth.window_imu_problem's records."""
import numpy as np
import pytest

from glio_b200 import api, synth
from tests import imu_factor_reference as ir
from tests import window_imu_reference as wr


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _qleft(q):
    """math_tools.h Qleft on (w, x, y, z)"""
    m = np.zeros((4, 4)); m[0, 0] = q[0]; m[0, 1:] = -q[1:]; m[1:, 0] = q[1:]; m[1:, 1:] = q[0] * np.eye(3) + _skew(q[1:])
    return m


def _qright(p):
    """math_tools.h Qright on (w, x, y, z)"""
    m = np.zeros((4, 4)); m[0, 0] = p[0]; m[0, 1:] = -p[1:]; m[1:, 0] = p[1:]; m[1:, 1:] = p[0] * np.eye(3) - _skew(p[1:])
    return m


def _left_quat_matrix(q):
    """math_tools.h LeftQuatMatrix: top-left 3 x 3 = w I + [v]x"""
    m = np.zeros((4, 4)); m[:3, :3] = q[0] * np.eye(3) + _skew(q[1:]); m[3, :3] = -q[1:]; m[:3, 3] = q[1:]; m[3, 3] = q[0]
    return m


def _qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def _qinv(q):
    return np.array([q[0], -q[1], -q[2], -q[3]]) / np.dot(q, q)


def _rot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _ambient_blocks(poses, sb, F):
    """ImuFactor::Evaluate's six Jacobian blocks for one factor F, as written (ImuFactor.h:63-165), stitched into the ambient
    15 x 32 matrix over (P_i, Q_i (4), SB_i, P_j, Q_j (4), SB_j); sqrt_info applied"""
    i, j = int(F["i"]), int(F["j"])
    Pi, Pj = poses[i, :3], poses[j, :3]
    Qi = poses[i, 3:] / np.linalg.norm(poses[i, 3:]); Qj = poses[j, 3:] / np.linalg.norm(poses[j, 3:])
    Vi, Bgi = sb[i, :3], sb[i, 6:]
    Vj = sb[j, :3]
    T, g = float(F["sum_dt"]), F["g_vec"]
    dp_dba, dp_dbg, dq_dbg, dv_dba, dv_dbg = F["dp_dba"], F["dp_dbg"], F["dq_dbg"], F["dv_dba"], F["dv_dbg"]
    S = F["sqrt_info"]
    cdq = _qmul(F["delta_q"], np.concatenate([[1.0], dq_dbg @ (Bgi - F["linearized_bg"]) / 2.0]))
    Ri_inv = _rot(_qinv(Qi))
    w, vec = Qi[0], Qi[1:]
    J0 = np.zeros((15, 3)); J0[0:3] = -Ri_inv
    J1 = np.zeros((15, 4))
    tmp = -0.5 * g * T * T + Pj - Pi - Vi * T
    J1[0:3, 0] = 2 * (w * tmp + _skew(vec) @ tmp)
    J1[0:3, 1:] = 2 * (vec.dot(tmp) * np.eye(3) + np.outer(vec, tmp) - np.outer(tmp, vec) - w * _skew(tmp))
    J1[3:6, :] = -2 * (_qleft(_qinv(Qj)) @ _qright(cdq))[1:, :]
    tmp1 = -g * T + Vj - Vi
    J1[6:9, 0] = 2 * (w * tmp1 + _skew(vec) @ tmp1)
    J1[6:9, 1:] = 2 * (vec.dot(tmp1) * np.eye(3) + np.outer(vec, tmp1) - np.outer(tmp1, vec) - w * _skew(tmp1))
    J2 = np.zeros((15, 9))
    J2[0:3, 0:3] = -Ri_inv * T; J2[0:3, 3:6] = -dp_dba; J2[0:3, 6:9] = -dp_dbg
    J2[3:6, 6:9] = -_left_quat_matrix(_qmul(_qmul(_qinv(Qj), Qi), cdq))[:3, :3] @ dq_dbg
    J2[6:9, 0:3] = -Ri_inv; J2[6:9, 3:6] = -dv_dba; J2[6:9, 6:9] = -dv_dbg
    J2[9:12, 3:6] = -np.eye(3); J2[12:15, 6:9] = -np.eye(3)
    J3 = np.zeros((15, 3)); J3[0:3] = Ri_inv
    J4 = np.zeros((15, 4)); J4[3:6, :] = 2 * _qleft(_qmul(_qinv(cdq), _qinv(Qi)))[1:, :]
    J5 = np.zeros((15, 9)); J5[6:9, 0:3] = Ri_inv; J5[9:12, 3:6] = np.eye(3); J5[12:15, 6:9] = np.eye(3)
    return S @ np.concatenate([J0, J1, J2, J3, J4, J5], axis=1)


def _quirky(P, seed):
    rng = np.random.default_rng(seed)
    W = len(P["poses_init"])
    poses = P["poses_init"].copy(); sb = P["sb_init"].copy()
    poses[:, 3:] *= rng.uniform(0.7, 1.4, (W, 1)); poses[1::3, 3:] *= -1.0
    poses[:, :3] += np.array([20_000.0, -12_000.0, 150.0])
    sb[:, 6:] += rng.normal(0.0, 0.01, (W, 3))
    return poses, sb


@pytest.fixture(scope="module")
def problem():
    return synth.window_imu_problem(W=6, Q=500, M=5000, seed=41)


def test_ambient_blocks_match_the_transliteration(problem):
    P = problem
    for poses, sb in ((P["poses_init"], P["sb_init"]), _quirky(P, 3)):
        f = api.imu_factor_records(**P["imu"])
        J4 = wr.ambient_jacobian4(poses, sb, f).astype(np.float64)
        for n in range(len(f)):
            T = _ambient_blocks(poses, sb, f[n])
            scale = np.max(np.abs(T), axis=0, keepdims=True) + 1e-300
            assert np.max(np.abs(J4[n] - T) / scale) <= 1e-10, n
        # the x, y, z columns are what imu_blocks (jac_kind 1) uses
        R = wr.factor_residuals(poses, sb, f)
        xyz = [c for h in (0, 16) for c in list(range(h, h + 3)) + list(range(h + 4, h + 16))]
        assert np.array_equal(R["J"].astype(np.float64), J4[:, :, xyz])


def test_ambient_times_local_jacobian_is_the_tangent_reference(problem):
    P = problem
    poses, sb = _quirky(P, 5)
    cols = dict(P["imu"]); i, j = cols["i"].copy(), cols["j"].copy()
    cols["i"][::2], cols["j"][::2] = j[::2], i[::2]                     # i > j: the pair's columns are (x_j, x_i)
    f = api.imu_factor_records(**cols)
    J4 = wr.ambient_jacobian4(poses, sb, f)
    tan = ir.factor_residuals(poses, sb, f)["J"]
    a = np.minimum(f["i"], f["j"]); b = np.maximum(f["i"], f["j"])
    for n in range(len(f)):
        out = []
        for h, k in ((0, a[n]), (16, b[n])):
            q = poses[k, 3:].astype(ir.LD)
            L = np.array([[-q[1], -q[2], -q[3]], [q[0], q[3], -q[2]], [-q[3], q[0], q[1]], [q[2], -q[1], q[0]]], ir.LD)
            out += [J4[n][:, h:h + 3], J4[n][:, h + 3:h + 7] @ L, J4[n][:, h + 7:h + 16]]
        mine = np.concatenate(out, axis=1)
        scale = np.max(np.abs(tan[n]), axis=0, keepdims=True) + 1e-300
        assert float(np.max(np.abs(mine - tan[n]) / scale)) <= 1e-15, n


def test_marginalisation_scatter_of_pair_01(problem):
    P = problem
    W = len(P["poses_init"]); N = 6 * W + 18
    poses, sb = _quirky(P, 7)
    f = api.imu_factor_records(**P["imu"])
    f = np.concatenate([f, f[:1]]); f["i"][-1], f["j"][-1] = 1, 0       # two factors on {0, 1}, one of them with i > j
    A, MA, b, Mb = wr.marg_pair01(poses, sb, f, N)
    only = f[(np.minimum(f["i"], f["j"]) == 0)]
    blk = wr.imu_blocks(poses[:2], sb[:2], only)                          # W = 2: KF0 and KF1 alone
    assert np.allclose(A[:15, :15], blk["Hdiag"][0], rtol=0, atol=1e-12 * np.max(np.abs(A)))
    assert np.allclose(A[15:30, 15:30], blk["Hdiag"][1], rtol=0, atol=1e-12 * np.max(np.abs(A)))
    assert np.allclose(A[:15, 15:30], blk["Hoff"][0], rtol=0, atol=1e-12 * np.max(np.abs(A)))
    assert np.array_equal(A[:15, 15:30], A[15:30, :15].T)
    assert np.allclose(b[:30], blk["g"].reshape(30), rtol=0, atol=1e-12 * np.max(np.abs(b)))
    assert not A[30:].any() and not A[:, 30:].any() and not b[30:].any()
    # factors away from slot 0, and inactive ones, take no part
    g = f.copy(); g["active"][0] = 0; g["active"][-1] = 0
    A0, _, b0, _ = wr.marg_pair01(poses, sb, g, N)
    assert not A0.any() and not b0.any()


def test_generator_records_and_noise():
    W = 20
    P = synth.window_imu_problem(W=W, Q=500, M=5000, seed=43)
    f = api.imu_factor_records(**P["imu"])
    assert f.dtype == api.IMU_FACTOR_DTYPE and len(f) == W - 1
    assert np.array_equal(f["i"], np.arange(W - 1)) and np.array_equal(f["j"], np.arange(1, W)) and np.all(f["active"] == 1)
    assert np.all(f["reserved"] == 0)
    assert np.allclose(f["sum_dt"], np.diff(P["kf_times"]), rtol=0, atol=0) and np.all((f["sum_dt"] > 0.25) & (f["sum_dt"] < 0.45))
    for n in range(len(f)):
        S = f["sqrt_info"][n]
        assert np.array_equal(S, np.triu(S))                                # LLT(cov^-1).matrixL()^T is upper triangular
        assert np.allclose(S, np.linalg.cholesky(np.linalg.inv(P["cov"][n])).T, rtol=1e-12, atol=0)
        assert np.allclose(S.T @ S, np.linalg.inv(P["cov"][n]), rtol=1e-9, atol=1e-9 * np.max(np.abs(S.T @ S)))
    assert np.allclose(np.linalg.norm(f["delta_q"], axis=1), 1.0, rtol=0, atol=1e-15)
    # at the truth the whitened residual is N(0, I) noise: 15 (W - 1) squares average about 1
    r = ir.factor_residuals(P["poses_true"], P["sb_true"], f)["r"].astype(np.float64)
    assert 0.6 < float(np.mean(r * r)) < 1.5
    # the window's own LiDAR problem is window_problem's
    Q = synth.window_problem(W=W, Q=500, M=5000, seed=43)
    assert np.array_equal(P["poses_init"], Q["poses_init"]) and np.array_equal(P["map_xyz"], Q["map_xyz"])
