"""Extended-precision reference of the window marginalisation's IMU blocks (glio_eval_window_imu_factors with jac_kind 1, and
the pair {0, 1} part of glio_window_marginalize).  Helper module for the tests (not collected).

The marginalisation reads ImuFactor's ambient 15 x 4 quaternion blocks (ImuFactor.h:77-100 and :139-150), of which
ThreadsConstructA keeps the x, y, z columns (rightCols(3), MarginalizationFactor.cpp:3-29).  tests/imu_factor_reference.py
restates the factor with its quaternion blocks multiplied by Ceres' local Jacobian; this module reuses that restatement as it is,
with the local Jacobian replaced by constant unit directions of the 4-vector parameter (ambient columns), so every other column,
sqrt_info and the magnitude shadows (and so the error bound, KAPPA 2^-53 M) are the same.
"""
import contextlib

import numpy as np

from tests import imu_factor_reference as ir

LD = ir.LD
AMBIENT_XYZ = (1, 2, 3)           # the x, y, z entries of (w, x, y, z)


@contextlib.contextmanager
def _ambient(cols):
    """imu_factor_reference with its quaternion columns along the unit directions e_c, c in cols, of the 4-vector parameter"""
    saved = ir.local_jac

    def select(q):
        shape = q[0].v.shape
        return [[ir.c(np.full(shape, 1.0 if r == k else 0.0)) for k in cols] for r in range(4)]
    ir.local_jac = select
    try:
        yield
    finally:
        ir.local_jac = saved


def factor_residuals(poses, sb, f, cols=AMBIENT_XYZ):
    """imu_factor_reference.factor_residuals with the quaternion columns of (x_a, x_b) along e_c, c in cols (three of 0..3)"""
    with _ambient(cols):
        return ir.factor_residuals(poses, sb, f)


def imu_blocks(poses, sb, f):
    """glio_eval_window_imu_factors' outputs with jac_kind 1 (ambient x, y, z columns), imu_factor_reference.imu_blocks' layout"""
    with _ambient(AMBIENT_XYZ):
        return ir.imu_blocks(poses, sb, f)


def ambient_jacobian4(poses, sb, f):
    """Per factor the full ambient Jacobian (N, 15, 32) over (t_a, q_a (4), v_a, ba_a, bg_a, t_b, q_b (4), ...), sqrt_info applied"""
    wxy = factor_residuals(poses, sb, f, (0, 1, 2))["J"]
    xyz = factor_residuals(poses, sb, f, AMBIENT_XYZ)["J"]
    out = []
    for h in (0, 15):
        out += [xyz[:, :, h:h + 3], wxy[:, :, h + 3:h + 4], xyz[:, :, h + 3:h + 15]]
    return np.concatenate(out, axis=2)


def marg_pair01(poses, sb, f, N):
    """What the marginalisation adds for the window IMU list f: the active factors on pair {0, 1}, ambient x, y, z columns, as
    A (N x N) and b (N) at the marginalisation ordering (KF0 [0, 15), KF1 [15, 30)), with their magnitude shadows (float64)."""
    A = np.zeros((N, N), LD); MA = np.zeros((N, N), LD); b = np.zeros(N, LD); Mb = np.zeros(N, LD)
    sel = (f["active"] != 0) & (np.minimum(f["i"], f["j"]) == 0) & (np.maximum(f["i"], f["j"]) == 1)
    if sel.any():
        R = factor_residuals(poses, sb, f[sel])
        J, MJ, r, Mr = R["J"], R["MJ"], R["r"], R["Mr"]
        A[:30, :30] = np.einsum("nra,nrb->ab", J, J)
        MA[:30, :30] = np.einsum("nra,nrb->ab", MJ, np.abs(J)) + np.einsum("nra,nrb->ab", np.abs(J), MJ)
        b[:30] = np.einsum("nra,nr->a", J, r)
        Mb[:30] = np.einsum("nra,nr->a", MJ, np.abs(r)) + np.einsum("nra,nr->a", np.abs(J), Mr)
    return A.astype(np.float64), MA.astype(np.float64), b.astype(np.float64), Mb.astype(np.float64)
