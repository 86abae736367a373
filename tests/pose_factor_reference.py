"""Extended-precision reference of the batch refinement's pose factors (K2p, glio_eval_pose_factors), independent of the device
code.  Helper module for the tests (not collected).

Both functors are restated as they are written, with Eigen's semantics at any quaternion (``inverse() = conj / |q|^2``,
``q * v = v + 2w (u x v) + 2 u x (u x v)``, products left to right):

* LidarPoseFactorBatchRelativeAutoDiff (blocks t_i, q_i, t_j, q_j):
  ``r[0..2] = 10 (2 vec(dq^-1 q_i^-1 q_j))``, ``r[3..5] = 20 (q_i^-1 (t_j - t_i) - dp)``;
* delta_q_factor_auto (blocks q_i, q_j): ``r = 10000 vec(dq^-1 q_i^-1 q_j)`` (rows 3..5 are zero here).

Derivatives are eval_reference's forward-mode duals in numpy.longdouble with Ceres' tangent seeding, over the 12 columns
(t_a, d_a, t_b, d_b) of the factor's pair (a, b) = (min(i, j), max(i, j)).  The error bound is eval_reference's: the chain is
about 30 roundings deep (two quaternion products, the inverse's division, the rotation polynomial), and the sums are a 6-term
dot product per entry, a pair's factors and a keyframe's pairs, far below KAPPA = 2^9.
"""
import numpy as np

from tests import eval_reference as ev

LD = ev.LD
KAPPA, U = ev.KAPPA, ev.U


def qmul(a, b):
    """Eigen's quaternion product on (w, x, y, z) lists of duals / constants."""
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
            a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]]


def qinv(q):
    n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    return [q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2]


def factor_residuals(poses, f):
    """Per factor of the POSE_FACTOR_DTYPE array f: r (N, 6), J (N, 6, 12) over (t_a, d_a, t_b, d_b), cost (N,) and their
    magnitude shadows."""
    poses = np.asarray(poses, np.float64)
    N, k = len(f), 12
    i, j = f["i"].astype(np.int64), f["j"].astype(np.int64)
    # lanes (t_i, d_i, t_j, d_j); the factors with i > j have their halves swapped at the end
    ti = ev.trans_dual(poses[i, :3], N, k, 0); qi = ev.quat_dual(poses[i, 3:], N, k, 3, 0)
    tj = ev.trans_dual(poses[j, :3], N, k, 6); qj = ev.quat_dual(poses[j, 3:], N, k, 9, 0)
    dq = f["dq"].astype(LD)
    A = qinv([ev.const(dq[:, c], N, k) for c in range(4)])
    E = qmul(qmul(A, qinv(qi)), qj)
    rel = f["kind"] == 0
    Bv = ev.qrot(qinv(qi), [tj[c] - ti[c] for c in range(3)])
    rows = []
    for c in range(3):
        rr = ev.const(np.where(rel, LD(10), LD(0)), N, k) * (LD(2) * E[1 + c]) + ev.const(np.where(rel, LD(0), LD(10000)), N, k) * E[1 + c]
        rows.append(rr)
    for c in range(3):
        rows.append(ev.const(np.where(rel, LD(20), LD(0)), N, k) * (Bv[c] - ev.const(f["dp"][:, c].astype(LD), N, k)))
    r = np.stack([x.v for x in rows], axis=1); Mr = np.stack([x.mv for x in rows], axis=1)
    J = np.stack([x.d.T for x in rows], axis=1); MJ = np.stack([x.md.T for x in rows], axis=1)
    sw = i > j
    J[sw] = np.concatenate([J[sw][:, :, 6:], J[sw][:, :, :6]], axis=2); MJ[sw] = np.concatenate([MJ[sw][:, :, 6:], MJ[sw][:, :, :6]], axis=2)
    cost = LD(0.5) * np.sum(r * r, axis=1); Mcost = np.sum(np.abs(r) * Mr, axis=1)
    return dict(r=r, Mr=Mr, J=J, MJ=MJ, cost=cost, Mcost=Mcost)


def pair_table(f):
    """The distinct pairs (a, b), a < b, in order of first appearance, and each factor's pair index."""
    index, pairs, fp = {}, [], np.zeros(len(f), np.int64)
    for n, (i, j) in enumerate(zip(f["i"], f["j"])):
        key = (int(min(i, j)), int(max(i, j)))
        if key not in index:
            index[key] = len(pairs); pairs.append(key)
        fp[n] = index[key]
    return pairs, fp


def pose_blocks(poses, f):
    """glio_eval_pose_factors' outputs for the active factors of f: Hdiag (K,6,6), g (K,6), Hoff (P,6,6) in pair-table order,
    cost, with shadows."""
    K = len(poses)
    pairs, fp = pair_table(f)
    P = len(pairs)
    out = dict(Hdiag=np.zeros((K, 6, 6), LD), MHdiag=np.zeros((K, 6, 6), LD), g=np.zeros((K, 6), LD), Mg=np.zeros((K, 6), LD),
               Hoff=np.zeros((P, 6, 6), LD), MHoff=np.zeros((P, 6, 6), LD), cost=LD(0), Mcost=LD(0), pairs=pairs)
    act = f["active"] != 0
    if act.any():
        R = factor_residuals(poses, f[act])
        J, MJ, r, Mr = R["J"], R["MJ"], R["r"], R["Mr"]
        H = np.einsum("nra,nrb->nab", J, J)
        MH = np.einsum("nra,nrb->nab", MJ, np.abs(J)) + np.einsum("nra,nrb->nab", np.abs(J), MJ)
        g = np.einsum("nra,nr->na", J, r)
        Mg = np.einsum("nra,nr->na", MJ, np.abs(r)) + np.einsum("nra,nr->na", np.abs(J), Mr)
        p = fp[act]
        ab = np.asarray(pairs, np.int64).reshape(-1, 2)
        a, b = ab[p, 0], ab[p, 1]
        for key, src, sl in (("Hdiag", H, np.s_[:, :6, :6]), ("MHdiag", MH, np.s_[:, :6, :6]), ("g", g, np.s_[:, :6]), ("Mg", Mg, np.s_[:, :6])):
            np.add.at(out[key], a, src[sl])
        for key, src, sl in (("Hdiag", H, np.s_[:, 6:, 6:]), ("MHdiag", MH, np.s_[:, 6:, 6:]), ("g", g, np.s_[:, 6:]), ("Mg", Mg, np.s_[:, 6:])):
            np.add.at(out[key], b, src[sl])
        np.add.at(out["Hoff"], p, H[:, :6, 6:]); np.add.at(out["MHoff"], p, MH[:, :6, 6:])
        out["cost"] = np.sum(R["cost"]); out["Mcost"] = np.sum(R["Mcost"])
    for key in ("Hdiag", "MHdiag", "g", "Mg", "Hoff", "MHoff"):
        out[key] = out[key].astype(np.float64)
    out["cost"], out["Mcost"] = float(out["cost"]), float(out["Mcost"])
    return out

