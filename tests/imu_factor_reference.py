"""Extended-precision reference of the batch refinement's IMU factor (K2i, glio_eval_imu_factors), independent of the device
code.  Helper module for the tests (not collected).

ImuFactor::Evaluate (ImuFactor.h:21-171, the residual of Preintegration::evaluate) is restated as written, with Eigen's semantics:
Q_i and Q_j normalised by normalize(), ``inverse() = conj / |q|^2``, ``q * v`` the _transformVector polynomial, deltaQ(theta) =
(1, theta / 2), products left to right.  The Jacobian is the factor's analytic one (not the derivative of r): its ambient 15 x 4
quaternion blocks are multiplied by Ceres' QuaternionParameterization local Jacobian at the unnormalised parameter, then every
column by sqrt_info.  Columns per factor: the 30 tangent columns (x_a, x_b), x = [t, delta, v, ba, bg], of its pair (a, b) =
(min(i, j), max(i, j)).

Error bound.  Every value carries eval_reference's magnitude shadow (a Dual without derivative lanes): sums add shadows, a product
ab gets M_a |b| + |a| M_b, the division and the 4-norm of the normalisation propagate them the same way.  The double evaluation
differs from the exact one by at most kappa 2^-53 M with kappa = 2^9: the residual chain is about 30 roundings deep (the
normalisation, the inverse, two or three quaternion products, the rotation polynomial, the 3 x 3 bias corrections), the sqrt_info
product adds 15, J^T J and J^T r 15 more, and the sums over a pair's factors and a keyframe's two pairs a handful; the cost is
summed over 15 rows by a 5-step butterfly.  All far below 512.
"""
import numpy as np

from tests import eval_reference as ev

LD = ev.LD
KAPPA, U = ev.KAPPA, ev.U
Dual = ev.Dual


def c(x):
    """a constant (N,) array as a Dual without derivative lanes"""
    v = np.asarray(x, LD)
    return Dual(v, np.zeros((0,) + v.shape, LD), np.abs(v), np.zeros((0,) + v.shape, LD))


def qmul(a, b):
    """Eigen's quaternion product on (w, x, y, z) lists"""
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
            a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]]


def qinv(q):
    n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    return [q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2]


def qnormalize(q):
    """Eigen's normalize(): q / sqrt(|q|^2); the norm's shadow as eval_reference.norm3 forms it"""
    v = np.sqrt(sum(x.v * x.v for x in q))
    mv = np.sqrt(sum(x.mv ** 2 for x in q)) + v
    n = Dual(v, np.zeros_like(q[0].d), mv, np.zeros_like(q[0].md))
    return [x / n for x in q]


def rotmat(q):
    """Eigen's toRotationMatrix() of q, as a 3 x 3 list of lists"""
    w, x, y, z = q
    tx, ty, tz = x + x, y + y, z + z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    one = c(np.ones_like(w.v))
    return [[one - (tyy + tzz), txy - twz, txz + twy], [txy + twz, one - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, one - (txx + tyy)]]


def mat3v(M, v):
    """M (N, 3, 3) constant times the list v"""
    return [c(M[:, r, 0]) * v[0] + c(M[:, r, 1]) * v[1] + c(M[:, r, 2]) * v[2] for r in range(3)]


def local_jac(q):
    """Ceres' QuaternionParameterization 4 x 3 local Jacobian at q (w, x, y, z): columns [0, e_k] (x) q"""
    w, x, y, z = q
    return [[-x, -y, -z], [w, z, -y], [-z, w, x], [y, -x, w]]


def _zero(N):
    return c(np.zeros(N))


def factor_residuals(poses, sb, f):
    """Per factor of the IMU_FACTOR_DTYPE array f at poses (K, 7), sb (K, 9): r (N, 15), J (N, 15, 30) over (x_a, x_b), cost (N,)
    and their magnitude shadows; also r_raw (N, 15) before sqrt_info."""
    poses = np.asarray(poses, np.float64); sb = np.asarray(sb, np.float64)
    N = len(f)
    i, j = f["i"].astype(np.int64), f["j"].astype(np.int64)
    Pi = [c(poses[i, k]) for k in range(3)]; Pj = [c(poses[j, k]) for k in range(3)]
    qi_raw = [c(poses[i, 3 + k]) for k in range(4)]; qj_raw = [c(poses[j, 3 + k]) for k in range(4)]
    Vi = [c(sb[i, k]) for k in range(3)]; Vj = [c(sb[j, k]) for k in range(3)]
    Bai = [c(sb[i, 3 + k]) for k in range(3)]; Baj = [c(sb[j, 3 + k]) for k in range(3)]
    Bgi = [c(sb[i, 6 + k]) for k in range(3)]; Bgj = [c(sb[j, 6 + k]) for k in range(3)]
    qi, qj = qnormalize(qi_raw), qnormalize(qj_raw)
    qii = qinv(qi)
    T = c(f["sum_dt"]); g = [c(f["g_vec"][:, k]) for k in range(3)]
    dba = [Bai[k] - c(f["linearized_ba"][:, k]) for k in range(3)]
    dbg = [Bgi[k] - c(f["linearized_bg"][:, k]) for k in range(3)]
    th = mat3v(f["dq_dbg"], dbg)
    dQ = [c(np.ones(N))] + [x / LD(2) for x in th]
    cdq = qmul([c(f["delta_q"][:, k]) for k in range(4)], dQ)
    ca, cb = mat3v(f["dp_dba"], dba), mat3v(f["dp_dbg"], dbg)
    cdp = [c(f["delta_p"][:, k]) + ca[k] + cb[k] for k in range(3)]
    ca, cb = mat3v(f["dv_dba"], dba), mat3v(f["dv_dbg"], dbg)
    cdv = [c(f["delta_v"][:, k]) + ca[k] + cb[k] for k in range(3)]
    tmp = [LD(-0.5) * g[k] * T * T + Pj[k] - Pi[k] - Vi[k] * T for k in range(3)]
    tmp1 = [-g[k] * T + Vj[k] - Vi[k] for k in range(3)]
    rp, rv = ev.qrot(qii, tmp), ev.qrot(qii, tmp1)
    E = qnormalize(qmul(qinv(cdq), qmul(qii, qj)))
    raw = ([rp[k] - cdp[k] for k in range(3)] + [LD(2) * E[1 + k] for k in range(3)] + [rv[k] - cdv[k] for k in range(3)]
           + [Baj[k] - Bai[k] for k in range(3)] + [Bgj[k] - Bgi[k] for k in range(3)])

    # the raw Jacobian, 15 rows x 30 columns (t_i, d_i, v_i, ba_i, bg_i, t_j, d_j, v_j, ba_j, bg_j)
    Jr = [[_zero(N) for _ in range(30)] for _ in range(15)]
    R = rotmat(qii)
    one = c(np.ones(N))
    for e in range(3):
        for m in range(3):
            Jr[m][e] = -R[m][e]                       # t_i
            Jr[m][15 + e] = R[m][e]                   # t_j
            Jr[m][6 + e] = -R[m][e] * T               # v_i, P rows
            Jr[6 + m][6 + e] = -R[m][e]               # v_i, V rows
            Jr[6 + m][21 + e] = R[m][e]               # v_j
            Jr[m][9 + e] = -c(f["dp_dba"][:, m, e])
            Jr[6 + m][9 + e] = -c(f["dv_dba"][:, m, e])
            Jr[m][12 + e] = -c(f["dp_dbg"][:, m, e])
            Jr[6 + m][12 + e] = -c(f["dv_dbg"][:, m, e])
        Jr[9 + e][9 + e] = -one; Jr[12 + e][12 + e] = -one
        Jr[9 + e][24 + e] = one; Jr[12 + e][27 + e] = one
    # bg_i, rotation rows: -LeftQuatMatrix(Q_j^-1 Q_i cdq).topLeftCorner<3,3>() dq_dbg
    M = qmul(qmul(qinv(qj), qi), cdq)
    for e in range(3):
        col = [c(f["dq_dbg"][:, k, e]) for k in range(3)]
        vxc = ev.cross(M[1:], col)
        for m in range(3):
            Jr[3 + m][12 + e] = -(M[0] * col[m] + vxc[m])
    # quaternion blocks: ambient 15 x 4, times the local Jacobian
    w, u = qi[0], qi[1:]

    def qi_rows(t, dcol):
        ut, td, ud = ev.dot(u, t), ev.dot(t, dcol[1:]), ev.dot(u, dcol[1:])
        uxt, txd = ev.cross(u, t), ev.cross(t, dcol[1:])
        return [LD(2) * (dcol[0] * (w * t[m] + uxt[m]) + ut * dcol[1 + m] + u[m] * td - t[m] * ud - w * txd[m]) for m in range(3)]
    Li, Lj = local_jac(qi_raw), local_jac(qj_raw)
    qji = qinv(qj)
    cinv_qii = qmul(qinv(cdq), qii)
    for e in range(3):
        di = [Li[r][e] for r in range(4)]
        dj = [Lj[r][e] for r in range(4)]
        p_rows, v_rows = qi_rows(tmp, di), qi_rows(tmp1, di)
        o4 = qmul(qji, qmul(di, cdq))
        o4j = qmul(cinv_qii, dj)
        for m in range(3):
            Jr[m][3 + e] = p_rows[m]
            Jr[6 + m][3 + e] = v_rows[m]
            Jr[3 + m][3 + e] = LD(-2) * o4[1 + m]
            Jr[3 + m][18 + e] = LD(2) * o4j[1 + m]

    rawv = np.stack([x.v for x in raw], axis=1); rawm = np.stack([x.mv for x in raw], axis=1)
    Jv = np.stack([np.stack([x.v for x in row], axis=1) for row in Jr], axis=1)
    Jm = np.stack([np.stack([x.mv for x in row], axis=1) for row in Jr], axis=1)
    S = f["sqrt_info"].astype(LD); aS = np.abs(S)
    r = np.einsum("nab,nb->na", S, rawv); Mr = np.einsum("nab,nb->na", aS, np.abs(rawv) + rawm)
    J = np.einsum("nab,nbc->nac", S, Jv); MJ = np.einsum("nab,nbc->nac", aS, np.abs(Jv) + Jm)
    sw = i > j
    J[sw] = np.concatenate([J[sw][:, :, 15:], J[sw][:, :, :15]], axis=2); MJ[sw] = np.concatenate([MJ[sw][:, :, 15:], MJ[sw][:, :, :15]], axis=2)
    cost = LD(0.5) * np.sum(r * r, axis=1); Mcost = np.sum(np.abs(r) * Mr, axis=1)
    return dict(r=r, Mr=Mr, J=J, MJ=MJ, cost=cost, Mcost=Mcost, r_raw=rawv)


def pair_table(f):
    """The distinct pairs (a, b), a < b, in order of first appearance, and each factor's pair index."""
    index, pairs, fp = {}, [], np.zeros(len(f), np.int64)
    for n, (i, j) in enumerate(zip(f["i"], f["j"])):
        key = (int(min(i, j)), int(max(i, j)))
        if key not in index:
            index[key] = len(pairs); pairs.append(key)
        fp[n] = index[key]
    return pairs, fp


def imu_blocks(poses, sb, f):
    """glio_eval_imu_factors' outputs for the active factors of f: Hdiag (K,15,15), g (K,15), Hoff (P,15,15) in pair-table order,
    cost, with shadows (float64)."""
    K = len(poses)
    pairs, fp = pair_table(f)
    P = len(pairs)
    out = dict(Hdiag=np.zeros((K, 15, 15), LD), MHdiag=np.zeros((K, 15, 15), LD), g=np.zeros((K, 15), LD), Mg=np.zeros((K, 15), LD),
               Hoff=np.zeros((P, 15, 15), LD), MHoff=np.zeros((P, 15, 15), LD), cost=LD(0), Mcost=LD(0), pairs=pairs)
    act = f["active"] != 0
    if act.any():
        R = factor_residuals(poses, sb, f[act])
        J, MJ, r, Mr = R["J"], R["MJ"], R["r"], R["Mr"]
        H = np.einsum("nra,nrb->nab", J, J)
        MH = np.einsum("nra,nrb->nab", MJ, np.abs(J)) + np.einsum("nra,nrb->nab", np.abs(J), MJ)
        g = np.einsum("nra,nr->na", J, r)
        Mg = np.einsum("nra,nr->na", MJ, np.abs(r)) + np.einsum("nra,nr->na", np.abs(J), Mr)
        p = fp[act]
        ab = np.asarray(pairs, np.int64).reshape(-1, 2)
        a, b = ab[p, 0], ab[p, 1]
        for key, src, sl in (("Hdiag", H, np.s_[:, :15, :15]), ("MHdiag", MH, np.s_[:, :15, :15]), ("g", g, np.s_[:, :15]), ("Mg", Mg, np.s_[:, :15])):
            np.add.at(out[key], a, src[sl])
        for key, src, sl in (("Hdiag", H, np.s_[:, 15:, 15:]), ("MHdiag", MH, np.s_[:, 15:, 15:]), ("g", g, np.s_[:, 15:]), ("Mg", Mg, np.s_[:, 15:])):
            np.add.at(out[key], b, src[sl])
        np.add.at(out["Hoff"], p, H[:, :15, 15:]); np.add.at(out["MHoff"], p, MH[:, :15, 15:])
        out["cost"] = np.sum(R["cost"]); out["Mcost"] = np.sum(R["Mcost"])
    for key in ("Hdiag", "MHdiag", "g", "Mg", "Hoff", "MHoff"):
        out[key] = out[key].astype(np.float64)
    out["cost"], out["Mcost"] = float(out["cost"]), float(out["Mcost"])
    return out
