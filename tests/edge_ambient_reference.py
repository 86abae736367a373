"""LidarEdgeFactor with the ambient x,y,z quaternion columns (the marginalisation's Jacobian, MarginalizationFactor.cpp:9-17), in
numpy.longdouble with dual-number derivatives: tests/eval_reference.py's edge_residuals with q's x, y, z seeded directly."""
import numpy as np

from tests import eval_reference as ev


def edge_residuals(pose, cp, pa, pb, s, q_lb, t_lb, huber_delta, jac_kind=1):
    cp = np.asarray(cp, np.float32).reshape(-1, 3).astype(ev.LD)
    pa = np.asarray(pa, np.float32).reshape(-1, 3).astype(ev.LD); pb = np.asarray(pb, np.float32).reshape(-1, 3).astype(ev.LD)
    N, k = len(cp), 6
    pose = np.asarray(pose, np.float64).reshape(-1, 7)
    t = ev.trans_dual(pose[:, :3], N, k, 0)
    q = ev.quat_dual(pose[:, 3:], N, k, 3, jac_kind)
    qi = ev.qinv_const(q_lb)
    tlb = np.asarray(t_lb, np.float64).astype(ev.LD)
    d = [ev.const(cp[:, c], N, k) - ev.const(tlb[c], N, k) for c in range(3)]
    lp = ev.qrot(q, ev.qrot([ev.const(qi[c], N, k) for c in range(4)], d))
    lp = [lp[c] + t[c] for c in range(3)]
    a = [ev.const(pa[:, c], N, k) for c in range(3)]; b = [ev.const(pb[:, c], N, k) for c in range(3)]
    e = ev.cross([lp[c] - a[c] for c in range(3)], [lp[c] - b[c] for c in range(3)])
    r = ev.norm3(e) / ev.norm3([a[c] - b[c] for c in range(3)]) * ev.const(np.asarray(s, np.float64).astype(ev.LD), N, k)
    rc, Mr, J, MJ, cost, Mc = ev.huber_correct(r, huber_delta)
    return dict(r=rc, Mr=Mr, J=J, MJ=MJ, cost=cost, Mcost=Mc)


def blocks(pose, cp, pa, pb, s, q_lb, t_lb, huber_delta, jac_kind=1):
    """6x6 H, g and cost of one keyframe's edges, in longdouble."""
    R = edge_residuals(pose, cp, pa, pb, s, q_lb, t_lb, huber_delta, jac_kind)
    J, r = R["J"], R["r"]
    return J.T @ J, J.T @ r, np.sum(R["cost"])
