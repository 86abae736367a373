"""Extended-precision reference of the binary point-to-edge factor (K2be, glio_eval_binary_edge), built on tests/eval_reference.py's
longdouble dual numbers and magnitude shadows.  Helper module for the tests (not collected).

  p_w = q_c * cp + t_c,  A = q_o * a + t_o,  B = q_o * b + t_o,  r = s |(p_w - A) x (p_w - B)| / |A - B|

with Eigen's quaternion polynomial and Ceres' tangent columns [t_c | d_c | t_o | d_o] (12 lanes); no loss.  The error bound of
eval_reference applies unchanged (the chain is the edge factor's with a second rotation, well below 64 roundings deep).
"""
import numpy as np

from tests import eval_reference as ev

LD = ev.LD


def binary_edge_residuals(pose_c, pose_o, cp, pa, pb, s):
    """Per-residual r, J (N, 12) and their shadows: pose_c / pose_o (7,) or (N, 7), cp in cur's frame, pa / pb in oth's (float32),
    s the score as the device stores it (float32 values)."""
    cp = np.asarray(cp, np.float32).reshape(-1, 3).astype(LD)
    pa = np.asarray(pa, np.float32).reshape(-1, 3).astype(LD); pb = np.asarray(pb, np.float32).reshape(-1, 3).astype(LD)
    N, k = len(cp), 12
    pc = np.asarray(pose_c, np.float64).reshape(-1, 7); po = np.asarray(pose_o, np.float64).reshape(-1, 7)
    tc = ev.trans_dual(pc[:, :3], N, k, 0); qc = ev.quat_dual(pc[:, 3:], N, k, 3, 0)
    to = ev.trans_dual(po[:, :3], N, k, 6); qo = ev.quat_dual(po[:, 3:], N, k, 9, 0)
    pw = ev.qrot(qc, [ev.const(cp[:, c], N, k) for c in range(3)]); pw = [pw[c] + tc[c] for c in range(3)]
    A = ev.qrot(qo, [ev.const(pa[:, c], N, k) for c in range(3)]); A = [A[c] + to[c] for c in range(3)]
    B = ev.qrot(qo, [ev.const(pb[:, c], N, k) for c in range(3)]); B = [B[c] + to[c] for c in range(3)]
    e = ev.cross([pw[c] - A[c] for c in range(3)], [pw[c] - B[c] for c in range(3)])
    sv = np.broadcast_to(np.asarray(s, np.float32).astype(LD), (N,))
    r = ev.norm3(e) / ev.norm3([A[c] - B[c] for c in range(3)]) * ev.const(sv, N, k)
    rc, Mr, J, MJ, cost, Mc = ev.huber_correct(r, 0.0)
    return dict(r=rc, Mr=Mr, J=J, MJ=MJ, cost=cost, Mcost=Mc)


def binary_edge_blocks(poses, pairs):
    """pairs: list of (cur, oth, dict(cp, pa, pb, s) or None) in pair-list order.  Returns Hdiag (K,6,6), g (K,6), Hoff (P,6,6),
    cost and their shadows, as eval_reference.binary_blocks does for the plane factor."""
    K = len(poses); P = len(pairs)
    out = dict(Hdiag=np.zeros((K, 6, 6), LD), MHdiag=np.zeros((K, 6, 6), LD), g=np.zeros((K, 6), LD), Mg=np.zeros((K, 6), LD),
               Hoff=np.zeros((P, 6, 6)), MHoff=np.zeros((P, 6, 6)), cost=LD(0), Mcost=LD(0))
    poses = np.asarray(poses, np.float64)
    c6, o6 = slice(0, 6), slice(6, 12)
    for p, (cur, oth, m) in enumerate(pairs):
        if m is None or len(m["cp"]) == 0:
            continue
        R = binary_edge_residuals(poses[cur], poses[oth], m["cp"], m["pa"], m["pb"], m["s"])
        J, MJ, r, Mr = R["J"], R["MJ"], R["r"], R["Mr"]
        for kfi, sl in ((cur, c6), (oth, o6)):
            H, MH, g, Mg, _, _ = ev._blocks(J, MJ, r, Mr, R["cost"], R["Mcost"], sl, sl)
            out["Hdiag"][kfi] += H; out["MHdiag"][kfi] += MH; out["g"][kfi] += g; out["Mg"][kfi] += Mg
        H, MH, _, _, c, Mc = ev._blocks(J, MJ, r, Mr, R["cost"], R["Mcost"], c6, o6)
        out["Hoff"][p], out["MHoff"][p] = H, MH
        out["cost"] += c; out["Mcost"] += Mc
    for key in ("Hdiag", "MHdiag", "g", "Mg"):
        out[key] = out[key].astype(np.float64)
    out["cost"], out["Mcost"] = float(out["cost"]), float(out["Mcost"])
    return out


def make_pair_edges(rng, pose_c, pose_o, n, noise=0.08):
    """n binary edge correspondences of pair (cur, oth): cp in cur's body frame, a line (pa, pb) in oth's, the world point near
    the world line; s in [1, 8] as float32 values."""
    tc, qc, to, qo = pose_c[:3], pose_c[3:], pose_o[:3], pose_o[3:]
    a = tc + rng.uniform(-20, 20, (n, 3)); d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1)[:, None]
    b = a + d * rng.uniform(0.2, 1.0, (n, 1))
    pw = a + d * rng.uniform(-1, 2, (n, 1)) + rng.normal(0, noise, (n, 3))
    cp = np.linalg.solve(ev.rot_poly(qc), (pw - tc).T).T.astype(np.float32)
    Ro = ev.rot_poly(qo)
    al = np.linalg.solve(Ro, (a - to).T).T.astype(np.float32); bl = np.linalg.solve(Ro, (b - to).T).T.astype(np.float32)
    s = rng.uniform(1.0, 8.0, n).astype(np.float32).astype(np.float64)
    return dict(cp=cp, pa=al, pb=bl, s=s)
