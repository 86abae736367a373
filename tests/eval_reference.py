"""Extended-precision reference of the LiDAR residual evaluation (K2 / K2b / K2e), independent of the device code and of the
oracle's Jets.  Helper module for the tests (not collected).

Each factor is evaluated the way the reference functors write it (LidarPlaneNormFactor, BinaryLidarPlaneNormFactor,
LidarEdgeFactor): Eigen's polynomial ``q * v = v + 2w (u x v) + 2 u x (u x v)`` for any (not necessarily unit) quaternion and
``inverse() = conj / |q|^2``.  Derivatives come from forward-mode dual numbers in ``numpy.longdouble``:

* tangent (jac_kind 0): Ceres' QuaternionParameterization, ``q [+] d = [1, d] (x) q`` to first order, and ``t + dt``;
* ambient (jac_kind 1): q's x, y, z coefficients seeded directly (the marginalisation's rightCols(3)).

Huber's loss and Ceres' corrector follow (sqrt(rho') scaling, rho' clamped at DBL_MIN; rho'' <= 0 keeps the simple branch).

Error bound.  Every value carries a magnitude shadow M >= |value|, propagated to first order through the same expression:
sums and differences add their operands' shadows (subtractions count as additions), a product ab gets M_a |b| + |a| M_b,
and the few non-polynomial steps (division, the 2-norm, Huber's sqrt(delta/|r|)) propagate their operands' shadows the same
way.  Inputs start at M = |input|.  A double-precision evaluation of the same operation in
any order then satisfies |x_fp64 - x| <= kappa * 2^-53 * M(x), where kappa bounds the number of roundings on any path:

  operation depth  <= 64   the unary chain is about 40 deep (cp - t_lb, two 3-term rotations of a degree-2 polynomial, the
                           matrix product the device folds them into, n.(a+t)+d, the score, Huber's sqrt and division,
                           J_p J_q); the edge chain, with its cross product, norms and division, stays below 64
  reduction depth  <= 448  per-thread serial sums (at most 16 residuals per thread at the shapes tested: item size / 256 /
                           2 x 2), the 5-step warp shuffle, 8 warps, and the per-keyframe sum of at most a few hundred items
  kappa = 64 + 448 = 512 = 2^9.

The reference's own error is negligible against that: longdouble has u = 2^-64 and its sums go through np.sum (pairwise).
"""
import numpy as np

LD = np.longdouble
if np.finfo(LD).eps > 1.1e-19:
    raise ImportError("eval_reference needs an extended long double (80-bit x87 or IEEE quad); this platform's is "
                      f"eps = {np.finfo(LD).eps}")

U = 2.0 ** -53           # unit roundoff of double precision
KAPPA = 2 ** 9           # see the module docstring
DBL_MIN = 2.2250738585072014e-308


def bound(M):
    """The admissible |fp64 - reference| for a quantity of magnitude shadow M."""
    return KAPPA * U * np.asarray(M, np.float64)


# ---------------------------------------------------------------------------------------------------------------------------
# forward-mode dual numbers with a magnitude shadow; v, mv: (N,), d, md: (k, N)
# ---------------------------------------------------------------------------------------------------------------------------
class Dual:
    __slots__ = ("v", "d", "mv", "md")

    def __init__(self, v, d, mv, md):
        self.v, self.d, self.mv, self.md = v, d, mv, md

    def __add__(self, o):
        o = _lift(o, self)
        return Dual(self.v + o.v, self.d + o.d, self.mv + o.mv, self.md + o.md)

    __radd__ = __add__

    def __sub__(self, o):
        o = _lift(o, self)
        return Dual(self.v - o.v, self.d - o.d, self.mv + o.mv, self.md + o.md)

    def __rsub__(self, o):
        return _lift(o, self) - self

    def __neg__(self):
        return Dual(-self.v, -self.d, self.mv, self.md)

    def __mul__(self, o):
        # first order: err(ab) <= err(a)|b| + |a|err(b) (+ the product's own rounding, covered since M_a >= |a|); after a
        # cancellation M_a >> |a|, and the product of the two shadows would count it twice
        o = _lift(o, self)
        aa, ab, da, db = np.abs(self.v), np.abs(o.v), np.abs(self.d), np.abs(o.d)
        return Dual(self.v * o.v, self.d * o.v + self.v * o.d, self.mv * ab + aa * o.mv,
                    self.md * ab + da * o.mv + self.mv * db + aa * o.md)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _lift(o, self)
        v = self.v / o.v
        d = (self.d - v * o.d) / o.v
        ab = np.abs(o.v)
        mv = (self.mv + np.abs(v) * o.mv) / ab
        md = (self.md + np.abs(d) * o.mv + np.abs(v) * o.md + np.abs(o.d) * mv) / ab
        return Dual(v, d, mv, md)


def _lift(x, like):
    if isinstance(x, Dual):
        return x
    x = np.asarray(x, LD)
    v = np.broadcast_to(x, like.v.shape).astype(LD)
    return Dual(v, np.zeros_like(like.d), np.abs(v), np.zeros_like(like.md))


def const(x, N, k):
    v = np.broadcast_to(np.asarray(x, LD), (N,)).astype(LD)
    return Dual(v, np.zeros((k, N), LD), np.abs(v), np.zeros((k, N), LD))


def var(x, lanes, N, k):
    """A value whose derivative lanes are `lanes`: {lane: seed array or scalar}."""
    out = const(x, N, k)
    for j, s in lanes.items():
        out.d[j] = s
        out.md[j] = np.abs(np.asarray(s, LD))
    return out


def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def norm3(x):
    v = np.sqrt(x[0].v * x[0].v + x[1].v * x[1].v + x[2].v * x[2].v)
    d = (x[0].v * x[0].d + x[1].v * x[1].d + x[2].v * x[2].d) / v
    mv = np.sqrt(x[0].mv ** 2 + x[1].mv ** 2 + x[2].mv ** 2) + v
    md = sum(x[i].mv * np.abs(x[i].d) + np.abs(x[i].v) * x[i].md for i in range(3)) / v + np.abs(d) * mv / v
    return Dual(v, d, mv, md)


def qrot(q, v):
    """Eigen's Quaternion * Vector3 (_transformVector): uv = u x v; uv += uv; return v + w uv + u x uv."""
    u = q[1:]
    uv = cross(u, v)
    uv = [c + c for c in uv]
    uuv = cross(u, uv)
    return [v[i] + q[0] * uv[i] + uuv[i] for i in range(3)]


def qinv_const(q):
    """Eigen's inverse() = conj / |q|^2 (of a constant quaternion)."""
    q = np.asarray(q, LD)
    n2 = np.sum(q * q)
    return np.array([q[0], -q[1], -q[2], -q[3]], LD) / n2


def quat_dual(q, N, k, first_lane, jac_kind):
    """Pose quaternion (N, 4) as duals.  jac_kind 0: lanes first..first+2 are Ceres' tangent [1, d] (x) q; 1: q's x, y, z."""
    q = np.asarray(q, LD).reshape(-1, 4)
    q = np.broadcast_to(q, (N, 4))
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    if jac_kind == 0:
        # columns of d([1, d] (x) q)/dd: (0, e_j) (x) (w, u) = (-e_j.u, w e_j + e_j x u)
        cols = [(-x, w, -z, y), (-y, z, w, -x), (-z, -y, x, w)]
        seeds = [{first_lane + j: cols[j][c] for j in range(3)} for c in range(4)]
    else:
        seeds = [{}, {first_lane: 1.0}, {first_lane + 1: 1.0}, {first_lane + 2: 1.0}]
    return [var(q[:, c], seeds[c], N, k) for c in range(4)]


def trans_dual(t, N, k, first_lane):
    t = np.broadcast_to(np.asarray(t, LD).reshape(-1, 3), (N, 3))
    return [var(t[:, c], {first_lane + c: 1.0}, N, k) for c in range(3)]


# ---------------------------------------------------------------------------------------------------------------------------
# loss
# ---------------------------------------------------------------------------------------------------------------------------
def huber_correct(r, delta):
    """Huber + Ceres' corrector on the raw residual dual r.  Returns (r, M_r, J (N, k), M_J (N, k), cost, M_cost)."""
    rv, J, Mr, MJ = r.v, r.d, r.mv, r.md
    sq = rv * rv
    outl = sq > LD(delta) * LD(delta) if delta > 0 else np.zeros(rv.shape, bool)
    a = np.abs(rv)
    safe = np.where(outl, a, LD(1))
    rho1 = np.maximum(LD(delta) / safe, LD(DBL_MIN))
    scale = np.where(outl, np.sqrt(rho1), LD(1))
    # scale = sqrt(delta / |r|): its relative error is half that of |r|
    rel = np.where(outl, Mr / safe, LD(0))
    cost = np.where(outl, LD(0.5) * (2 * LD(delta) * a - LD(delta) * LD(delta)), LD(0.5) * sq)
    Mcost = np.where(outl, LD(delta) * Mr + LD(0.5) * LD(delta) * LD(delta), a * Mr)
    Jc = J * scale
    MJc = scale * (MJ + np.abs(J) * rel)
    rc = rv * scale
    Mrc = scale * (Mr + a * rel)
    return rc, Mrc, Jc.T, MJc.T, cost, Mcost


# ---------------------------------------------------------------------------------------------------------------------------
# factors: per-residual r, J (tangent/ambient [t | rot]) and their magnitudes
# ---------------------------------------------------------------------------------------------------------------------------
def unary_residuals(pose, cp, nsd, weight, q_lb, t_lb, lidar_const, huber_delta, jac_kind=0, unit_score=False):
    """LidarPlaneNormFactor of one keyframe or per residual: pose (7,) or (N, 7); cp (N, 3) float32; nsd (N, 4) float32
    (n, negOA); weight (N,) float32.  Returns dict(r, Mr, J (N, 6), MJ, cost, Mcost) in longdouble."""
    cp = np.asarray(cp, np.float32).reshape(-1, 3).astype(LD); nsd = np.asarray(nsd, np.float32).reshape(-1, 4).astype(LD)
    N, k = len(cp), 6
    pose = np.asarray(pose, np.float64).reshape(-1, 7)
    t = trans_dual(pose[:, :3], N, k, 0)
    q = quat_dual(pose[:, 3:], N, k, 3, jac_kind)
    qi = qinv_const(q_lb)
    qic = [const(qi[c], N, k) for c in range(4)]
    tlb = np.asarray(t_lb, np.float64).astype(LD)
    d = [const(cp[:, c], N, k) - const(tlb[c], N, k) for c in range(3)]
    pb = qrot(qic, d)
    pw = qrot(q, pb)
    pw = [pw[c] + t[c] for c in range(3)]
    n = [const(nsd[:, c], N, k) for c in range(3)]
    s = LD(lidar_const) if unit_score else LD(lidar_const) * np.asarray(weight, np.float32).astype(LD)
    r = const(s, N, k) * (dot(n, pw) + const(nsd[:, 3], N, k))
    rc, Mr, J, MJ, cost, Mc = huber_correct(r, huber_delta)
    return dict(r=rc, Mr=Mr, J=J, MJ=MJ, cost=cost, Mcost=Mc)


def binary_residuals(pose_c, pose_o, cp, normal_cent, weight, batch_score, huber_delta=0.0):
    """BinaryLidarPlaneNormFactor, tangent Jacobians [t_c | d_c | t_o | d_o] (N, 12)."""
    cp = np.asarray(cp, np.float32).reshape(-1, 3).astype(LD); nc = np.asarray(normal_cent, np.float64).reshape(-1, 6).astype(LD)
    N, k = len(cp), 12
    tc = trans_dual(np.asarray(pose_c, np.float64).reshape(-1, 7)[:, :3], N, k, 0)
    qc = quat_dual(np.asarray(pose_c, np.float64).reshape(-1, 7)[:, 3:], N, k, 3, 0)
    to = trans_dual(np.asarray(pose_o, np.float64).reshape(-1, 7)[:, :3], N, k, 6)
    qo = quat_dual(np.asarray(pose_o, np.float64).reshape(-1, 7)[:, 3:], N, k, 9, 0)
    p = [const(cp[:, c], N, k) for c in range(3)]
    pw = qrot(qc, p); pw = [pw[c] + tc[c] for c in range(3)]
    Nw = qrot(qo, [const(nc[:, c], N, k) for c in range(3)])
    cw = qrot(qo, [const(nc[:, 3 + c], N, k) for c in range(3)]); cw = [cw[c] + to[c] for c in range(3)]
    s = LD(batch_score) * np.asarray(weight, np.float32).astype(LD)
    r = const(s, N, k) * dot(Nw, [pw[c] - cw[c] for c in range(3)])
    rc, Mr, J, MJ, cost, Mc = huber_correct(r, huber_delta)
    return dict(r=rc, Mr=Mr, J=J, MJ=MJ, cost=cost, Mcost=Mc)


def edge_residuals(pose, cp, pa, pb, s, q_lb, t_lb, huber_delta):
    """LidarEdgeFactor r = s |(lp - a) x (lp - b)| / |a - b|, tangent Jacobian (N, 6).  s: the score as the device stores it."""
    cp = np.asarray(cp, np.float32).reshape(-1, 3).astype(LD)
    pa = np.asarray(pa, np.float32).reshape(-1, 3).astype(LD); pb = np.asarray(pb, np.float32).reshape(-1, 3).astype(LD)
    N, k = len(cp), 6
    pose = np.asarray(pose, np.float64).reshape(-1, 7)
    t = trans_dual(pose[:, :3], N, k, 0)
    q = quat_dual(pose[:, 3:], N, k, 3, 0)
    qi = qinv_const(q_lb)
    tlb = np.asarray(t_lb, np.float64).astype(LD)
    d = [const(cp[:, c], N, k) - const(tlb[c], N, k) for c in range(3)]
    lp = qrot(q, qrot([const(qi[c], N, k) for c in range(4)], d))
    lp = [lp[c] + t[c] for c in range(3)]
    a = [const(pa[:, c], N, k) for c in range(3)]; b = [const(pb[:, c], N, k) for c in range(3)]
    e = cross([lp[c] - a[c] for c in range(3)], [lp[c] - b[c] for c in range(3)])
    r = norm3(e) / norm3([a[c] - b[c] for c in range(3)]) * const(np.asarray(s, np.float64).astype(LD), N, k)
    rc, Mr, J, MJ, cost, Mc = huber_correct(r, huber_delta)
    return dict(r=rc, Mr=Mr, J=J, MJ=MJ, cost=cost, Mcost=Mc)


# ---------------------------------------------------------------------------------------------------------------------------
# normal-equation blocks
# ---------------------------------------------------------------------------------------------------------------------------
def _blocks(J, MJ, r, Mr, cost, Mcost, rows, cols):
    """sum over residuals of J_rows^T J_cols, J_rows^T r and cost, with their magnitude shadows (pairwise np.sum).  A product's
    shadow is first order, M(ab) = M_a |b| + |a| M_b: after Huber's scaling M_J / |J| carries the relative error of sqrt(delta/|r|),
    which the plain product of shadows would square."""
    Ja, Jb, Ma, Mb = J[:, rows], J[:, cols], MJ[:, rows], MJ[:, cols]
    H = np.sum(Ja[:, :, None] * Jb[:, None, :], axis=0)
    MH = np.sum(Ma[:, :, None] * np.abs(Jb)[:, None, :] + np.abs(Ja)[:, :, None] * Mb[:, None, :], axis=0)
    g = np.sum(Ja * r[:, None], axis=0)
    Mg = np.sum(Ma * np.abs(r)[:, None] + np.abs(Ja) * Mr[:, None], axis=0)
    return H, MH, g, Mg, np.sum(cost), np.sum(Mcost)


def unary_blocks(poses, per_kf, q_lb, t_lb, lidar_const, huber_delta, jac_kind=0, unit_score=False, fn=None):
    """Per-keyframe 6x6 H, g, cost of the unary (fn=None) or edge factor.  per_kf[k]: dict(cp, nsd, weight) (unary) or
    dict(cp, pa, pb, s) (edge fn given), or None.  Returns float64 arrays H (W,6,6), g (W,6), cost (W,) and their shadows."""
    W = len(poses)
    out = dict(H=np.zeros((W, 6, 6)), MH=np.zeros((W, 6, 6)), g=np.zeros((W, 6)), Mg=np.zeros((W, 6)), cost=np.zeros(W), Mcost=np.zeros(W))
    # runs of keyframes are evaluated in one vectorised pass (the poses gathered per residual, about 2^17 residuals at a time;
    # a larger keyframe alone) and reduced per keyframe slice
    groups, cur, size = [], [], 0
    for k in range(W):
        m = per_kf[k] if k < len(per_kf) else None
        if m is None or len(m["cp"]) == 0:
            continue
        cur.append(k); size += len(m["cp"])
        if size >= 1 << 17:
            groups.append(cur); cur, size = [], 0
    if cur:
        groups.append(cur)
    r6 = slice(0, 6)
    for ks in groups:
        kf = np.concatenate([np.full(len(per_kf[k]["cp"]), k) for k in ks])
        P = np.asarray(poses, np.float64)[kf]
        cat = {key: np.concatenate([per_kf[k][key] for k in ks]) for key in per_kf[ks[0]]}
        if fn is None:
            R = unary_residuals(P, cat["cp"], cat["nsd"], cat["weight"], q_lb, t_lb, lidar_const, huber_delta, jac_kind, unit_score)
        else:
            R = edge_residuals(P, cat["cp"], cat["pa"], cat["pb"], cat["s"], q_lb, t_lb, huber_delta)
        bounds = np.flatnonzero(np.diff(kf)) + 1
        starts = np.concatenate([[0], bounds]); ends = np.concatenate([bounds, [len(kf)]])
        for s0, s1 in zip(starts, ends):
            k = kf[s0]; sl = slice(s0, s1)
            H, MH, g, Mg, c, Mc = _blocks(R["J"][sl], R["MJ"][sl], R["r"][sl], R["Mr"][sl], R["cost"][sl], R["Mcost"][sl], r6, r6)
            out["H"][k], out["MH"][k], out["g"][k], out["Mg"][k], out["cost"][k], out["Mcost"][k] = H, MH, g, Mg, c, Mc
    return out


def binary_blocks(poses, pairs, batch_score, huber_delta=0.0):
    """pairs: list of (cur, oth, dict(cp, nc, weight)) in declaration order.  Returns Hdiag (K,6,6), g (K,6), Hoff (P,6,6),
    cost (total) and shadows; the device's diagonal block of a keyframe sums its incident pairs in pair order."""
    K = len(poses); P = len(pairs)
    out = dict(Hdiag=np.zeros((K, 6, 6), LD), MHdiag=np.zeros((K, 6, 6), LD), g=np.zeros((K, 6), LD), Mg=np.zeros((K, 6), LD),
               Hoff=np.zeros((P, 6, 6)), MHoff=np.zeros((P, 6, 6)), cost=LD(0), Mcost=LD(0))
    poses = np.asarray(poses, np.float64)
    c6, o6 = slice(0, 6), slice(6, 12)
    for p, (cur, oth, m) in enumerate(pairs):
        if m is None or len(m["cp"]) == 0:
            continue
        R = binary_residuals(poses[cur], poses[oth], m["cp"], m["nc"], m["weight"], batch_score, huber_delta)
        J, MJ, r, Mr = R["J"], R["MJ"], R["r"], R["Mr"]
        for kfi, sl in ((cur, c6), (oth, o6)):
            H, MH, g, Mg, _, _ = _blocks(J, MJ, r, Mr, R["cost"], R["Mcost"], sl, sl)
            out["Hdiag"][kfi] += H; out["MHdiag"][kfi] += MH; out["g"][kfi] += g; out["Mg"][kfi] += Mg
        H, MH, _, _, c, Mc = _blocks(J, MJ, r, Mr, R["cost"], R["Mcost"], c6, o6)
        out["Hoff"][p], out["MHoff"][p] = H, MH
        out["cost"] += c; out["Mcost"] += Mc
    for key in ("Hdiag", "MHdiag", "g", "Mg"):
        out[key] = out[key].astype(np.float64)
    out["cost"], out["Mcost"] = float(out["cost"]), float(out["Mcost"])
    return out


def excess(dev, ref, M):
    """max over entries of |dev - ref| / (2^-53 M): the observed error in units of the bound's scale (<= KAPPA passes)."""
    dev = np.asarray(dev, np.float64); ref = np.asarray(ref, np.float64); M = np.asarray(M, np.float64)
    err = np.abs(dev - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(err == 0, 0.0, err / (U * M))
    return float(np.max(q)) if q.size else 0.0


def assert_within(dev, ref, M, what=""):
    dev = np.asarray(dev, np.float64); ref = np.asarray(ref, np.float64)
    assert np.all(np.isfinite(dev)), f"{what}: non-finite device values"
    e = excess(dev, ref, M)
    assert e <= KAPPA, f"{what}: |device - reference| reaches {e:.3g} x 2^-53 M (bound {KAPPA})"
    return e


# ---------------------------------------------------------------------------------------------------------------------------
# fixtures shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------------------
def rot_poly(q):
    """3x3 matrix of Eigen's polynomial q * v (float64)."""
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def make_poses(W, rng, offset=0.0, qnorm=1.0, w_zero=False, spread=20.0):
    """W body poses (t, q): translations `offset` metres from the origin (a scalar or per-keyframe array, along a random
    direction each) plus +-spread, quaternions of norm `qnorm` (scalar or per keyframe), w = 0 (180 degree turns) if asked."""
    off = np.broadcast_to(np.asarray(offset, np.float64), (W,))
    dirs = rng.normal(size=(W, 3)); dirs /= np.linalg.norm(dirs, axis=1)[:, None]
    t = dirs * off[:, None] + rng.uniform(-spread, spread, (W, 3))
    q = rng.normal(size=(W, 4))
    if w_zero:
        q[:, 0] = 0.0
    q /= np.linalg.norm(q, axis=1)[:, None]
    q *= np.broadcast_to(np.asarray(qnorm, np.float64), (W,))[:, None]
    return np.concatenate([t, q], axis=1)


def make_unary(rng, pose, n, q_lb, t_lb, noise=0.08, zero_weight_frac=0.0, exact_zero=0):
    """n plane correspondences of one keyframe: lidar-frame points near planes in the world, (n, d = -n.c) as float32, weights
    in [0.3, 1] (a fraction of them 0); the first `exact_zero` correspondences have an exactly zero residual."""
    t, q = pose[:3], pose[3:]
    pw = t + rng.uniform(-30, 30, (n, 3))
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    # body point from world: solve the functor's polynomial rotations (non-unit quaternions included)
    pbody = np.linalg.solve(rot_poly(q), (pw - t).T).T
    qi = np.array([q_lb[0], -q_lb[1], -q_lb[2], -q_lb[3]]) / np.dot(q_lb, q_lb)
    cp = (np.linalg.solve(rot_poly(qi), pbody.T).T + t_lb).astype(np.float32)
    c = pw + nrm * rng.normal(0, noise, (n, 1))
    nsd = np.concatenate([nrm, -np.sum(nrm * c, axis=1, keepdims=True)], axis=1).astype(np.float32)
    w = rng.uniform(0.3, 1.0, n).astype(np.float32)
    if zero_weight_frac:
        w[rng.random(n) < zero_weight_frac] = 0.0
    if exact_zero:
        nsd[:exact_zero] = 0.0        # n = 0, d = 0: r and J are exactly zero at any pose
    return dict(cp=cp, nsd=nsd, weight=w)


def make_edges(rng, pose, n, q_lb, t_lb, noise=0.08):
    t, q = pose[:3], pose[3:]
    a = t + rng.uniform(-20, 20, (n, 3)); d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1)[:, None]
    b = a + d * rng.uniform(0.2, 1.0, (n, 1))
    pw = a + d * rng.uniform(-1, 2, (n, 1)) + rng.normal(0, noise, (n, 3))
    pbody = np.linalg.solve(rot_poly(q), (pw - t).T).T
    qi = np.array([q_lb[0], -q_lb[1], -q_lb[2], -q_lb[3]]) / np.dot(q_lb, q_lb)
    cp = (np.linalg.solve(rot_poly(qi), pbody.T).T + t_lb).astype(np.float32)
    s = rng.uniform(1.0, 8.0, n).astype(np.float32).astype(np.float64)       # the score rides in a float32 lane on the device
    return dict(cp=cp, pa=a.astype(np.float32), pb=b.astype(np.float32), s=s)


def make_pair(rng, pose_c, pose_o, n, noise=0.08):
    """n binary correspondences of pair (cur, oth): cp in cur's body frame, normal and centroid in oth's (float64)."""
    tc, qc, to, qo = pose_c[:3], pose_c[3:], pose_o[:3], pose_o[3:]
    pw = tc + rng.uniform(-30, 30, (n, 3))
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    cw = pw + nrm * rng.normal(0, noise, (n, 1)) + np.cross(nrm, rng.normal(size=(n, 3))) * 0.3
    cp = np.linalg.solve(rot_poly(qc), (pw - tc).T).T.astype(np.float32)
    Ro = rot_poly(qo)
    nl = np.linalg.solve(Ro, nrm.T).T
    cl = np.linalg.solve(Ro, (cw - to).T).T
    w = rng.uniform(0.3, 1.0, n).astype(np.float32)
    return dict(cp=cp, nc=np.concatenate([nl, cl], axis=1), weight=w)


Q_LB_NONUNIT = np.array([0.9, 0.1, -0.3, 0.25]) * 1.3
T_LB = np.array([0.05, -0.02, 0.28])
