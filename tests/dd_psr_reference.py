"""Extended-precision reference of the batch refinement's double-differenced pseudorange factors (K2g, glio_eval_dd_psr_factors),
independent of the device code.  Helper module for the tests (not collected).

dd_psr_factor_20's Evaluate (dd_psr_factor.hpp:25-171) is restated row by row in numpy.longdouble, with the constant yaw and
anchor blocks folded into R = R_ecef_local and anchor:

* ``P = R (ratio t_i + (1 - ratio) t_j) + anchor``; rows k = 0 .. n_sat-2 are the satellites s != master in index order;
* ``e_k = (|su_s - P| - |sr_s - st|) - (|su_m - P| - |sr_m - st|) - ((pu_s - pr_s) - (pu_m - pr_m))``;
* ``w_k = 0.05 if |e_k| > threshold else 1``, ``r_k = w_k e_k``;
* ``J_i row k = w_k ratio (u_m - u_s)^T R``, ``J_j row k = w_k (1 - ratio) (u_m - u_s)^T R``, ``u = normalized(su - P)``
  (Eigen 3.3: the vector itself when its squared norm is 0);
* with a weight matrix, ``r = W r``, ``J = W J``; ``cost = 0.5 |r|^2``.

The Jacobian columns are (t_a, t_b) of the factor's pair (a, b) = (min(i, j), max(i, j)).  Magnitude shadows: a row's residual is
a difference of ranges of up to ~2.7e7 m, so its shadow is the sum of the magnitudes it is formed from (four ranges, four
pseudoranges and |P| for P's own rounding); a Jacobian entry's shadow is the sum of |u| |R| terms times (1 + (|su| + |P|) / range),
the relative error a rounded P and su carry into a unit vector; W multiplies both by |W|.  The block shadows follow as in
tests/pose_factor_reference.py, and the bound is eval_reference's KAPPA = 2^9 times 2^-53 times the shadow.
"""
import numpy as np

from tests import eval_reference as ev

LD = ev.LD


def _ld(x):
    return np.asarray(x, np.float64).astype(LD)


def factor_rows(poses, F, sats, R, anchor, W=None):
    """One glio_dd_psr_factor record F: r (nr,), J (nr, 6) over (t_i, t_j), their shadows, the raw residuals e and the
    weights w."""
    R = _ld(R).reshape(3, 3); anchor = _ld(anchor).reshape(3)
    n, m = int(F["n_sat"]), int(F["master"])
    ra = LD(float(F["ratio"])); rb = LD(1) - ra
    ti, tj = _ld(poses[int(F["i"]), :3]), _ld(poses[int(F["j"]), :3])
    P = R @ (ra * ti + rb * tj) + anchor
    st = _ld(F["station"])
    S = sats[int(F["sat_offset"]):int(F["sat_offset"]) + n]
    su, sr = _ld(S["sat_user"]), _ld(S["sat_ref"])
    pu, pr = _ld(S["psr_user"]), _ld(S["psr_ref"])
    du = su - P; dr = sr - st
    nu = np.sqrt(np.sum(du * du, axis=1)); nr_ = np.sqrt(np.sum(dr * dr, axis=1))
    u = np.where((nu > 0)[:, None], du / np.where(nu > 0, nu, 1)[:, None], du)
    rows = [s for s in range(n) if s != m]
    e = np.array([(nu[s] - nr_[s]) - (nu[m] - nr_[m]) - ((pu[s] - pr[s]) - (pu[m] - pr[m])) for s in rows], LD)
    thr = LD(float(F["threshold"]))
    w = np.where(np.abs(e) > thr, LD(0.05), LD(1))
    r = w * e
    nP = np.sqrt(np.sum(P * P))
    Mr = w * np.array([nu[s] + nr_[s] + nu[m] + nr_[m] + abs(pu[s]) + abs(pr[s]) + abs(pu[m]) + abs(pr[m]) + 2 * nP for s in rows], LD)
    J = np.zeros((len(rows), 6), LD); MJ = np.zeros((len(rows), 6), LD)
    nsu = np.sqrt(np.sum(su * su, axis=1))
    for k, s in enumerate(rows):
        v = (u[m] - u[s]) @ R
        Mv = (np.abs(u[m]) + np.abs(u[s])) @ np.abs(R)
        amp = 1 + (nsu[s] + nP) / max(nu[s], LD(1)) + (nsu[m] + nP) / max(nu[m], LD(1))
        J[k, :3], J[k, 3:] = w[k] * ra * v, w[k] * rb * v
        MJ[k, :3], MJ[k, 3:] = w[k] * abs(ra) * Mv * amp, w[k] * abs(rb) * Mv * amp
    if W is not None and int(F["w_offset"]) >= 0:
        nr = n - 1
        Wf = _ld(W[int(F["w_offset"]):int(F["w_offset"]) + nr * nr]).reshape(nr, nr)
        r, Mr = Wf @ r, np.abs(Wf) @ Mr
        J, MJ = Wf @ J, np.abs(Wf) @ MJ
    return dict(r=r, Mr=Mr, J=J, MJ=MJ, e=e, w=w)


def pair_table(f):
    """The distinct pairs (a, b), a < b, in order of first appearance, and each factor's pair index."""
    index, pairs, fp = {}, [], np.zeros(len(f), np.int64)
    for n, (i, j) in enumerate(zip(f["i"], f["j"])):
        key = (int(min(i, j)), int(max(i, j)))
        if key not in index:
            index[key] = len(pairs); pairs.append(key)
        fp[n] = index[key]
    return pairs, fp


def dd_blocks(poses, f, sats, R, anchor, W=None):
    """glio_eval_dd_psr_factors' outputs for the active factors of f: Hdiag (K,6,6), g (K,6), Hoff (P,6,6) in pair-table order,
    cost, their shadows, and gate_margin: the smallest | |e_k| - threshold | over all rows (the gate is decided on the same side
    as the device when it is far above the residual's error bound)."""
    K = len(poses)
    pairs, fp = pair_table(f)
    out = dict(Hdiag=np.zeros((K, 6, 6), LD), MHdiag=np.zeros((K, 6, 6), LD), g=np.zeros((K, 6), LD), Mg=np.zeros((K, 6), LD),
               Hoff=np.zeros((len(pairs), 6, 6), LD), MHoff=np.zeros((len(pairs), 6, 6), LD), cost=LD(0), Mcost=LD(0), pairs=pairs,
               gate_margin=np.inf)
    for n, F in enumerate(f):
        if not F["active"]:
            continue
        rw = factor_rows(poses, F, sats, R, anchor, W)
        out["gate_margin"] = min(out["gate_margin"], float(np.min(np.abs(np.abs(rw["e"]) - LD(float(F["threshold"]))))))
        J, MJ, r, Mr = rw["J"], rw["MJ"], rw["r"], rw["Mr"]
        lo = int(F["i"]) < int(F["j"])
        Jab = J if lo else np.concatenate([J[:, 3:], J[:, :3]], axis=1)
        Mab = MJ if lo else np.concatenate([MJ[:, 3:], MJ[:, :3]], axis=1)
        H = Jab.T @ Jab; MH = Mab.T @ np.abs(Jab) + np.abs(Jab).T @ Mab
        g = Jab.T @ r; Mg = Mab.T @ np.abs(r) + np.abs(Jab).T @ Mr
        a, b = pairs[fp[n]]
        out["Hdiag"][a, :3, :3] += H[:3, :3]; out["MHdiag"][a, :3, :3] += MH[:3, :3]
        out["Hdiag"][b, :3, :3] += H[3:, 3:]; out["MHdiag"][b, :3, :3] += MH[3:, 3:]
        out["g"][a, :3] += g[:3]; out["Mg"][a, :3] += Mg[:3]
        out["g"][b, :3] += g[3:]; out["Mg"][b, :3] += Mg[3:]
        out["Hoff"][fp[n], :3, :3] += H[:3, 3:]; out["MHoff"][fp[n], :3, :3] += MH[:3, 3:]
        out["cost"] += LD(0.5) * np.sum(r * r); out["Mcost"] += np.sum(np.abs(r) * Mr)
    for key in ("Hdiag", "MHdiag", "g", "Mg", "Hoff", "MHoff"):
        out[key] = out[key].astype(np.float64)
    out["cost"], out["Mcost"] = float(out["cost"]), float(out["Mcost"])
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# fixtures shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------------------
def frame(yaw=0.3):
    """(R_ecef_local, anchor, station): an anchor in Hong Kong, the local frame `yaw` from ENU, a station 3 km away."""
    from glio_b200 import synth
    anchor = synth.geo_to_ecef(22.3, 114.18, 5.0)
    station = anchor + synth.ecef_local_rotation(anchor, 0.0) @ np.array([2400.0, -1800.0, 25.0])
    return synth.ecef_local_rotation(anchor, yaw), anchor, station


def random_sats(rng, n, P, station, anchor, noise=2.0, outlier_frac=0.15):
    """n satellites above the anchor's horizon on GNSS orbit radii, station positions a few metres off, pseudoranges from the
    ECEF position P with receiver and satellite clocks, noise and outliers of 20 .. 60 m (so the 10 / 8 / 6 m gates act)."""
    from glio_b200 import api, synth
    R_enu = synth.ecef_local_rotation(anchor, 0.0)
    az, el = rng.uniform(0, 2 * np.pi, n), rng.uniform(np.deg2rad(10), np.deg2rad(88), n)
    d = np.stack([np.sin(az) * np.cos(el), np.cos(az) * np.cos(el), np.sin(el)], axis=1) @ R_enu.T
    radius = rng.choice([25_510e3, 26_560e3, 27_900e3, 29_600e3, 42_164e3], n)
    bd = d @ anchor
    su = anchor + (-bd + np.sqrt(bd * bd - (anchor @ anchor - radius * radius)))[:, None] * d
    sr = su + rng.uniform(-3, 3, (n, 3))
    clk_s = rng.uniform(-3e5, 3e5, n)
    pu = np.linalg.norm(su - P, axis=1) + rng.uniform(-3e5, 3e5) - clk_s + rng.normal(0, noise, n)
    pu += np.where(rng.random(n) < outlier_frac, rng.uniform(20, 60, n), 0.0)
    pr = np.linalg.norm(sr - station, axis=1) + rng.uniform(-3e5, 3e5) - clk_s + rng.normal(0, 0.3, n)
    return api.dd_psr_sat_records(su, sr, pu, pr)


def random_list(rng, poses_true, ij, n_sat, master=None, ratio=None, thresholds=(1e9, 10.0, 8.0, 6.0), with_w=False, yaw=0.3):
    """A DD list over the keyframe pairs ij (n, 2), satellites from poses_true's interpolated positions: returns
    (f, sats, W, R, anchor).  master: per factor or random; ratio: per factor or uniform in [0, 1]; with_w: a random
    well-conditioned weight per factor (half of them identity)."""
    from glio_b200 import api
    R, anchor, station = frame(yaw)
    n = len(ij)
    n_sat = np.broadcast_to(np.asarray(n_sat), (n,)).astype(np.int32)
    master = np.array([rng.integers(0, k) for k in n_sat]) if master is None else np.broadcast_to(np.asarray(master), (n,))
    ratio = rng.uniform(0, 1, n) if ratio is None else np.broadcast_to(np.asarray(ratio, np.float64), (n,))
    sats, W, w_off = [], [], []
    for k in range(n):
        i, j = ij[k]
        P = R @ (ratio[k] * poses_true[i, :3] + (1 - ratio[k]) * poses_true[j, :3]) + anchor
        sats.append(random_sats(rng, int(n_sat[k]), P, station, anchor))
        if with_w and rng.random() < 0.5:
            m = int(n_sat[k]) - 1
            w_off.append(sum(len(x) for x in W)); W.append((np.eye(m) + rng.normal(0, 0.1, (m, m))).ravel())
        else:
            w_off.append(-1)
    f = api.dd_psr_factor_records(ij[:, 0], ij[:, 1], n_sat, master, ratio, rng.choice(thresholds, n), station, w_offset=w_off)
    Wa = np.concatenate(W) if W else None
    return f, np.concatenate(sats) if n else np.zeros(0, api.DD_PSR_SAT_DTYPE), Wa, R, anchor
