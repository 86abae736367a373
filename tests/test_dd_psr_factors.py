"""CPU checks of the DD-pseudorange pieces: the longdouble reference (tests/dd_psr_reference.py) against 50-digit mpmath central
differences, synth.ecef_local_rotation against gnss_comm's closed form in mpmath, and synth.dd_psr_factors against a literal
transliteration of the Estimator's loops (Estimator.cpp:3086-3272 with getGlobalLowerUpperIdx and prepare*DDPsrData)."""
import numpy as np
import pytest

from glio_b200 import synth
from tests import dd_psr_reference as dr
from tests import eval_reference as er

mp = pytest.importorskip("mpmath")


# ---------------------------------------------------------------------------------------------------------------------------
# the reference against central differences
# ---------------------------------------------------------------------------------------------------------------------------
def _mp_residual(F, sats, R, anchor, W, ti, tj, gate_w):
    """r of the factor at translations ti, tj (mp vectors), with the weights gate_w (the gate is piecewise constant)."""
    ra = mp.mpf(float(F["ratio"])); rb = 1 - ra
    loc = [ra * ti[c] + rb * tj[c] for c in range(3)]
    P = [sum(mp.mpf(float(R[a, b])) * loc[b] for b in range(3)) + mp.mpf(float(anchor[a])) for a in range(3)]
    n, m, off = int(F["n_sat"]), int(F["master"]), int(F["sat_offset"])
    st = [mp.mpf(float(x)) for x in F["station"]]

    def rng_(a, b):
        return mp.sqrt(sum((mp.mpf(float(a[c])) - b[c]) ** 2 for c in range(3)))
    S = sats[off:off + n]
    um, rm = rng_(S[m]["sat_user"], P), rng_(S[m]["sat_ref"], st)
    r = []
    for s in range(n):
        if s == m:
            continue
        e = (rng_(S[s]["sat_user"], P) - rng_(S[s]["sat_ref"], st)) - (um - rm) \
            - ((mp.mpf(float(S[s]["psr_user"])) - mp.mpf(float(S[s]["psr_ref"]))) - (mp.mpf(float(S[m]["psr_user"])) - mp.mpf(float(S[m]["psr_ref"]))))
        r.append(mp.mpf(float(gate_w[len(r)])) * e)
    if W is not None and int(F["w_offset"]) >= 0:
        nr = n - 1
        Wf = np.asarray(W[int(F["w_offset"]):int(F["w_offset"]) + nr * nr]).reshape(nr, nr)
        r = [sum(mp.mpf(float(Wf[k, l])) * r[l] for l in range(nr)) for k in range(nr)]
    return r


@pytest.mark.parametrize("n_sat,master,ratio,with_w,offset", [(2, 0, 0.37, False, 0.0), (3, 2, 0.0, True, 0.0), (5, 2, 1.0, True, 3000.0),
                                                             (20, 0, 0.81, True, 3000.0), (20, 19, 0.5, False, 0.0), (12, 5, 0.2, True, 20.0)])
def test_reference_matches_central_differences(n_sat, master, ratio, with_w, offset):
    mp.mp.dps = 50
    rng = np.random.default_rng(n_sat * 7 + master)
    poses = er.make_poses(4, rng, offset=offset)
    for ij in ((0, 1), (3, 1)):                                              # i < j and i > j
        for thr in (1e9, 6.0):
            f, sats, W, R, anchor = dr.random_list(rng, poses, np.array([ij]), n_sat, master, ratio, thresholds=(thr,), with_w=with_w)
            if with_w and W is None:                                         # random_list gives half of the factors identity
                f, sats, W, R, anchor = dr.random_list(np.random.default_rng(1), poses, np.array([ij]), n_sat, master, ratio,
                                                       thresholds=(thr,), with_w=True)
            F = f[0]
            ref = dr.factor_rows(poses, F, sats, R, anchor, W)
            assert np.min(np.abs(np.abs(ref["e"]) - dr.LD(thr))) > 1e-3       # rows away from the gate
            if thr == 6.0:
                assert np.all(ref["w"][np.abs(ref["e"]) > 6.0] == dr.LD(0.05))
            ti = [mp.mpf(float(x)) for x in poses[ij[0], :3]]; tj = [mp.mpf(float(x)) for x in poses[ij[1], :3]]
            r0 = _mp_residual(F, sats, R, anchor, W, ti, tj, ref["w"])
            assert np.max(np.abs(np.array([float(x) for x in r0]) - ref["r"].astype(np.float64))) <= 2.0 ** -56 * float(np.max(ref["Mr"]))
            h = mp.mpf("1e-12")
            Jmp = np.zeros((n_sat - 1, 6))
            for col in range(6):
                which, c = (ti, col) if col < 3 else (tj, col - 3)
                plus = list(which); minus = list(which)
                plus[c] += h; minus[c] -= h
                rp = _mp_residual(F, sats, R, anchor, W, plus if col < 3 else ti, tj if col < 3 else plus, ref["w"])
                rm_ = _mp_residual(F, sats, R, anchor, W, minus if col < 3 else ti, tj if col < 3 else minus, ref["w"])
                Jmp[:, col] = [float((a - b) / (2 * h)) for a, b in zip(rp, rm_)]
            J = ref["J"].astype(np.float64)
            assert np.max(np.abs(J - Jmp)) <= 1e-15 * max(1.0, np.max(np.abs(Jmp)))


def test_zero_line_of_sight_follows_eigen():
    """normalized() of a zero vector is the zero vector: a satellite at P contributes a zero Jacobian row part"""
    rng = np.random.default_rng(3)
    poses = np.zeros((2, 7)); poses[:, 3] = 1.0
    f, sats, W, R, anchor = dr.random_list(rng, poses, np.array([(0, 1)]), 3, 0, 0.5, thresholds=(1e9,))
    sats["sat_user"][1] = anchor                                             # P = anchor at t = 0
    rw = dr.factor_rows(poses, f[0], sats, R, anchor)
    u_m = (sats["sat_user"][0] - anchor) / np.linalg.norm(sats["sat_user"][0] - anchor)
    assert np.allclose(rw["J"][0, :3].astype(np.float64), 0.5 * (u_m @ R), rtol=1e-15, atol=1e-16)


# ---------------------------------------------------------------------------------------------------------------------------
# ecef_local_rotation
# ---------------------------------------------------------------------------------------------------------------------------
def _mp_rotation(anchor, yaw):
    mp.mp.dps = 50
    x, y, z = (mp.mpf(float(v)) for v in anchor)
    a, e2 = mp.mpf(6378137), mp.mpf("6.69437999014e-3")
    a2 = a * a; b2 = a2 * (1 - e2); b = mp.sqrt(b2); ep2 = (a2 - b2) / b2
    p = mp.sqrt(x * x + y * y)
    s1, s2 = z * a, p * b
    h = mp.sqrt(s1 * s1 + s2 * s2)
    st, ct = s1 / h, s2 / h
    lat = mp.atan((z + ep2 * b * st ** 3) / (p - a * e2 * ct ** 3))
    lon = mp.atan2(y, x)
    sl, cl, so, co = mp.sin(lat), mp.cos(lat), mp.sin(lon), mp.cos(lon)
    Re = mp.matrix([[-so, -sl * co, cl * co], [co, -sl * so, cl * so], [0, cl, sl]])
    cy, sy = mp.cos(mp.mpf(yaw)), mp.sin(mp.mpf(yaw))
    return np.array((Re * mp.matrix([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])).tolist(), dtype=float)


@pytest.mark.parametrize("lat,lon,h,yaw", [(22.3, 114.18, 5.0, 0.3), (-33.9, 151.2, 40.0, -1.2), (64.1, -21.9, 10.0, 3.0), (0.5, -179.0, 0.0, 0.0)])
def test_ecef_local_rotation_matches_mpmath(lat, lon, h, yaw):
    anchor = synth.geo_to_ecef(lat, lon, h)
    R = synth.ecef_local_rotation(anchor, yaw)
    assert np.max(np.abs(R - _mp_rotation(anchor, yaw))) <= 1e-15
    assert np.max(np.abs(R @ R.T - np.eye(3))) <= 1e-15


# ---------------------------------------------------------------------------------------------------------------------------
# the generator against the Estimator's loops
# ---------------------------------------------------------------------------------------------------------------------------
def _prepare(gnss_data, ref_gnss_data, is_sys, psr_check):
    """prepare{GPS,BDS,GLO,GAL}DDPsrData (Estimator.cpp:1702-1837), literally"""
    ref_tmp, user_tmp = [], []
    for i in range(len(gnss_data)):
        prn = int(gnss_data[i]["prn"])
        for j in range(len(ref_gnss_data)):
            if prn == int(ref_gnss_data[j]["prn"]) and is_sys(prn) and (not psr_check or gnss_data[i]["psr"] > 1000):
                ref_tmp.append(ref_gnss_data[j]); user_tmp.append(gnss_data[i])
    mPrn, maxEle = -1, 0.0
    for m in range(len(user_tmp)):
        ele = float(user_tmp[m]["elevation"])
        if abs(ele) > maxEle:
            maxEle = ele
            mPrn = m
    return user_tmp, ref_tmp, mPrn


def _estimator_loops(epochs, keyframe_time, gl_tmpTrans, station, threshold, keyframe_idx0=1):
    """Estimator.cpp:3086-3272 with getGlobalLowerUpperIdx (:1635-1662), pose_info_keyframe_batch->points.size() = K"""
    K = len(keyframe_time)
    out = []
    P_add_idx = np.zeros(3)
    for i in range(len(epochs)):
        obs_local_ts, gnss_data, ref_gnss_data = epochs[i]
        lower_idx, upper_idx = -1, 10000000
        if obs_local_ts > keyframe_time[len(keyframe_time) - 1] or obs_local_ts < keyframe_time[0]:
            continue
        diff = 10000000
        for ii in range(keyframe_idx0, K):
            t = keyframe_time[ii - 1]; diffTmp = abs(t - obs_local_ts)
            if diffTmp < diff and t < obs_local_ts:
                lower_idx = ii; diff = diffTmp
        diff = 10000000
        for ii in range(keyframe_idx0, K):
            t = keyframe_time[ii - 1]; diffTmp = abs(t - obs_local_ts)
            if diffTmp < diff and t > obs_local_ts:
                upper_idx = ii; diff = diffTmp
        if (lower_idx < 0 or lower_idx >= K) or (upper_idx < 0 or upper_idx >= K):
            continue
        lower_ts, upper_ts = keyframe_time[lower_idx - 1], keyframe_time[upper_idx - 1]
        ts_ratio = (upper_ts - obs_local_ts) / (upper_ts - lower_ts)
        leftKey, rightKey = lower_idx - 1, upper_idx - 1
        Pj = np.array(gl_tmpTrans[rightKey])
        if np.linalg.norm(Pj - P_add_idx) < 1:
            continue
        P_add_idx = Pj
        for is_sys, psr_check in ((synth.prn_is_gps, True), (synth.prn_is_bds, True), (synth.prn_is_glo, False), (synth.prn_is_gal, False)):
            user, ref, mPrn = _prepare(gnss_data, ref_gnss_data, is_sys, psr_check)
            if len(user) > 2:
                out.append((leftKey, rightKey, ts_ratio, mPrn, user, ref))
    return out


def _mutate(epochs, kf_times, rng):
    """quirks the plain generator rarely meets: epochs exactly at keyframe times, PRN 84 (GPS and Galileo), negative elevations
    (the |ele| > maxEle test), a station PRN listed twice, zero pseudoranges on every system"""
    out = []
    for n, (t, u, r) in enumerate(epochs):
        u, r = u.copy(), r.copy()
        if n % 17 == 3:
            t = float(kf_times[np.argmin(np.abs(kf_times - t))])
        if n % 5 == 1 and len(u) > 3:
            u["prn"][0] = 84; r = np.concatenate([r, u[:1]])
        if n % 7 == 2 and len(u):
            u["elevation"][rng.integers(0, len(u))] *= -1
        if n % 11 == 4 and len(r):
            r = np.concatenate([r, r[:1]])
        if n % 13 == 5 and len(u):
            u["psr"][rng.integers(0, len(u))] = 0.0
        out.append((t, u, r))
    return out


@pytest.mark.parametrize("outer_pass", [0, 1, 3])
def test_generator_equals_estimator_loops(outer_pass):
    P = synth.dd_psr_problem(K=80, outer_pass=outer_pass, seed=synth.SEED0 + 40 + outer_pass)
    epochs = _mutate(P["epochs"], P["kf_times"], np.random.default_rng(outer_pass))
    thr = synth.DD_PSR_THRESHOLDS[outer_pass]
    trans = P["poses_init"][:, :3]
    cols, sats = synth.dd_psr_factors(epochs, P["kf_times"], trans, P["station"], thr)
    lit = _estimator_loops(epochs, P["kf_times"], trans, P["station"], thr)
    assert len(lit) == len(cols["i"]) > 50
    assert [x[0] for x in lit] == cols["i"].tolist() and [x[1] for x in lit] == cols["j"].tolist()
    assert [x[2] for x in lit] == cols["ratio"].tolist() and [x[3] for x in lit] == cols["master"].tolist()
    assert [len(x[4]) for x in lit] == cols["n_sat"].tolist()
    assert np.all(cols["threshold"] == thr) and np.all(cols["station"] == P["station"])
    su = np.concatenate([[s["sat_pos"] for s in x[4]] for x in lit]); sr = np.concatenate([[s["sat_pos"] for s in x[5]] for x in lit])
    pu = np.concatenate([[s["psr"] for s in x[4]] for x in lit]); pr = np.concatenate([[s["psr"] for s in x[5]] for x in lit])
    assert np.array_equal(su, sats["sat_user"]) and np.array_equal(sr, sats["sat_ref"])
    assert np.array_equal(pu, sats["psr_user"]) and np.array_equal(pr, sats["psr_ref"])
    # the kept epochs' right keyframes at least 1 m apart in turn; every factor brackets with adjacent candidates
    assert np.all((cols["ratio"] > 0) & (cols["ratio"] < 1)) and np.all(cols["i"] < cols["j"])


def test_generator_sample_run_counts():
    """the sample run's size: the factor count the DESIGN table quotes, and the 1 m rule keeping at most one epoch per keyframe"""
    P = synth.dd_psr_problem(K=3457)
    d = P["dd"]
    assert len(d["i"]) == 8848 and len(set(zip(d["i"].tolist(), d["j"].tolist()))) == 2212
    assert np.all(d["n_sat"] <= 20) and np.all(d["n_sat"] >= 3)
