"""The batch refinement's pose factors on the CPU: the extended-precision reference (tests/pose_factor_reference.py) against
50-digit central differences of both functors, the generator's factor lists (synth.attitude_factors, synth.relative_pose_factors)
against a literal transliteration of the Estimator's loops, and the Python mirror of glio_pose_factor."""
import mpmath as mp
import numpy as np
import pytest

from glio_b200 import dist as gdist
from glio_b200 import synth
from tests import eval_reference as er
from tests import pose_factor_reference as pr

POSE_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("kind", "<i4"), ("active", "<i4"), ("dq", "<f8", (4,)), ("dp", "<f8", (3,))])


def _records(i, j, kind, dq, dp):
    f = np.zeros(len(i), POSE_DTYPE)
    f["i"], f["j"], f["kind"], f["active"], f["dq"], f["dp"] = i, j, kind, 1, dq, dp
    return f


# ---------------------------------------------------------------------------------------------------------------------------
# 50-digit functors, Ceres' exact quaternion plus
# ---------------------------------------------------------------------------------------------------------------------------
def _mq(a, b):
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]]


def _minv(q):
    n2 = sum(c * c for c in q)
    return [q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2]


def _mrot(q, v):
    cr = lambda a, b: [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    uv = [2 * c for c in cr(q[1:], v)]
    uuv = cr(q[1:], uv)
    return [v[k] + q[0] * uv[k] + uuv[k] for k in range(3)]


def _mp_factor(ti, qi, tj, qj, kind, dq, dp):
    E = _mq(_mq(_minv([mp.mpf(float(x)) for x in dq]), _minv(qi)), qj)
    if kind == 1:
        return [10000 * E[1 + c] for c in range(3)] + [mp.mpf(0)] * 3
    Bv = _mrot(_minv(qi), [tj[c] - ti[c] for c in range(3)])
    return [10 * (2 * E[1 + c]) for c in range(3)] + [20 * (Bv[c] - mp.mpf(float(dp[c]))) for c in range(3)]


def _mp_plus(pose, lane, h):
    t = [mp.mpf(float(x)) for x in pose[:3]]; q = [mp.mpf(float(x)) for x in pose[3:]]
    if lane < 3:
        t[lane] += h
    else:
        e = [mp.cos(h), mp.mpf(0), mp.mpf(0), mp.mpf(0)]; e[lane - 2] = mp.sin(h)
        q = _mq(e, q)
    return t, q


CASES = [dict(offset=0.0), dict(offset=3000.0), dict(offset=20000.0), dict(qnorm=2.0), dict(qnorm=0.5, w_zero=True), dict(w_zero=True)]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_duals_match_50_digit_differences(case):
    rng = np.random.default_rng(40 + case)
    P = er.make_poses(4, rng, **CASES[case])
    i = np.array([0, 1, 2, 3, 0, 3], np.int32); j = np.array([1, 0, 3, 2, 2, 1], np.int32)
    kind = np.array([0, 1, 1, 0, 1, 0], np.int32)
    dq = rng.normal(size=(6, 4)); dq /= np.linalg.norm(dq, axis=1)[:, None]
    f = _records(i, j, kind, dq, rng.normal(0, 2, (6, 3)))
    R = pr.factor_residuals(P, f)
    with mp.workdps(50):
        for n in range(len(f)):
            a, b = min(i[n], j[n]), max(i[n], j[n])
            def r_at(lane, h):
                ta, qa = _mp_plus(P[a], lane if lane < 6 else 0, h if lane < 6 else 0)
                tb, qb = _mp_plus(P[b], lane - 6 if lane >= 6 else 0, h if lane >= 6 else 0)
                (ti, qi), (tj, qj) = ((ta, qa), (tb, qb)) if i[n] < j[n] else ((tb, qb), (ta, qa))
                return _mp_factor(ti, qi, tj, qj, kind[n], f["dq"][n], f["dp"][n])
            r0 = r_at(0, 0)
            for row in range(6):
                assert abs(float(R["r"][n, row] - np.longdouble(mp.nstr(r0[row], 30)))) <= 1e-18 * float(R["Mr"][n, row]) + 1e-300
            h = mp.mpf("1e-20")
            for lane in range(12):
                rp, rm = r_at(lane, h), r_at(lane, -h)
                for row in range(6):
                    d = (rp[row] - rm[row]) / (2 * h)
                    assert abs(float(R["J"][n, row, lane]) - float(d)) <= 1e-16 * float(R["MJ"][n, row, lane]) + 1e-300


# ---------------------------------------------------------------------------------------------------------------------------
# the Estimator's loops, transliterated (Estimator.cpp:2831-2891 and 2897-2954)
# ---------------------------------------------------------------------------------------------------------------------------
def _estimator_lists(kf, search_range, start_idx, cur_batch_size):
    att, rel = [], []
    for i in range(start_idx, cur_batch_size):
        qi = kf[i, 3:].copy()
        if qi[0] < 0:                                     # unifyQuaternion
            qi = -qi
        pi = kf[i, :3]
        p_tmp = pi
        factor_count = 0
        j = i
        while j >= start_idx:                             # backward attitude constraint
            if factor_count == search_range:
                factor_count = 0
                break
            if j != i:
                pj = kf[j, :3]
                p_range = np.linalg.norm(p_tmp - pj)
                if p_range > int(5 / search_range):       # C++ integer division
                    p_tmp = pj
                    att.append((i, j, synth.quat_mul(synth.quat_conj(qi) / np.dot(qi, qi), kf[j, 3:])))
                    factor_count += 1
            j -= 1
        j = i
        while j < cur_batch_size:                         # forward attitude constraint
            if factor_count == search_range:
                factor_count = 0
                break
            if j != i:
                pj = kf[j, :3]
                p_range = np.linalg.norm(p_tmp - pj)
                if p_range > int(5 / search_range):
                    p_tmp = pj
                    att.append((i, j, synth.quat_mul(synth.quat_conj(qi) / np.dot(qi, qi), kf[j, 3:])))
                    factor_count += 1
            j += 1
    def rel_factor(a, b):
        qa = kf[a, 3:]
        qinv = synth.quat_conj(qa) / np.dot(qa, qa)
        return (a, b, synth.quat_mul(qinv, kf[b, 3:]), synth.quat_to_R(qinv) @ (kf[b, :3] - kf[a, :3]))
    idx = start_idx + search_range
    while idx < cur_batch_size:
        for ms_i in range(1, search_range):
            rel.append(rel_factor(idx - ms_i, idx))
        idx += 1
    idx = start_idx
    while idx < cur_batch_size - search_range:
        for ms_i in range(1, search_range):
            rel.append(rel_factor(idx, idx + ms_i))
        idx += 1
    return att, rel


def _kf_with_stops(K, rng):
    """keyframe poses with runs of repeated positions (the vehicle standing still), so the attitude walks skip keyframes"""
    kf = synth.perturb(synth.trajectory(K, rng), rng, 0.01, 0.05)
    for s in range(3, K, 9):
        kf[s:s + 3, :3] = kf[s, :3]
    kf[::5, 3:] *= -1.0                                   # w < 0: unifyQuaternion applies to q_i
    return kf


@pytest.mark.parametrize("K,search_range,start_idx", [(40, 6, 0), (40, 6, 7), (23, 3, 0), (30, 5, 2), (12, 1, 0), (5, 6, 0),
                                                      (13, 6, 0), (2, 6, 0), (9, 4, 4)])
def test_generator_lists_equal_the_estimator_loops(K, search_range, start_idx):
    kf = _kf_with_stops(K, np.random.default_rng(K * 7 + search_range))
    att, rel = _estimator_lists(kf, search_range, start_idx, K)
    ai, aj, adq = synth.attitude_factors(kf, search_range, start_idx)
    ri, rj, rdq, rdp = synth.relative_pose_factors(kf, search_range, start_idx)
    assert [(a, b) for a, b, _ in att] == list(zip(ai.tolist(), aj.tolist()))
    assert [(a, b) for a, b, _, _ in rel] == list(zip(ri.tolist(), rj.tolist()))
    if att:
        assert np.array_equal(np.array([d for _, _, d in att]), adq)
    if rel:
        assert np.array_equal(np.array([d for _, _, d, _ in rel]), rdq) and np.array_equal(np.array([d for _, _, _, d in rel]), rdp)
    assert all(a < b for a, b in zip(ri, rj))


def test_generator_quirks_show_up():
    # threshold 5 / search_range: 0 at search_range 6 (every moved keyframe counts), 1 at 5 (skips keyframes closer than 1 m)
    kf = _kf_with_stops(60, np.random.default_rng(3))
    a6 = synth.attitude_factors(kf, 6); a5 = synth.attitude_factors(kf, 5)
    assert np.any(a6[0] > a6[1]) and np.any(a6[0] < a6[1])                  # backward and forward walks
    gaps = np.abs(a5[0] - a5[1])
    assert gaps.max() > 5                                                    # 1 m threshold with 1 m spacing skips keyframes
    # factor_count carries over near the start: keyframe 2 walks back 2 steps, so its forward walk stops after 4
    i, j, _ = synth.attitude_factors(synth.perturb(synth.trajectory(30, np.random.default_rng(1)), np.random.default_rng(2)), 6)
    assert np.sum((i == 2) & (j > 2)) == 4 and np.sum((i == 2) & (j < 2)) == 2
    # interior pairs twice, always i < j
    ri, rj, _, _ = synth.relative_pose_factors(kf, 6)
    pairs = list(zip(ri.tolist(), rj.tolist()))
    assert pairs.count((20, 23)) == 2 and pairs.count((0, 1)) == 1


def test_level0_problem_has_the_sample_runs_size():
    P = synth.pose_graph_problem(K=3457)
    n = len(P["i"])
    assert 70000 < n < 80000
    assert np.all(P["kind"][:np.sum(P["kind"] == 1)] == 1)                  # attitude factors first, as the Estimator adds them
    L1 = synth.pose_graph_problem(K=40, level=1)
    assert np.all(L1["kind"] == 1) and len(L1["pairs"][0]) > 0


def test_python_mirror_and_shard_mask():
    from glio_b200 import api
    assert api.POSE_FACTOR_DTYPE == POSE_DTYPE and api.POSE_FACTOR_DTYPE.itemsize == 72
    assert [api.POSE_FACTOR_DTYPE.fields[k][1] for k in ("i", "j", "kind", "active", "dq", "dp")] == [0, 4, 8, 12, 16, 48]
    f = api.pose_factor_records([0, 5, 9], [1, 3, 2], [0, 1, 1], np.tile([1.0, 0, 0, 0], (3, 1)))
    assert list(f["active"]) == [1, 1, 1] and np.all(f["dp"] == 0)
    i = np.array([0, 5, 9, 4, 3]); j = np.array([1, 3, 2, 6, 9])
    m0 = gdist.pose_factor_active(i, j, 10, 2, 0); m1 = gdist.pose_factor_active(i, j, 10, 2, 1)
    assert list(m0) == [1] * 5 and list(m1) == [0] * 5                      # lower keyframes 0, 3, 2, 4, 3: all on rank 0 of [0, 5)
    m1 = gdist.pose_factor_active(i + 3, j + 3, 10, 2, 1)
    assert list(m1) == [0, 1, 1, 1, 1]
