"""The extended-precision evaluation reference (tests/eval_reference.py) checked on the CPU: its dual-number derivatives against
50-digit central differences of the same functors, and the oracle (Jets, mode 0, and the closed forms, mode 1) against it
within the a-priori bound, on the fixtures the GPU edge-case tests use."""
import mpmath as mp
import numpy as np
import pytest

from tests import eval_reference as er

Q_LB, T_LB = er.Q_LB_NONUNIT, er.T_LB
LIDAR_CONST, BATCH_SCORE = 7.5, 2.5


# ---------------------------------------------------------------------------------------------------------------------------
# 50-digit functors and Ceres' exact quaternion plus (exp map)
# ---------------------------------------------------------------------------------------------------------------------------
def _mpq_mul(a, b):
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]]


def _mp_cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _mp_rot(q, v):
    uv = _mp_cross(q[1:], v); uv = [2 * c for c in uv]
    uuv = _mp_cross(q[1:], uv)
    return [v[i] + q[0] * uv[i] + uuv[i] for i in range(3)]


def _mp_inv(q):
    n2 = sum(c * c for c in q)
    return [q[0] / n2, -q[1] / n2, -q[2] / n2, -q[3] / n2]


def _mp_plus(pose, lane, h, jac_kind, first=0):
    """pose perturbed along derivative lane `lane` (0..5 relative to `first`) by h."""
    t = [mp.mpf(float(x)) for x in pose[:3]]; q = [mp.mpf(float(x)) for x in pose[3:]]
    j = lane - first
    if j < 3:
        t[j] += h
    elif jac_kind == 0:
        e = [mp.cos(h), mp.mpf(0), mp.mpf(0), mp.mpf(0)]; e[j - 2] = mp.sin(h)
        q = _mpq_mul(e, q)
    else:
        q[j - 2] += h
    return t, q


def _mp_unary(t, q, cp, nsd, s):
    qi = _mp_inv([mp.mpf(float(x)) for x in Q_LB])
    d = [mp.mpf(float(cp[i])) - mp.mpf(float(T_LB[i])) for i in range(3)]
    pw = _mp_rot(q, _mp_rot(qi, d))
    return s * (sum(mp.mpf(float(nsd[i])) * (pw[i] + t[i]) for i in range(3)) + mp.mpf(float(nsd[3])))


def _mp_edge(t, q, cp, a, b, s):
    qi = _mp_inv([mp.mpf(float(x)) for x in Q_LB])
    d = [mp.mpf(float(cp[i])) - mp.mpf(float(T_LB[i])) for i in range(3)]
    lp = _mp_rot(q, _mp_rot(qi, d)); lp = [lp[i] + t[i] for i in range(3)]
    A = [mp.mpf(float(x)) for x in a]; B = [mp.mpf(float(x)) for x in b]
    e = _mp_cross([lp[i] - A[i] for i in range(3)], [lp[i] - B[i] for i in range(3)])
    return s * mp.sqrt(sum(c * c for c in e)) / mp.sqrt(sum((A[i] - B[i]) ** 2 for i in range(3)))


def _mp_binary(tc, qc, to, qo, cp, nc, s):
    pw = _mp_rot(qc, [mp.mpf(float(x)) for x in cp]); pw = [pw[i] + tc[i] for i in range(3)]
    N = _mp_rot(qo, [mp.mpf(float(x)) for x in nc[:3]])
    cw = _mp_rot(qo, [mp.mpf(float(x)) for x in nc[3:]]); cw = [cw[i] + to[i] for i in range(3)]
    return s * sum(N[i] * (pw[i] - cw[i]) for i in range(3))


def _central(f, h=mp.mpf("1e-20")):
    return (f(h) - f(-h)) / (2 * h)


POSE_CASES = [dict(offset=0.0), dict(offset=20000.0), dict(qnorm=2.0), dict(qnorm=0.5, w_zero=True)]


@pytest.mark.parametrize("jac_kind", [0, 1])
@pytest.mark.parametrize("case", range(len(POSE_CASES)))
def test_unary_duals_match_50_digit_differences(jac_kind, case):
    rng = np.random.default_rng(10 + case)
    pose = er.make_poses(1, rng, **POSE_CASES[case])[0]
    m = er.make_unary(rng, pose, 24, Q_LB, T_LB)
    R = er.unary_residuals(pose, m["cp"], m["nsd"], m["weight"], Q_LB, T_LB, LIDAR_CONST, 0.0, jac_kind=jac_kind)
    with mp.workdps(50):
        for i in range(len(m["cp"])):
            s = mp.mpf(LIDAR_CONST) * mp.mpf(float(m["weight"][i]))
            r_mp = _mp_unary(*_mp_plus(pose, 0, 0, jac_kind), m["cp"][i], m["nsd"][i], s)
            assert abs(float(R["r"][i] - np.longdouble(float(r_mp)))) <= 1e-18 * float(R["Mr"][i]) + 1e-300
            for lane in range(6):
                d = _central(lambda h: _mp_unary(*_mp_plus(pose, lane, h, jac_kind), m["cp"][i], m["nsd"][i], s))
                assert abs(float(R["J"][i, lane]) - float(d)) <= 1e-16 * float(R["MJ"][i, lane])


@pytest.mark.parametrize("case", range(len(POSE_CASES)))
def test_edge_duals_match_50_digit_differences(case):
    rng = np.random.default_rng(20 + case)
    pose = er.make_poses(1, rng, **POSE_CASES[case])[0]
    m = er.make_edges(rng, pose, 24, Q_LB, T_LB)
    R = er.edge_residuals(pose, m["cp"], m["pa"], m["pb"], m["s"], Q_LB, T_LB, 0.0)
    with mp.workdps(50):
        for i in range(len(m["cp"])):
            s = mp.mpf(float(m["s"][i]))
            for lane in range(6):
                d = _central(lambda h: _mp_edge(*_mp_plus(pose, lane, h, 0), m["cp"][i], m["pa"][i], m["pb"][i], s))
                assert abs(float(R["J"][i, lane]) - float(d)) <= 1e-16 * float(R["MJ"][i, lane])


@pytest.mark.parametrize("case", range(len(POSE_CASES)))
def test_binary_duals_match_50_digit_differences(case):
    rng = np.random.default_rng(30 + case)
    P = er.make_poses(2, rng, **POSE_CASES[case])
    m = er.make_pair(rng, P[0], P[1], 24)
    R = er.binary_residuals(P[0], P[1], m["cp"], m["nc"], m["weight"], BATCH_SCORE)
    with mp.workdps(50):
        for i in range(len(m["cp"])):
            s = mp.mpf(BATCH_SCORE) * mp.mpf(float(m["weight"][i]))
            for lane in range(12):
                def f(h):
                    tc, qc = _mp_plus(P[0], lane if lane < 6 else 0, h if lane < 6 else 0, 0)
                    to, qo = _mp_plus(P[1], lane if lane >= 6 else 6, h if lane >= 6 else 0, 0, first=6)
                    return _mp_binary(tc, qc, to, qo, m["cp"][i], m["nc"][i], s)
                assert abs(float(R["J"][i, lane]) - float(_central(f))) <= 1e-16 * float(R["MJ"][i, lane])


# ---------------------------------------------------------------------------------------------------------------------------
# the oracle against the reference, within the bound
# ---------------------------------------------------------------------------------------------------------------------------
FIXTURES = {
    "near": dict(offset=0.0), "3km": dict(offset=3000.0), "20km": dict(offset=20000.0),
    "q_nonunit": dict(qnorm=[0.5, 2.0, 1.0]), "w_zero": dict(w_zero=True),
}


def _unit(fx):
    return "qnorm" not in fx


@pytest.mark.parametrize("huber", [1.0, 0.0])
@pytest.mark.parametrize("name", list(FIXTURES))
def test_oracle_unary_within_bound(oracle, name, huber):
    rng = np.random.default_rng(sum(map(ord, name)))
    W = 3
    poses = er.make_poses(W, rng, **FIXTURES[name])
    per = [er.make_unary(rng, poses[k], 700, Q_LB, T_LB) for k in range(W)]
    kf = np.repeat(np.arange(W, dtype=np.int32), 700)
    cp = np.concatenate([m["cp"] for m in per]); nsd = np.concatenate([m["nsd"] for m in per])
    score = LIDAR_CONST * np.concatenate([m["weight"] for m in per]).astype(np.float64)
    for jk in (0, 1):
        R = er.unary_blocks(poses, per, Q_LB, T_LB, LIDAR_CONST, huber, jac_kind=jk)
        for mode in (0, 1):
            o = oracle.eval_unary(poses, Q_LB, T_LB, kf, cp, nsd, score, huber_delta=huber, mode=mode, jac_kind=jk)
            for k in range(W):
                b = slice(6 * k, 6 * k + 6)
                er.assert_within(o["H"][b, b], R["H"][k], R["MH"][k], f"H mode {mode}")
                er.assert_within(o["g"][b], R["g"][k], R["Mg"][k], f"g mode {mode}")
                er.assert_within(o["cost"][kf == k].sum(), R["cost"][k], R["Mcost"][k], f"cost mode {mode}")
            if name == "near":
                # the bound is tight enough that a dropped residual fails it by orders of magnitude
                assert np.all(er.KAPPA * er.U * R["MH"].max(axis=(1, 2)) < 1e-9 * np.abs(R["H"]).max(axis=(1, 2)))
                o2 = oracle.eval_unary(poses, Q_LB, T_LB, kf[1:], cp[1:], nsd[1:], score[1:], huber_delta=huber, mode=mode, jac_kind=jk)
                assert er.excess(o2["H"][:6, :6], R["H"][0], R["MH"][0]) > 1e3 * er.KAPPA


@pytest.mark.parametrize("name", list(FIXTURES))
def test_oracle_edge_within_bound(oracle, name):
    rng = np.random.default_rng(100 + sum(map(ord, name)))
    W = 3
    poses = er.make_poses(W, rng, **FIXTURES[name])
    per = [er.make_edges(rng, poses[k], 500, Q_LB, T_LB) for k in range(W)]
    kf = np.repeat(np.arange(W, dtype=np.int32), 500)
    cat = {key: np.concatenate([m[key] for m in per]) for key in ("cp", "pa", "pb", "s")}
    R = er.unary_blocks(poses, per, Q_LB, T_LB, 0.0, 1.0, fn="edge")
    # the closed form (mode 1) writes the rotation columns as 2 R(q)p_b x gv, which is Ceres' tangent only for |q| = 1
    for mode in ((0, 1) if _unit(FIXTURES[name]) else (0,)):
        o = oracle.eval_edge(poses, Q_LB, T_LB, kf, cat["cp"], cat["pa"], cat["pb"], cat["s"], huber_delta=1.0, mode=mode)
        for k in range(W):
            b = slice(6 * k, 6 * k + 6)
            er.assert_within(o["H"][b, b], R["H"][k], R["MH"][k], f"edge H mode {mode}")
            er.assert_within(o["g"][b], R["g"][k], R["Mg"][k], f"edge g mode {mode}")
            er.assert_within(o["cost"][kf == k].sum(), R["cost"][k], R["Mcost"][k], f"edge cost mode {mode}")


@pytest.mark.parametrize("name", list(FIXTURES))
def test_oracle_binary_within_bound(oracle, name):
    rng = np.random.default_rng(200 + sum(map(ord, name)))
    K = 3
    poses = er.make_poses(K, rng, **FIXTURES[name])
    layout = [(0, 1), (1, 0), (2, 0)]
    pairs = [(c, o, er.make_pair(rng, poses[c], poses[o], 400)) for c, o in layout]
    R = er.binary_blocks(poses, pairs, BATCH_SCORE)
    kc = np.repeat([c for c, _ in layout], 400).astype(np.int32); ko = np.repeat([o for _, o in layout], 400).astype(np.int32)
    cp = np.concatenate([m["cp"] for _, _, m in pairs]); nc = np.concatenate([m["nc"] for _, _, m in pairs])
    score = BATCH_SCORE * np.concatenate([m["weight"] for _, _, m in pairs]).astype(np.float64)
    for mode in ((0, 1) if _unit(FIXTURES[name]) else (0,)):
        o = oracle.eval_binary(poses, kc, ko, cp, nc, score, huber_delta=0.0, mode=mode)
        for k in range(K):
            b = slice(6 * k, 6 * k + 6)
            er.assert_within(o["H"][b, b], R["Hdiag"][k], R["MHdiag"][k], f"binary Hdiag mode {mode}")
            er.assert_within(o["g"][b], R["g"][k], R["Mg"][k], f"binary g mode {mode}")
        # the oracle's dense (0, 1) block holds pair (0, 1) and the transpose of pair (1, 0)
        er.assert_within(o["H"][0:6, 6:12], R["Hoff"][0] + R["Hoff"][1].T, R["MHoff"][0] + R["MHoff"][1].T, f"binary Hoff mode {mode}")
        er.assert_within(o["H"][12:18, 0:6], R["Hoff"][2], R["MHoff"][2], f"binary Hoff mode {mode}")
        er.assert_within(o["cost_total"], R["cost"], R["Mcost"], f"binary cost mode {mode}")


def test_plan_items_mirror():
    """The GPU tests recompute capi.cu's plan_items to assert which item shapes they exercise."""
    from tests.test_gpu_eval_edges import ITEM_COUNTS, plan_items
    item, plan = plan_items(ITEM_COUNTS, 264)
    assert item == 2048
    assert [len(p) for p in plan][-6:] == [7, 8, 9, 16, 17, 9] and plan[-1][-1] == 1
    assert all(sum(p) == n for p, n in zip(plan, ITEM_COUNTS))
    item, plan = plan_items([600000], 264)
    assert item == 2304 and len(plan[0]) == 261 and plan[0][-1] == 600000 - 260 * 2304
