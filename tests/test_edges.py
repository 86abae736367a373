"""The edge association's reference arithmetic (tests/edge_reference.py) on the CPU: the specified cyclic Jacobi against
numpy.linalg.eigh and an extended-precision residual, degenerate neighbourhoods, and the seeded corner generator."""
import numpy as np
import pytest

from glio_b200 import synth
from tests import edge_reference as er

# Bounds of the Jacobi against LAPACK (both backward stable): eigenvalues within 64 ulp of the largest one; the direction of the
# largest eigenvalue within 1e-9 rad when its gap is at least 1e-4 of it (sin of the angle ~ eps |C| / gap).
EIG_ULPS = 64
DIR_GAP = 1e-4


def _neighbourhoods(rng, n):
    """n sets of five float32 points: lines, planes, blobs, at scales from mm to m and offsets up to 20 km."""
    out = []
    for i in range(n):
        kind = i % 3
        scale = 10.0 ** rng.uniform(-3, 0)
        off = rng.choice([0.0, 3e3, 2e4]) * rng.standard_normal(3)
        d = rng.standard_normal(3); d /= np.linalg.norm(d)
        if kind == 0:
            p = np.outer(rng.uniform(-1, 1, 5), d) * scale + rng.normal(0, 0.05 * scale, (5, 3))
        elif kind == 1:
            e = np.cross(d, rng.standard_normal(3)); e /= np.linalg.norm(e)
            p = (np.outer(rng.uniform(-1, 1, 5), d) + np.outer(rng.uniform(-1, 1, 5), e)) * scale
        else:
            p = rng.normal(0, scale, (5, 3))
        out.append((p + off).astype(np.float32))
    return out


def test_jacobi_against_eigh_and_longdouble():
    rng = np.random.default_rng(synth.SEED0 + 40)
    n_gap = 0
    for nb in _neighbourhoods(rng, 3000):
        _, A = er.centroid_scatter(nb)
        lam, v, sweeps = er.jacobi_eig3(A)
        assert sweeps <= 10
        A = np.array(A)
        w, V = np.linalg.eigh(A)
        lmax = max(abs(w[2]), np.finfo(float).tiny)
        assert np.all(np.abs(np.array(lam) - w) <= EIG_ULPS * np.spacing(lmax)), (lam, w)
        assert lam[0] <= lam[1] <= lam[2]
        m = int(np.argmax(np.abs(v)))
        assert v[m] > 0 and np.all(np.abs(v[:m]) < abs(v[m]))                 # sign rule, lowest index on ties
        vl = np.array(v, np.longdouble); Al = np.array(A, np.longdouble)
        res = Al @ vl - np.longdouble(lam[2]) * vl                               # residual in extended precision
        assert float(np.sqrt(np.sum(res * res))) <= EIG_ULPS * np.spacing(lmax)
        assert abs(float(np.sqrt(np.sum(vl * vl))) - 1.0) <= 1e-14
        if w[2] - w[1] >= DIR_GAP * lmax:
            n_gap += 1
            assert abs(abs(float(np.dot(v, V[:, 2]))) - 1.0) <= 1e-12
    assert n_gap > 1000


def test_gate_decisions_match_eigh_outside_the_bound():
    rng = np.random.default_rng(synth.SEED0 + 41)
    flagged = agree = 0
    for nb in _neighbourhoods(rng, 3000):
        _, A = er.centroid_scatter(nb)
        lam, _, _ = er.jacobi_eig3(A)
        w = np.linalg.eigh(np.array(A))[0]
        for r in (1.5, 3.0, 10.0):
            ours = lam[2] > r * lam[1]
            theirs = w[2] > r * w[1]
            if abs(w[2] - r * w[1]) <= 4 * EIG_ULPS * np.spacing(max(abs(w[2]), np.finfo(float).tiny)) * (1 + r):
                flagged += 1                                                      # within the bound of min_ratio: may differ
                continue
            assert ours == theirs
            agree += 1
    assert agree > 8000


def test_degenerate_neighbourhoods():
    base = np.array([10.0, 20.0, 5.0])
    same = np.tile(base, (5, 1)).astype(np.float32)
    st, eig, _, _ = er.line_fit(same, np.float32(0.0))
    assert st == er.FAIL_LINE and np.all(eig == 0.0)                            # 0 > 3 * 0 is false
    line = (base + np.outer([0.0, 0.25, -0.25, 0.5, -0.5], [1.0, 0.0, 0.0])).astype(np.float32)
    st, eig, pa, pb = er.line_fit(line, np.float32(0.25))
    assert st == er.VALID and eig[1] == 0.0 and eig[2] == 0.625
    assert np.array_equal(pa, np.float32(base + [0.1, 0, 0])) and np.array_equal(pb, np.float32(base - [0.1, 0, 0]))
    square = (base + np.array([[0, 0, 0], [0.5, 0, 0], [-0.5, 0, 0], [0, 0.5, 0], [0, -0.5, 0]])).astype(np.float32)
    st, eig, _, _ = er.line_fit(square, np.float32(0.25))
    assert st == er.FAIL_LINE and eig[1] == eig[2] == 0.5                       # coplanar, isotropic in its plane
    # dyadic: C = diag(6, 2, 0) s^2 exactly, so lambda_2 = 3 lambda_1 and the strict gate rejects it
    dy = (base + 0.125 * np.array([[2, 0, 0], [-1, 1, 0], [-1, -1, 0], [0, 0, 0], [0, 0, 0]])).astype(np.float32)
    st, eig, _, _ = er.line_fit(dy, np.float32(0.0625))
    assert eig[2] == 3 * eig[1] and st == er.FAIL_LINE
    assert er.line_fit(dy, np.float32(0.0625), dict(min_ratio=2.999))[0] == er.VALID
    # the radius gate is strict too
    assert er.line_fit(line, np.float32(1.0))[0] == er.FAIL_RADIUS
    assert er.line_fit(line, np.float32(0.999))[0] == er.VALID


def test_theta_overflow_gives_no_rotation():
    # |a_qq - a_pp| / (2 a_pq) overflows: t = 0, the element is zeroed, the diagonal is kept
    lam, v, _ = er.jacobi_eig3([[0.0, 1e-310, 0.0], [1e-310, 1.0, 0.0], [0.0, 0.0, 0.5]])
    assert lam == [0.0, 0.5, 1.0] and v == [0.0, 1.0, 0.0]


def test_corner_generator_is_seeded_and_on_edges():
    a = synth.window_edge_problem(W=3, Q=500, M=4000, seed=3)
    b = synth.window_edge_problem(W=3, Q=500, M=4000, seed=3)
    assert np.array_equal(a["map_xyz"], b["map_xyz"]) and all(np.array_equal(x, y) for x, y in zip(a["scans"], b["scans"]))
    assert a["map_xyz"].dtype == np.float32 and a["map_xyz"].shape == (4000, 3) and a["scans"][0].shape == (500, 3)
    # corner points are near a line, not spread over a plane: most neighbourhoods pass the line gate
    m = a["map_xyz"]
    i = np.random.default_rng(0).choice(len(m), 200, replace=False)
    d = ((m[i][:, None, :] - m[None, :, :]) ** 2).sum(-1)
    nn = np.argsort(d, axis=1, kind="stable")[:, :5]
    ok = sum(er.line_fit(m[nn[j]], np.float32(0.0))[0] == er.VALID for j in range(len(i)))
    assert ok > 0.5 * len(i)


@pytest.mark.parametrize("opts", [dict(max_sqdist=0.5), dict(min_ratio=10.0), dict(half_length=1.0, score=2.5)])
def test_reference_association_on_the_oracle_knn(oracle, opts):
    """kd-tree and brute-force 5-NN give the same edge lists; the options act where they should."""
    P = synth.window_edge_problem(W=1, Q=800, M=20000, seed=9)
    t2, q2 = synth.lidar_pose_in_world(P["poses_init"][0, :3], P["poses_init"][0, 3:])
    a = er.associate_edges(oracle, P["map_xyz"], P["scans"][0], t2, q2, opts, tree=oracle.KdTree(P["map_xyz"]))
    b = er.associate_edges(oracle, P["map_xyz"], P["scans"][0], t2, q2, opts)
    for k in ("status", "eig", "cp", "pa", "pb", "s", "src"):
        assert np.array_equal(a[k], b[k])
    d = er.associate_edges(oracle, P["map_xyz"], P["scans"][0], t2, q2)
    assert a["n"] > 0
    if "half_length" in opts:
        assert np.all(a["s"] == 2.5) and np.array_equal(a["src"], d["src"])
        assert np.allclose(a["pa"] - a["pb"], 10.0 * (d["pa"] - d["pb"]), atol=5e-3)
    else:
        assert a["n"] < d["n"]


def test_ambient_edge_jacobian_against_central_differences():
    """the dual-number ambient edge Jacobian (tests/edge_ambient_reference.py) against central differences of the residual in
    q's x, y, z (the rotation polynomial, not renormalised), and its tangent lanes against tests/eval_reference.py"""
    from tests import edge_ambient_reference as ea
    from tests import eval_reference as ev
    rng = np.random.default_rng(synth.SEED0 + 42)
    q_lb, t_lb = np.array([1.0, 0, 0, 0]), np.array([0.0, 0.0, 0.28])
    pose = np.concatenate([[3.0, -1.0, 0.5], synth.quat_from_rpy(0.1, -0.2, 0.3)])
    cp = rng.uniform(-10, 10, (20, 3)).astype(np.float32)
    pa = rng.uniform(-10, 10, (20, 3)).astype(np.float32); pb = (pa + rng.normal(0, 0.2, (20, 3))).astype(np.float32)
    s = np.ones(20)
    R = ea.edge_residuals(pose, cp, pa, pb, s, q_lb, t_lb, 0.0)
    h = 1e-6
    for j in range(3):
        pp, pm = pose.copy(), pose.copy(); pp[4 + j] += h; pm[4 + j] -= h
        fd = (ea.edge_residuals(pp, cp, pa, pb, s, q_lb, t_lb, 0.0)["r"] - ea.edge_residuals(pm, cp, pa, pb, s, q_lb, t_lb, 0.0)["r"]) / (2 * h)
        assert np.allclose(np.asarray(R["J"][:, 3 + j], float), np.asarray(fd, float), rtol=1e-6, atol=1e-7)
    T = ea.edge_residuals(pose, cp, pa, pb, s, q_lb, t_lb, 0.5, jac_kind=0)
    E = ev.edge_residuals(pose, cp, pa, pb, s, q_lb, t_lb, 0.5)
    assert np.array_equal(T["J"], E["J"]) and np.array_equal(T["r"], E["r"])
