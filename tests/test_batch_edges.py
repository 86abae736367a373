"""CPU checks of the batch edge path's references and Python mirror: the pair-mode association reference (tests/
batch_edge_reference.py) against numpy's eigen-decomposition and an independent local line fit; the binary point-to-edge dual-number
reference (tests/binary_edge_reference.py) against 50-digit central differences and the closed-form Jacobians; the new C symbols and
the argument lists the ctypes mirror passes; synth.batch_edge_problem's per-frame streams."""
import ctypes as C
import os
import re

import mpmath
import numpy as np
import pytest

from glio_b200 import synth
from tests import batch_edge_reference as ber
from tests import binary_edge_reference as bref
from tests import edge_reference as er
from tests import eval_reference as ev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["glio_batch_set_edge_frame", "glio_batch_associate_edges_pairs", "glio_batch_get_edges", "glio_batch_set_pair_edges",
       "glio_eval_binary_edge", "glio_batch_use_edges"]


def _clusters(rng, n):
    """five-point neighbourhoods: lines with noise, planes, blobs, exact collinear and identical points (float32)"""
    out = []
    for i in range(n):
        kind = i % 5
        c = rng.uniform(-50, 50, 3)
        if kind == 0:
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            p = c + np.outer(rng.uniform(-0.5, 0.5, 5), d) + rng.normal(0, 0.01, (5, 3))
        elif kind == 1:
            p = c + rng.normal(0, 0.3, (5, 3)) * [1, 1, 0.01]
        elif kind == 2:
            p = c + rng.normal(0, 0.2, (5, 3))
        elif kind == 3:
            p = c + np.outer(np.arange(5) * 0.125, [1.0, 0.0, 0.0])
        else:
            p = np.tile(c, (5, 1))
        out.append(p.astype(np.float32))
    return out


def test_pair_reference_jacobi_and_gates_match_eigh():
    rng = np.random.default_rng(11)
    seen = set()
    for nb in _clusters(rng, 200):
        st, lam, pa, pb = er.line_fit(nb, np.float32(0.5))
        _, A = er.centroid_scatter(nb)
        w = np.linalg.eigvalsh(np.array(A))
        scale = max(abs(w).max(), 1e-300)
        assert np.allclose(lam, w, rtol=0, atol=1e-12 * scale)
        # the gate decides as lambda_2 > 3 lambda_1 on eigh's values, away from the boundary
        if abs(w[2] - 3.0 * w[1]) > 1e-9 * scale:
            assert (st == er.VALID) == (w[2] > 3.0 * w[1])
        seen.add(int(st))
    assert seen == {er.VALID, er.FAIL_LINE}
    assert er.line_fit(_clusters(rng, 1)[0], np.float32(1.0))[0] == er.FAIL_RADIUS      # gate: sqd[4] < max_sqdist is strict


def test_local_refit_matches_an_independent_numpy_fit():
    rng = np.random.default_rng(12)
    n = 0
    for nb in _clusters(rng, 100)[::5]:
        q = synth.quat_from_rotvec(rng.normal(0, 0.5, 3)); t = rng.uniform(-30, 30, 3)
        local = ((nb.astype(np.float64) - t) @ synth.quat_to_R(q)).astype(np.float32)     # the searched frame's stored points
        pa, pb, c, v = ber.local_line(local, 0.1)
        x = local.astype(np.float64)
        cn = x.mean(axis=0)
        w, V = np.linalg.eigh((x - cn).T @ (x - cn))
        vn = V[:, 2] * np.sign(V[np.argmax(np.abs(V[:, 2])), 2])
        assert np.allclose(c, cn, rtol=0, atol=1e-12 * (1 + np.abs(cn).max()))
        assert np.allclose(v, vn, atol=1e-9)
        assert np.allclose(pa, cn + 0.1 * vn, rtol=0, atol=4e-6 * (1 + np.abs(cn).max()))
        assert np.allclose(pb, cn - 0.1 * vn, rtol=0, atol=4e-6 * (1 + np.abs(cn).max()))
        n += 1
    assert n > 0


def _mp_residual(pc, po, cp, a, b, s, delta):
    """r at the poses moved by the 12 tangent coordinates delta (Ceres: t + dt, q <- exp(d) (x) q), in mpmath."""
    def quat_plus(q, d):
        nd = mpmath.sqrt(sum(x * x for x in d))
        if nd == 0:
            return q
        dq = [mpmath.cos(nd)] + [mpmath.sin(nd) / nd * x for x in d]
        w1, x1, y1, z1 = dq; w2, x2, y2, z2 = q
        return [w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2]

    def rot(q, v):
        w, u = q[0], q[1:]
        uv = [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]
        uv = [2 * x for x in uv]
        uuv = [u[1] * uv[2] - u[2] * uv[1], u[2] * uv[0] - u[0] * uv[2], u[0] * uv[1] - u[1] * uv[0]]
        return [v[i] + w * uv[i] + uuv[i] for i in range(3)]
    tc = [pc[i] + delta[i] for i in range(3)]; qc = quat_plus(pc[3:], delta[3:6])
    to = [po[i] + delta[6 + i] for i in range(3)]; qo = quat_plus(po[3:], delta[9:12])
    pw = [x + y for x, y in zip(rot(qc, cp), tc)]
    A = [x + y for x, y in zip(rot(qo, a), to)]; B = [x + y for x, y in zip(rot(qo, b), to)]
    u = [pw[i] - A[i] for i in range(3)]; v = [pw[i] - B[i] for i in range(3)]
    e = [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]
    return s * mpmath.sqrt(sum(x * x for x in e)) / mpmath.sqrt(sum((A[i] - B[i]) ** 2 for i in range(3)))


def test_dual_reference_matches_50_digit_central_differences():
    rng = np.random.default_rng(13)
    P = ev.make_poses(2, rng, offset=3000.0)
    m = bref.make_pair_edges(rng, P[0], P[1], 4)
    R = bref.binary_edge_residuals(P[0], P[1], m["cp"], m["pa"], m["pb"], m["s"])
    mpmath.mp.dps = 50
    h = mpmath.mpf("1e-20")
    for i in range(4):
        args = ([mpmath.mpf(float(x)) for x in P[0]], [mpmath.mpf(float(x)) for x in P[1]], [mpmath.mpf(float(x)) for x in m["cp"][i]],
                [mpmath.mpf(float(x)) for x in m["pa"][i]], [mpmath.mpf(float(x)) for x in m["pb"][i]], mpmath.mpf(float(m["s"][i])))
        r0 = _mp_residual(*args, [0] * 12)
        # the longdouble reference is within one double-precision unit of its own magnitude shadow: far inside the 2^9 bound
        assert abs(float(R["r"][i]) - float(r0)) <= ev.U * float(R["Mr"][i])
        for j in range(12):
            d = [0] * 12; d[j] = h
            dp = _mp_residual(*args, d); d[j] = -h; dm = _mp_residual(*args, d)
            fd = (dp - dm) / (2 * h)
            assert abs(mpmath.mpf(float(R["J"][i, j])) - fd) <= ev.U * float(R["MJ"][i, j]), (i, j)


def test_dual_jacobians_match_the_closed_form():
    rng = np.random.default_rng(14)
    P = ev.make_poses(2, rng, offset=20000.0)
    m = bref.make_pair_edges(rng, P[0], P[1], 64)
    R = bref.binary_edge_residuals(P[0], P[1], m["cp"], m["pa"], m["pb"], m["s"])
    tc, qc, to, qo = (np.array(P[0][:3], ev.LD), P[0][3:], np.array(P[1][:3], ev.LD), P[1][3:])
    Rc = ev.rot_poly(np.array(qc, ev.LD)); Ro = ev.rot_poly(np.array(qo, ev.LD))
    cp = m["cp"].astype(ev.LD); a = m["pa"].astype(ev.LD); b = m["pb"].astype(ev.LD); s = m["s"].astype(ev.LD)
    rcp = cp @ Rc.T
    pw = rcp + tc; A = a @ Ro.T + to; B = b @ Ro.T + to
    e = np.cross(pw - A, pw - B); de = A - B
    g = (s / np.linalg.norm(de, axis=1))[:, None] * np.cross(de, e / np.linalg.norm(e, axis=1)[:, None])
    Jc = np.concatenate([g, 2 * np.cross(rcp, g)], axis=1)
    Jo = np.concatenate([-g, 2 * np.cross(g, pw - to)], axis=1)
    J = np.asarray(R["J"], np.float64)
    scale = np.abs(J).max(axis=1, keepdims=True)
    assert np.max(np.abs(J[:, :6] - np.asarray(Jc, np.float64)) / scale) < 1e-10
    assert np.max(np.abs(J[:, 6:] - np.asarray(Jo, np.float64)) / scale) < 1e-10


def _header_params():
    src = open(os.path.join(ROOT, "include", "glio_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for name in NEW:
        m = re.search(r"\b" + name + r"\s*\(([^)]*)\)\s*;", src)
        assert m, name
        out[name] = [p.strip() for p in m.group(1).split(",")]
    return out


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return 0
        return f


def _ctype_ok(decl, arg):
    if decl.startswith("glio_ctx*"):
        return arg is None
    if "*" in decl:
        return arg is None or isinstance(arg, C.c_void_p) or type(arg).__name__ == "CArgObject"     # _ptr(array) or byref(struct)
    if decl.startswith("int64_t"):
        return isinstance(arg, C.c_int64)
    if decl.startswith("int "):
        return isinstance(arg, C.c_int)
    return False


def test_new_symbols_are_exported_and_the_mirror_passes_their_arguments():
    from glio_b200 import api
    lib = C.CDLL(os.path.join(ROOT, "glio_b200", "libglio_b200.so"))
    for n in NEW:
        assert hasattr(lib, n), n
    params = _header_params()
    ctx = object.__new__(api.Context)
    rec = _Recorder()
    ctx._lib = rec; ctx._h = None; ctx._chk = lambda rc: None
    xyz = np.zeros((7, 3), np.float32)
    ctx.batch_set_edge_frame(0, xyz)
    ctx.batch_set_edge_frame(1, np.zeros((0, 3), np.float32))
    opt = api.EdgeOptions()
    ctx.batch_associate_edges_pairs([0], [1], options=opt)
    ctx.batch_get_edges(0, 1)
    ctx.batch_set_pair_edges(0, 1, xyz, xyz, xyz, np.ones(7))
    ctx.eval_binary_edge(np.zeros((2, 7)))
    ctx.batch_use_edges(True)
    called = [c for c in rec.calls if c[0] in NEW]
    assert {c[0] for c in called} == set(NEW)
    for name, args in called:
        decl = params[name]
        assert len(args) == len(decl), (name, len(args), decl)
        for d, a in zip(decl, args):
            assert _ctype_ok(d, a), (name, d, a)
    # the empty corner scan goes out as Q = 0 with stride 3
    empty = [a for n, a in rec.calls if n == "glio_batch_set_edge_frame"][1]
    assert empty[3].value == 0 and empty[4].value == 3


def test_batch_edge_problem_streams_and_poses():
    full = synth.batch_edge_problem(K=6, Q=500, seed=5, search_range=2)
    part = synth.batch_edge_problem(K=6, Q=500, seed=5, search_range=2, frames=[1, 4])
    surf = synth.batch_problem(K=6, Q=10, seed=5, search_range=2, frames=[])
    assert np.array_equal(full["poses_init"], surf["poses_init"]) and np.array_equal(full["poses_true"], surf["poses_true"])
    for k in range(6):
        if k in (1, 4):
            assert np.array_equal(part["corner_scans"][k], full["corner_scans"][k])
        else:
            assert part["corner_scans"][k] is None
    s = full["corner_scans"][2]
    assert s.dtype == np.float32 and s.shape == (500, 3)
    # body frame of the true pose: back in the world the points lie within the sampled x range
    T = full["poses_true"][2]
    pw = s.astype(np.float64) @ synth.quat_to_R(T[3:]).T + T[:3]
    assert np.all(np.abs(pw[:, 0] - T[0]) <= 50.0 + 0.2)


@pytest.mark.parametrize("n_oth", [0, 4])
def test_pair_reference_small_searched_frame_fails_radius(oracle, n_oth):
    rng = np.random.default_rng(15)
    cur = rng.normal(size=(9, 3)).astype(np.float32)
    oth = rng.normal(size=(n_oth, 3)).astype(np.float32)
    pose = np.array([0.0, 0, 0, 1, 0, 0, 0])
    o = ber.associate_pair(oracle, cur, pose, oth, pose)
    assert o["n"] == 0 and np.all(o["status"] == ber.FAIL_RADIUS)
