"""Edge blocks in the window solve and marginalisation (glio_window_use_edges, glio_eval_edge_kind).

The reference never instantiates LidarEdgeFactor, so the oracle has no edge term; these tests check the wiring against the same
problem composed outside the library: the plane blocks of the device plus the edge blocks handed in as host factors (solve), or
added into the marginalisation's normal equations and marginalised with glio_marginalize (prior).  The ambient edge Jacobian is
checked against the longdouble dual-number reference."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth

pytestmark = pytest.mark.gpu
W = 4


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _setup(api, P, E, ctx=None, edges=True):
    c = ctx or api.Context(0)
    c.set_map(P["map_xyz"]); c.window_set_scans(P["scans"]); c.window_associate(P["poses_init"])
    if edges:
        c.set_edge_map(E["map_xyz"])
        for k in range(W):
            c.window_set_edge_scan(k, E["scans"][k])
        assert c.window_associate_edges(P["poses_init"]).min() > 100
    return c


@pytest.fixture(scope="module")
def problem():
    return synth.window_problem(W=W, Q=3000, M=40000, seed=31), synth.window_edge_problem(W=W, Q=1500, M=40000, seed=32)


def test_eval_edge_kind(api, problem):
    from tests import edge_ambient_reference as ea
    P, E = problem
    c = _setup(api, P, E)
    try:
        a, b = c.eval_edge(P["poses_init"]), c.eval_edge_kind(P["poses_init"], 0)
        assert all(np.array_equal(a[k], b[k]) for k in ("H", "g", "cost"))
        m = c.eval_edge_kind(P["poses_init"], 1)
        assert not np.array_equal(m["H"], a["H"]) and np.array_equal(m["cost"], a["cost"])
        for k in range(W):
            e = c.get_edges(k)
            H, g, cost = ea.blocks(P["poses_init"][k], e["cp"], e["pa"], e["pb"], e["s"], P["q_lb"], P["t_lb"], c.params.huber_delta)
            assert np.max(np.abs(m["H"][k] - np.asarray(H, float))) <= 1e-11 * float(np.max(np.abs(H)))
            assert np.max(np.abs(m["g"][k] - np.asarray(g, float))) <= 1e-10 * float(np.max(np.abs(g)))
            assert abs(m["cost"][k] - float(cost)) <= 1e-11 * float(cost)
        with pytest.raises(api.GlioError, match="error -3"):
            c.eval_edge_kind(P["poses_init"], 2)
    finally:
        c.close()


def test_use_edges_off_ignores_edges(api, problem):
    """off (the default, and after on -> off) a context holding edges solves and marginalises like one that never had any; on with
    no edge in the window changes nothing either"""
    P, E = problem
    a, b, z = _setup(api, P, E, edges=False), _setup(api, P, E), _setup(api, P, E, edges=False)
    try:
        b.set_edges(0, np.zeros((3, 3), np.float32) + 1, np.zeros((3, 3), np.float32), np.ones((3, 3), np.float32), np.ones(3))
        b.window_associate_edges(P["poses_init"])
        b.window_use_edges(True); b.window_use_edges(False)
        z.window_use_edges(True)
        sb = np.zeros((W, 9))
        ra = a.window_solve(P["poses_init"])
        pa = a.window_marginalize(ra["poses"], sb).arrays()
        for c in (b, z):
            rc = c.window_solve(P["poses_init"])
            assert np.array_equal(ra["poses"], rc["poses"]) and np.array_equal(ra["steps"], rc["steps"])
            pc = c.window_marginalize(rc["poses"], sb).arrays()
            assert all(np.array_equal(pa[k], pc[k]) for k in ("lin_jac", "lin_res", "x0_pose", "A_info", "b_info"))
    finally:
        for c in (a, b, z):
            c.close()


def _composed_callback(api, edge_ctx, hf, nt):
    """host factors = hf (may be None) + the edge blocks edge_ctx evaluates (tangent columns), in the solver's dense layout"""
    def cb(user, Wc, poses, speed_bias, want_jac, H, g, cost):
        pz = np.ctypeslib.as_array(poses, (Wc * 7,)).reshape(Wc, 7).copy()
        sb = np.ctypeslib.as_array(speed_bias, (Wc * 9,)).reshape(Wc, 9).copy() if speed_bias else None
        n = Wc * nt
        ct = 0.0
        Hd = np.zeros((n, n)); gd = np.zeros(n)
        if hf is not None:
            Hh, gh, ch = hf.evaluate(pz, sb, bool(want_jac)); Hd += Hh; gd += gh; ct += ch
        e = edge_ctx.eval_edge(pz, want_jac=bool(want_jac))
        ct += float(e["cost"].sum())
        if want_jac:
            for k in range(Wc):
                Hd[nt * k:nt * k + 6, nt * k:nt * k + 6] += e["H"][k]; gd[nt * k:nt * k + 6] += e["g"][k]
            np.ctypeslib.as_array(H, (n * n,))[:] = Hd.ravel()
            np.ctypeslib.as_array(g, (n,))[:] += gd
        cost[0] = cost[0] + ct
        return 0
    return api.HOST_FACTORS_FN(cb)


def _host_factors(api, P, sb, prior=None):
    hf = api.HostFactorSet()
    T = P["poses_init"]
    sw = np.full(15, 10.0)
    hf.add_prior(0, T[0, :3], T[0, 3:], sb[0], sw)
    for i in range(W - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        hf.add_between(i, i + 1, dp, dq, np.zeros(3), 0.1, sw * 0.5)
    if prior is not None:
        hf.set_marg_prior(prior)
    return hf


@pytest.mark.parametrize("variant", ["poses", "speed_bias", "speed_bias_prior"])
def test_solve_with_edges_matches_composed_problem(api, problem, variant):
    P, E = problem
    a = _setup(api, P, E)                               # edges inside the solve
    b = _setup(api, P, E, edges=False)                  # plane blocks only; edges come in as host factors
    e = _setup(api, P, E)                               # evaluates those edge blocks
    try:
        a.window_use_edges(True)
        sb = np.zeros((W, 9)) if variant != "poses" else None
        prior = None
        if variant == "speed_bias_prior":
            prior = b.window_marginalize(P["poses_init"], np.zeros((W, 9)))
        hf = _host_factors(api, P, np.zeros((W, 9)), prior) if sb is not None else None
        nt = 15 if sb is not None else 6
        ra = a.window_solve(P["poses_init"], sb, host_factors=hf)
        rb = b.window_solve(P["poses_init"], sb, host_factors=_composed_callback(api, e, hf, nt))
        plane_only = b.window_solve(P["poses_init"], sb, host_factors=hf)
        ia, ib = ra["iterations"], rb["iterations"]
        assert len(ia) == len(ib) and ra["summary"].num_iterations > 1
        assert [x["step_is_successful"] for x in ia] == [x["step_is_successful"] for x in ib]
        assert len(ra["steps"]) == len(rb["steps"]) > 0
        for sa, sb_ in zip(ra["steps"], rb["steps"]):
            for k in range(W):
                assert np.max(np.abs(sa[nt * k:nt * k + 3] - sb_[nt * k:nt * k + 3])) <= 1e-6
                assert 2 * np.linalg.norm(sa[nt * k + 3:nt * k + 6] - sb_[nt * k + 3:nt * k + 6]) <= 1e-8
        assert abs(ra["summary"].initial_cost - rb["summary"].initial_cost) <= 1e-9 * rb["summary"].initial_cost
        assert ra["summary"].initial_cost > plane_only["summary"].initial_cost          # the edges are in the problem
    finally:
        for c in (a, b, e):
            c.close()


def test_marginalize_with_edges(api, problem):
    """the prior of a marginalisation with edges equals glio_marginalize of the normal equations with the edge blocks (ambient
    columns) added; the asynchronous pass is bit-identical to the synchronous one"""
    P, E = problem
    a = _setup(api, P, E)
    try:
        a.window_use_edges(True)
        poses = P["poses_init"]; sb = np.zeros((W, 9))
        hf = _host_factors(api, P, sb)
        pr = a.window_marginalize(poses, sb, hf).arrays()
        pj = a.window_marginalize_async(poses, sb, hf).wait().arrays()
        assert all(np.array_equal(pr[k], pj[k]) for k in ("lin_jac", "lin_res", "x0_pose", "A_info", "b_info"))
        A, b = hf.marg_evaluate(poses, sb)
        pl, ed = a.eval_unary(poses, jac_kind=1), a.eval_edge_kind(poses, 1)
        base = [0, 15] + [30 + 6 * (k - 2) for k in range(2, W)]                  # marginalisation ordering (csrc/marg.h)
        for k in range(W):
            A[base[k]:base[k] + 6, base[k]:base[k] + 6] += pl["H"][k] + ed["H"][k]
            b[base[k]:base[k] + 6] += pl["g"][k] + ed["g"][k]
        N = 6 * W + 18; n = N - 15
        J = np.zeros((n, n)); r = np.zeros(n)
        L = api.lib()
        assert L.glio_marginalize(api._ptr(np.ascontiguousarray(A)), api._ptr(b), C.c_int(N), C.c_int(15), C.c_double(1e-8), api._ptr(J), api._ptr(r)) == 0
        JtJ, Jtr = J.T @ J, J.T @ r
        dJtJ, dJtr = pr["lin_jac"].T @ pr["lin_jac"], pr["lin_jac"].T @ pr["lin_res"]
        assert np.max(np.abs(dJtJ - JtJ)) <= 1e-9 * np.max(np.abs(JtJ))
        assert np.max(np.abs(dJtr - Jtr)) <= 1e-8 * np.max(np.abs(Jtr))
        a.window_use_edges(False)
        off = a.window_marginalize(poses, sb, hf).arrays()
        assert not np.allclose(off["lin_jac"].T @ off["lin_jac"], dJtJ, rtol=1e-6, atol=0)   # the edges were in the prior
    finally:
        a.close()
