"""Scan-to-multiscan edges on the device: K1be (glio_batch_associate_edges_pairs) bit for bit against the pair-mode reference
(tests/batch_edge_reference.py), K2be (glio_eval_binary_edge) within the a-priori bound of the longdouble reference
(tests/binary_edge_reference.py), the batch solve with edges against the same problem with the edge blocks handed in as host
factors, and what the edge calls must leave alone."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import dist as gdist
from glio_b200 import synth
from tests import batch_edge_reference as ber
from tests import binary_edge_reference as bref
from tests import eval_reference as ev

pytestmark = pytest.mark.gpu
STATUSES = set()


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _load(ctx, corner, poses, surf=None):
    for k, s in corner.items():
        ctx.batch_set_frame(int(k), surf[k] if surf is not None else np.zeros((1, 3), np.float32), poses[k])
        ctx.batch_set_edge_frame(int(k), s)


def _host(a):
    if hasattr(a, "cpu"):
        return a.cpu().numpy()
    return a


def _check_pairs(ctx, oracle, corner, poses, cur, oth, ne, sample=None, opts=None):
    """compare the listed pairs (or a sample of their indices) with the reference; returns the reference statuses"""
    idx = range(len(cur)) if sample is None else sample
    sts = []
    for i in idx:
        c, o = int(cur[i]), int(oth[i])
        ref = ber.associate_pair(oracle, _host(corner[c]), poses[c], _host(corner[o]), poses[o], opts)
        e = ctx.batch_get_edges(c, o)
        assert e["n"] == ne[i] == ref["n"], (c, o, e["n"], ne[i], ref["n"])
        for key in ("cp", "pa", "pb", "s", "src"):
            assert np.array_equal(e[key], ref[key]), (c, o, key)
        sts.append(ref["status"])
    st = np.concatenate(sts) if sts else np.zeros(0, np.uint8)
    STATUSES.update(int(x) for x in np.unique(st))
    return st


@pytest.mark.parametrize("offset", [0.0, 3000.0, 20000.0])
def test_parity_k16(api, oracle, offset):
    K, sr = 16, 6
    E = synth.batch_edge_problem(K=K, Q=2000, seed=41, search_range=sr)
    poses = E["poses_init"].copy(); poses[:, :3] += offset
    cur, oth = gdist.batch_pairs(K, sr)
    ctx = api.Context(0)
    try:
        corner = {k: E["corner_scans"][k] for k in range(K)}
        _load(ctx, corner, poses)
        ne = ctx.batch_associate_edges_pairs(cur, oth)
        assert ne.sum() > 0
        sample = np.random.default_rng(1).choice(len(cur), 12, replace=False)
        st = _check_pairs(ctx, oracle, corner, poses, cur, oth, ne, sample)
        assert (st == ber.VALID).any() and (st == ber.FAIL_LINE).any() and (st == ber.FAIL_RADIUS).any()
    finally:
        ctx.close()


def test_parity_stride8_device_input_one_big_pair_and_reassociation(api, oracle):
    import torch
    E = synth.batch_edge_problem(K=3, Q=10000, seed=42, search_range=1)
    rng = np.random.default_rng(42)
    poses = E["poses_init"].copy()
    s8 = [np.concatenate([s, rng.standard_normal((len(s), 5)).astype(np.float32)], axis=1) for s in E["corner_scans"]]
    corner = {0: s8[0], 1: torch.from_numpy(s8[1]).cuda(), 2: E["corner_scans"][2]}
    ctx = api.Context(0)
    try:
        _load(ctx, corner, poses)
        cur, oth = np.array([0, 1, 2, 1]), np.array([1, 0, 1, 2])
        ne = ctx.batch_associate_edges_pairs(cur, oth)
        _check_pairs(ctx, oracle, corner, poses, cur, oth, ne)
        # a moved pose drops the searched frame's grid: re-association at the new poses matches the reference again
        poses[1, :3] += [0.3, -0.2, 0.1]
        ctx.batch_set_pose(1, poses[1])
        ne2 = ctx.batch_associate_edges_pairs(cur, oth)
        assert not np.array_equal(ne, ne2)
        _check_pairs(ctx, oracle, corner, poses, cur, oth, ne2)
        # a gate exactly at a query's 5th squared distance rejects it (strict comparison)
        ref = ber.associate_pair(oracle, s8[0], poses[0], s8[1], poses[1])
        i = int(np.nonzero(ref["status"] == ber.VALID)[0][0])
        gate = float(ref["sqd5"][i, 4])
        ne3 = ctx.batch_associate_edges_pairs([0], [1], max_sqdist=gate)
        r3 = _check_pairs(ctx, oracle, corner, poses, [0], [1], ne3, opts=dict(max_sqdist=gate))
        assert r3[i] == ber.FAIL_RADIUS
    finally:
        ctx.close()


def test_small_and_degenerate_corner_frames(api, oracle):
    rng = np.random.default_rng(43)
    ident = np.array([0.0, 0, 0, 1, 0, 0, 0])
    # searched frame: exactly collinear runs of five (pass the line gate), five identical points (fail it), spaced 10 m apart
    line = np.array([[x, 0.0, 0.0] for x in (0.0, 0.125, 0.25, 0.375, 0.5)], np.float32)
    same = np.tile(np.array([[10.0, 0.0, 0.0]], np.float32), (5, 1))
    line2 = line + np.float32([20.0, 3.0, 1.0])
    oth_pts = np.concatenate([line, same, line2])
    near = lambda c: (c + rng.normal(0, 0.05, (20, 3))).astype(np.float32)
    cur_pts = np.concatenate([near(np.array([0.25, 0, 0])), near(np.array([10.0, 0, 0])), near(np.array([20.25, 3, 1]))])
    frames = {0: cur_pts, 1: oth_pts, 2: np.zeros((0, 3), np.float32), 3: oth_pts[:4].copy(), 4: oth_pts[:5].copy(), 5: np.zeros((0, 3), np.float32)}
    poses = {k: ident.copy() for k in frames}
    poses[1] = np.array([0.01, -0.02, 0.0, 1, 0, 0, 0])
    ctx = api.Context(0)
    try:
        _load(ctx, frames, poses)
        cur = np.array([0, 0, 0, 0, 5]); oth = np.array([1, 2, 3, 4, 1])
        ne = ctx.batch_associate_edges_pairs(cur, oth)
        st = _check_pairs(ctx, oracle, frames, poses, cur, oth, ne)
        assert ne[1] == 0 and ne[2] == 0 and ne[4] == 0              # 0 and 4 points searched, an empty cur
        r1 = ber.associate_pair(oracle, cur_pts, poses[0], oth_pts, poses[1])
        assert (r1["status"][:20] == ber.VALID).all() and (r1["status"][20:40] == ber.FAIL_LINE).all()
        assert (st == ber.VALID).any() and (st == ber.FAIL_LINE).any() and (st == ber.FAIL_RADIUS).any()
    finally:
        ctx.close()


def test_cfg3_shape_sample(api, oracle):
    K, sr = 200, 6
    E = synth.batch_edge_problem(K=K, Q=10000, seed=44, search_range=sr)
    cur, oth = gdist.batch_pairs(K, sr)
    assert len(cur) == 2400
    ctx = api.Context(0)
    try:
        corner = {k: E["corner_scans"][k] for k in range(K)}
        _load(ctx, corner, E["poses_init"])
        ne = ctx.batch_associate_edges_pairs(cur, oth)
        sample = np.random.default_rng(44).choice(len(cur), 20, replace=False)
        _check_pairs(ctx, oracle, corner, E["poses_init"], cur, oth, ne, sample)
    finally:
        ctx.close()


def test_fixtures_cover_every_status():
    assert STATUSES >= {ber.VALID, ber.FAIL_RADIUS, ber.FAIL_LINE}


def test_argument_errors_change_nothing(api):
    E = synth.batch_edge_problem(K=4, Q=300, seed=45, search_range=1)
    ctx = api.Context(0)
    try:
        for k in range(3):
            ctx.batch_set_frame(k, E["corner_scans"][k], E["poses_init"][k])
        ctx.batch_set_edge_frame(0, E["corner_scans"][0]); ctx.batch_set_edge_frame(1, E["corner_scans"][1])
        with pytest.raises(api.GlioError, match="error -4"):
            ctx.batch_set_edge_frame(3, E["corner_scans"][3])               # frame never registered
        with pytest.raises(api.GlioError, match="error -3"):
            ctx.batch_associate_edges_pairs([0], [3])
        with pytest.raises(api.GlioError, match="error -3"):
            ctx.batch_associate_edges_pairs([1], [1])
        with pytest.raises(api.GlioError, match="error -3"):
            ctx.batch_associate_edges_pairs([0], [1], half_length=0.0)
        with pytest.raises(api.GlioError, match="error -4"):
            ctx.batch_associate_edges_pairs([0, 2], [1, 1])                 # frame 2 has no corner scan
        assert len(ctx.batch_pair_list()[0]) == 0
        with pytest.raises(api.GlioError, match="error -3"):
            ctx.batch_get_edges(0, 1)
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# K2be evaluation
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0.0, 3000.0, 20000.0])
def test_eval_binary_edge_within_bound(api, offset):
    K = 200
    rng = np.random.default_rng(46)
    poses = ev.make_poses(K, rng, offset=offset)
    spec = [(5, 0, 1), (0, 5, 2048), (20, 30, 2049), (40, 31, 300), (100, 110, 0), (150, 141, 17), (199, 189, 64), (60, 61, 1)]
    ctx = api.Context(0)
    try:
        pairs = []
        ctx.batch_set_pair_matches(70, 72, np.zeros((3, 3), np.float32), np.tile([0, 0, 1.0, 0, 0, 0], (3, 1)), np.ones(3, np.float32))
        pairs.append((70, 72, None))                                       # plane matches, no edges
        for c, o, n in spec:
            m = bref.make_pair_edges(rng, poses[c], poses[o], n) if n else None
            if m is None:
                ctx.batch_set_pair_edges(c, o, np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros(0))
            else:
                ctx.batch_set_pair_edges(c, o, m["cp"], m["pa"], m["pb"], m["s"])
                e = ctx.batch_get_edges(c, o)
                assert np.all(e["src"] == -1) and np.array_equal(e["s"], m["s"])
            pairs.append((c, o, m))
        d = ctx.eval_binary_edge(poses)
        ref = bref.binary_edge_blocks(poses, pairs)
        ev.assert_within(d["Hdiag"], ref["Hdiag"], ref["MHdiag"], "Hdiag")
        ev.assert_within(d["g"], ref["g"], ref["Mg"], "g")
        ev.assert_within(d["Hoff"], ref["Hoff"], ref["MHoff"], "Hoff")
        ev.assert_within(d["cost"], ref["cost"], ref["Mcost"], "cost")
        c = ctx.eval_binary_edge(poses, want_jac=False)
        assert c["cost"] == d["cost"]
        assert not np.any(d["Hoff"][0]) and not np.any(d["Hdiag"][70])     # the plane-only pair has no edge blocks
    finally:
        ctx.close()


def test_point_on_its_line_follows_k2e(api):
    """|e| = 0 exactly: r = 0 and a non-finite Jacobian, in K2be as in the window's K2e"""
    ident = np.array([[0.0, 0, 0, 1, 0, 0, 0]] * 2)
    cp = np.array([[1.0, 2.0, 3.0]], np.float32); pa = cp.copy(); pb = np.array([[1.5, 2.0, 3.0]], np.float32)
    ctx = api.Context(0)
    w = api.Context(0, q_lb=[1.0, 0, 0, 0], t_lb=[0.0, 0, 0])
    try:
        ctx.batch_set_pair_edges(0, 1, cp, pa, pb, np.ones(1))
        b = ctx.eval_binary_edge(ident)
        w.set_edges(0, cp, pa, pb, np.ones(1))
        u = w.eval_edge(ident[:1])
        assert b["cost"] == 0.0 and u["cost"][0] == 0.0
        assert not np.isfinite(b["Hdiag"][0]).all() and not np.isfinite(u["H"][0]).all()
    finally:
        ctx.close(); w.close()


# ---------------------------------------------------------------------------------------------------------------------------
# batch solve with edges
# ---------------------------------------------------------------------------------------------------------------------------
def _problem(K=10, sr=2):
    B = synth.batch_problem(K=K, Q=4000, seed=47, search_range=sr, rng_range=8.0)
    E = synth.batch_edge_problem(K=K, Q=3000, seed=47, search_range=sr, rng_range=8.0)
    cur, oth = gdist.batch_pairs(K, sr)
    return B, E, cur, oth


def _ctx(api, B, E, cur, oth, edges=True, planes=True):
    c = api.Context(0)
    for k in range(B["K"]):
        c.batch_set_frame(k, B["scans"][k], B["poses_init"][k])
        if edges:
            c.batch_set_edge_frame(k, E["corner_scans"][k])
    c.batch_declare_pairs(cur, oth)
    if planes:
        c.batch_associate_pairs(cur, oth)
    if edges:
        assert c.batch_associate_edges_pairs(cur, oth).sum() > 100
    return c


def _host_factor_set(api, B, sb, prior_only=False):
    hf = api.HostFactorSet(); T = B["poses_true"]; rng = np.random.default_rng(7)
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0 if sb else 0.0)])
    hf.add_prior(0, T[0, :3], T[0, 3:], np.zeros(9) if sb else None, sw * 3)
    if not prior_only:
        for i in range(B["K"] - 1):
            dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
            hf.add_between(i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw)
    return hf


def _solve_with_band_callback(api, ctx, poses, sb, hf, edge_ctx, pair_list, max_iter):
    """glio_batch_solve with host factors = hf + the edge blocks edge_ctx evaluates, written into the band"""
    L = ctx._lib
    pb = np.array(poses, np.float64).copy(); K = len(pb)
    sbv = None if sb is None else np.array(sb, np.float64).copy()
    nt = 15 if sbv is not None else 6
    cur, oth = pair_list

    def cb(user, Kc, p, s, want_jac, H, hb, g, cost):
        rc = L.glio_hf_evaluate_band(hf._h, Kc, p, s, want_jac, H, hb, g, cost)
        if rc != 0:
            return rc
        pz = np.ctypeslib.as_array(p, (Kc * 7,)).reshape(Kc, 7).copy()
        e = edge_ctx.eval_binary_edge(pz, want_jac=bool(want_jac))
        cost[0] = cost[0] + e["cost"]
        if want_jac:
            w = hb + 1
            band = np.ctypeslib.as_array(H, (Kc * nt * w,)).reshape(Kc * nt, w)
            gv = np.ctypeslib.as_array(g, (Kc * nt,))
            for k in range(Kc):
                for i in range(6):
                    for j in range(i + 1):
                        band[nt * k + i, j - i + hb] += e["Hdiag"][k, i, j]
                gv[nt * k:nt * k + 6] += e["g"][k]
            for p_, (kc, ko) in enumerate(zip(cur, oth)):
                Ho = e["Hoff"][p_]
                for a in range(6):
                    for b in range(6):
                        if kc > ko:
                            i, j = nt * kc + a, nt * ko + b
                        else:
                            i, j = nt * ko + b, nt * kc + a
                        band[i, j - i + hb] += Ho[a, b]
        return 0
    fn = api.HOST_FACTORS_BAND_FN(cb)
    opt = api.batch_solver_options(max_num_iterations=max_iter)
    summ = api.SolverSummary(); log = (api.Iteration * 64)(); n = K * nt; steps = np.zeros((64, n))
    ctx._chk(L.glio_batch_solve(ctx._h, C.c_int(K), api._ptr(pb), api._ptr(sbv), fn, None, C.byref(opt), C.byref(summ), log,
                                C.c_int(64), api._ptr(steps), C.c_int64(steps.size)))
    return dict(poses=pb, summary=summ, iterations=api.iterations_to_dicts(log, min(summ.num_iterations, 64)), steps=steps[:summ.num_valid_steps])


@pytest.mark.parametrize("with_sb", [False, True])
def test_solve_with_edges_matches_host_factor_composition(api, with_sb):
    B, E, cur, oth = _problem()
    K = B["K"]
    a = _ctx(api, B, E, cur, oth)                              # edges inside the solve
    p = _ctx(api, B, E, cur, oth, edges=False)                 # planes only, the edge blocks come from e as host factors
    e = _ctx(api, B, E, cur, oth, planes=False)
    try:
        assert np.array_equal(np.array(p.batch_pair_list()), np.array(a.batch_pair_list()))
        hf = _host_factor_set(api, B, with_sb)
        sb = np.zeros((K, 9)) if with_sb else None
        a.batch_use_edges(True)
        ra = a.batch_solve(B["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=10))
        rb = _solve_with_band_callback(api, p, B["poses_init"], sb, hf, e, a.batch_pair_list(), 10)
        sa, sb_ = ra["summary"], rb["summary"]
        assert sa.num_iterations == sb_.num_iterations >= 3 and sa.num_valid_steps == sb_.num_valid_steps
        assert [it["step_is_successful"] for it in ra["iterations"]] == [it["step_is_successful"] for it in rb["iterations"]]
        nt = 15 if with_sb else 6
        for x, y in zip(ra["steps"], rb["steps"]):
            x = x.reshape(K, nt); y = y.reshape(K, nt)
            assert np.max(np.abs(x[:, :3] - y[:, :3])) <= 1e-6 and np.max(2 * np.linalg.norm(x[:, 3:6] - y[:, 3:6], axis=1)) <= 1e-8
        assert abs(sa.final_cost - sb_.final_cost) <= 1e-9 * abs(sb_.final_cost)
    finally:
        for c in (a, p, e):
            c.close()


def test_corner_only_solve_reduces_pose_error(api):
    B, E, cur, oth = _problem()
    c = _ctx(api, B, E, cur, oth, planes=False)
    try:
        c.batch_use_edges(True)
        hf = _host_factor_set(api, B, False, prior_only=True)
        r = c.batch_solve(B["poses_init"], None, hf, api.batch_solver_options(max_num_iterations=30))
        err = lambda P: np.mean(np.linalg.norm(P[:, :3] - B["poses_true"][:, :3], axis=1))
        assert r["summary"].final_cost < r["summary"].initial_cost
        assert err(r["poses"]) < err(B["poses_init"])
    finally:
        c.close()


def test_switch_off_or_no_edges_changes_nothing(api):
    B, E, cur, oth = _problem()
    plain = _ctx(api, B, E, cur, oth, edges=False)
    off = _ctx(api, B, E, cur, oth)                            # edges associated, switch turned on and off again
    off.batch_use_edges(True); off.batch_use_edges(False)
    empty = _ctx(api, B, E, cur, oth, edges=False)             # switch on, no edges
    empty.batch_use_edges(True)
    try:
        hf = _host_factor_set(api, B, False)
        opts = api.batch_solver_options(max_num_iterations=6)
        r0 = plain.batch_solve(B["poses_init"], None, hf, opts); e0 = plain.eval_binary(B["poses_init"])
        for c in (off, empty):
            assert np.array_equal(np.array(c.batch_pair_list()), np.array(plain.batch_pair_list()))
            e1 = c.eval_binary(B["poses_init"])
            assert all(np.array_equal(e0[k], e1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
            r1 = c.batch_solve(B["poses_init"], None, hf, opts)
            assert np.array_equal(r0["poses"], r1["poses"]) and np.array_equal(r0["steps"], r1["steps"])
        # selection: bit-identical, and it leaves the edge lists alone
        before = {(int(a), int(b)): off.batch_get_edges(int(a), int(b)) for a, b in zip(cur, oth)}
        n0 = plain.batch_select_random(cur, oth, 1, batch_feature_res_num=25, seed=3)
        n1 = off.batch_select_random(cur, oth, 1, batch_feature_res_num=25, seed=3)
        assert np.array_equal(n0, n1)
        for a, b in zip(cur, oth):
            s0, s1 = plain.batch_get_selection(int(a), int(b)), off.batch_get_selection(int(a), int(b))
            assert (s0 is None and s1 is None) or np.array_equal(s0, s1)
            after = off.batch_get_edges(int(a), int(b))
            assert all(np.array_equal(after[k], before[(int(a), int(b))][k]) for k in ("cp", "pa", "pb", "s", "src"))
        e0 = plain.eval_binary(B["poses_init"]); e1 = off.eval_binary(B["poses_init"])
        assert all(np.array_equal(e0[k], e1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
    finally:
        for c in (plain, off, empty):
            c.close()


def test_interleaved_edge_calls_leave_planes_alone(api):
    B, E, cur, oth = _problem()
    plain = _ctx(api, B, E, cur, oth, edges=False)
    mixed = api.Context(0)
    try:
        for k in range(B["K"]):
            mixed.batch_set_frame(k, B["scans"][k], B["poses_init"][k])
            mixed.batch_set_edge_frame(k, E["corner_scans"][k])
        mixed.batch_declare_pairs(cur, oth)
        half = len(cur) // 2
        mixed.batch_associate_edges_pairs(cur[:half], oth[:half])
        mixed.batch_associate_pairs(cur[:half], oth[:half])
        mixed.batch_associate_edges_pairs(cur, oth)
        mixed.batch_associate_pairs(cur[half:], oth[half:])
        for a, b in zip(cur, oth):
            m0, m1 = plain.batch_get_matches(int(a), int(b), 4000), mixed.batch_get_matches(int(a), int(b), 4000)
            assert all(np.array_equal(m0[k], m1[k]) for k in ("cp", "weight", "normal_cent", "src"))
        e0 = plain.eval_binary(B["poses_init"]); e1 = mixed.eval_binary(B["poses_init"])
        assert all(np.array_equal(e0[k], e1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
    finally:
        plain.close(); mixed.close()
