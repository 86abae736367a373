"""K2g on the device: glio_eval_dd_psr_factors within the a-priori bound of the longdouble reference (tests/dd_psr_reference.py),
the gate decided exactly at its threshold, the argument checks of glio_batch_set_dd_psr_factors, glio_batch_solve with the DD
factors on against the same problem with the DD blocks handed in through the band host callback, and what the switch must leave
alone when it is off."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import dist, synth
from tests import dd_psr_reference as dr
from tests import eval_reference as er
from tests import test_gpu_pose_factors as tp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _exact_pairs(rng, K, n_pairs, n, span):
    """n (i, j) over exactly n_pairs distinct pairs, b - a <= span: each pair once, then repeats; random orientation"""
    cand = [(a, b) for a in range(K) for b in range(a + 1, min(K, a + span + 1))]
    pick = np.array(cand)[rng.choice(len(cand), n_pairs, replace=False)]
    ab = pick[np.concatenate([np.arange(n_pairs), rng.integers(0, n_pairs, n - n_pairs)])]
    flip = rng.random(n) < 0.5
    return np.stack([np.where(flip, ab[:, 1], ab[:, 0]), np.where(flip, ab[:, 0], ab[:, 1])], axis=1)


def _check(ctx, poses, f, sats, W, R, anchor):
    ctx.batch_set_dd_psr_factors(f, sats, R, anchor, W)
    a, b = ctx.batch_dd_psr_pair_list()
    ref = dr.dd_blocks(poses, f, sats, R, anchor, W)
    assert list(zip(a.tolist(), b.tolist())) == ref["pairs"]
    assert ref["gate_margin"] > 1e-6                                          # the gate is decided on the same side
    d = ctx.eval_dd_psr_factors(poses)
    er.assert_within(d["Hdiag"], ref["Hdiag"], ref["MHdiag"], "Hdiag")
    er.assert_within(d["g"], ref["g"], ref["Mg"], "g")
    if len(a):
        er.assert_within(d["Hoff"], ref["Hoff"], ref["MHoff"], "Hoff")
    er.assert_within(d["cost"], ref["cost"], ref["Mcost"], "cost")
    c = ctx.eval_dd_psr_factors(poses, want_jac=False)                        # the cost-only kernel
    er.assert_within(c["cost"], ref["cost"], ref["Mcost"], "cost without Jacobians")
    return d


@pytest.mark.parametrize("offset", [0.0, 3000.0])
@pytest.mark.parametrize("K,n_pairs,n", [(2, 1, 1), (6, 3, 3), (8, 4, 4), (8, 5, 12), (20, 8, 8), (20, 9, 30), (64, 150, 300),
                                         (4096, 3000, 5000)])
def test_eval_matches_reference(api, offset, K, n_pairs, n):
    """exact pair counts around the kernel's 4 pairs per block; n_sat 2, 3, 19 and 20 and others, the master first, last and in
    between, with and without W, ratio 0, 1 and between, i > j, repeated pairs; km-scale translations"""
    rng = np.random.default_rng(K * 131 + n)
    poses = er.make_poses(K, rng, offset=offset)
    ij = _exact_pairs(rng, K, n_pairs, n, span=6)
    n_sat = np.resize([2, 3, 19, 20, 7, 12], n)
    master = np.array([(0, s - 1, s // 2)[k % 3] for k, s in enumerate(n_sat)])
    ratio = np.resize([0.0, 1.0, 0.37, 0.81], n)
    f, sats, W, R, anchor = dr.random_list(rng, poses, ij, n_sat, master, ratio, with_w=True)
    ctx = api.Context(0)
    try:
        _check(ctx, poses, f, sats, W, R, anchor)
        assert len(ctx.batch_dd_psr_pair_list()[0]) == n_pairs
    finally:
        ctx.close()


def test_eval_duplicates_and_inactive(api):
    rng = np.random.default_rng(5)
    K = 12
    poses = er.make_poses(K, rng, offset=3000.0)
    ij = _exact_pairs(rng, K - 2, 10, 30, span=3)
    ij = np.concatenate([ij, ij[:12], [(10, 11), (11, 10)]])                 # long per-pair runs; a pair of inactive factors only
    f, sats, W, R, anchor = dr.random_list(rng, poses, ij, rng.integers(2, 21, len(ij)), with_w=True)
    f["active"][-2:] = 0
    ctx = api.Context(0)
    try:
        d = _check(ctx, poses, f, sats, W, R, anchor)
        a, b = ctx.batch_dd_psr_pair_list()
        k = list(zip(a.tolist(), b.tolist())).index((10, 11))
        assert np.all(d["Hoff"][k] == 0.0) and np.all(d["Hdiag"][11] == 0.0)
        _check(ctx, poses, f[::-1].copy(), sats, W, R, anchor)               # another order inside the pairs
    finally:
        ctx.close()


def test_eval_sample_run_size_and_empty_list(api):
    P = synth.dd_psr_problem(K=3457)
    f = api.dd_psr_factor_records(**P["dd"])
    sats = api.dd_psr_sat_records(**P["dd_sats"])
    ctx = api.Context(0)
    try:
        _check(ctx, P["poses_init"], f, sats, None, P["R"], P["anchor"])
        ctx.batch_set_dd_psr_factors(f[:0], sats[:0], P["R"], P["anchor"])
        assert len(ctx.batch_dd_psr_pair_list()[0]) == 0
        d = ctx.eval_dd_psr_factors(P["poses_init"][:1])
        assert np.all(d["Hdiag"] == 0) and d["cost"] == 0.0
    finally:
        ctx.close()


def test_gate_is_exact_at_the_threshold(api):
    """t_i = t_j = 0, station = anchor, sat_ref = sat_user: P is the anchor bit for bit, the estimated double difference is exactly
    0 and r = -DD_psr is an integer; |r| == threshold keeps weight 1, one ulp less gives 0.05"""
    R, anchor, _ = dr.frame()
    poses = np.zeros((2, 7)); poses[:, 3] = 1.0
    rng = np.random.default_rng(2)
    sats = dr.random_sats(rng, 3, anchor, anchor, anchor)
    sats["sat_ref"] = sats["sat_user"]
    sats["psr_user"] = [21_000_123.0, 22_000_456.0, 23_500_001.0]; sats["psr_ref"] = [21_000_100.0, 22_000_437.0, 23_499_990.0]
    e = -np.array([(22_000_456.0 - 22_000_437.0) - (21_000_123.0 - 21_000_100.0), (23_500_001.0 - 23_499_990.0) - (21_000_123.0 - 21_000_100.0)])
    assert np.all(e == [4.0, 12.0])
    ctx = api.Context(0)
    try:
        out = {}
        for name, thr in (("equal", 12.0), ("below", np.nextafter(12.0, 0.0))):
            f = api.dd_psr_factor_records([0], [1], [3], [0], [0.3], [thr], anchor)
            ctx.batch_set_dd_psr_factors(f, sats, R, anchor)
            out[name] = ctx.eval_dd_psr_factors(poses)
        assert out["equal"]["cost"] == 0.5 * (4.0 * 4.0 + 12.0 * 12.0)
        r = 0.05 * 12.0
        assert out["below"]["cost"] == 0.5 * 4.0 * 4.0 + 0.5 * r * r
    finally:
        ctx.close()


def test_argument_checks_keep_the_previous_list(api):
    rng = np.random.default_rng(9)
    K = 10
    poses = er.make_poses(K, rng)
    ij = _exact_pairs(rng, K, 8, 16, span=3)
    good, sats, W, R, anchor = dr.random_list(rng, poses, ij, rng.integers(3, 21, 16), with_w=True)
    w_any = int(np.nonzero(good["w_offset"] >= 0)[0][0])
    ctx = api.Context(0)
    try:
        ctx.batch_set_dd_psr_factors(good, sats, R, anchor, W)
        ref = ctx.eval_dd_psr_factors(poses)
        pairs = ctx.batch_dd_psr_pair_list()
        bads = [("i", 0, -1), ("j", 3, -2), ("i", 7, api.DD_PSR_MAX_KF), ("n_sat", 2, 1), ("n_sat", 2, 21), ("master", 4, -1),
                ("master", 5, int(good["n_sat"][5])), ("sat_offset", 6, -1), ("sat_offset", 15, len(sats) - int(good["n_sat"][15]) + 1),
                ("w_offset", 1, -2), ("w_offset", w_any, len(W))]
        for field, k, val in bads:
            bad = good.copy(); bad[field][k] = val
            with pytest.raises(api.GlioError):
                ctx.batch_set_dd_psr_factors(bad, sats, R, anchor, W)
        bad = good.copy(); bad["j"][3] = bad["i"][3]
        with pytest.raises(api.GlioError):
            ctx.batch_set_dd_psr_factors(bad, sats, R, anchor, W)
        f = np.ascontiguousarray(good)
        assert ctx._lib.glio_batch_set_dd_psr_factors(ctx._h, api._ptr(f), C.c_int64(len(f)), api._ptr(sats), C.c_int64(len(sats)),
                                                      api._ptr(W), C.c_int64(len(W)), None, api._ptr(anchor)) != 0
        assert ctx._lib.glio_batch_set_dd_psr_factors(ctx._h, None, C.c_int64(3), None, C.c_int64(0), None, C.c_int64(0), None, None) != 0
        hi = good.copy(); hi["j"][0] = K                                     # accepted, but K keyframes are too few
        ctx.batch_set_dd_psr_factors(hi, sats, R, anchor, W)
        with pytest.raises(api.GlioError):
            ctx.eval_dd_psr_factors(poses)
        ctx.batch_use_dd_psr_factors(True)
        with pytest.raises(api.GlioError):
            ctx.batch_solve(poses, options=api.batch_solver_options(max_num_iterations=2))
        ctx.batch_set_dd_psr_factors(good, sats, R, anchor, W)
        for field, k, val in bads[:3]:                                      # refused after a replacement as well
            bad = good.copy(); bad[field][k] = val
            with pytest.raises(api.GlioError):
                ctx.batch_set_dd_psr_factors(bad, sats, R, anchor, W)
        assert all(np.array_equal(x, y) for x, y in zip(ctx.batch_dd_psr_pair_list(), pairs))
        again = ctx.eval_dd_psr_factors(poses)
        assert all(np.array_equal(ref[k], again[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
        ctx.batch_clear()
        assert len(ctx.batch_dd_psr_pair_list()[0]) == 0
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the batch solve
# ---------------------------------------------------------------------------------------------------------------------------
def _problem(api, K, lidar=False):
    P = synth.dd_psr_problem(K=K)
    if lidar:
        P["pairs"] = dist.batch_pairs(K, P["search_range"])
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    f = api.dd_psr_factor_records(**P["dd"])
    sats = api.dd_psr_sat_records(**P["dd_sats"])
    return P, pf, f, sats


def _solve_with_dd_callback(api, ctx, P, sb, hf, f, sats, max_iter):
    """glio_batch_solve with host factors = hf + the reference's DD blocks (rounded to float64), written into the band"""
    L = ctx._lib
    pb = np.array(P["poses_init"], np.float64).copy(); K = len(pb)
    sbv = None if sb is None else np.array(sb, np.float64).copy()
    nt = 15 if sbv is not None else 6
    pairs = np.array(dr.pair_table(f)[0], np.int32).reshape(-1, 2)
    ctx.batch_declare_pairs(pairs[:, 0], pairs[:, 1])                        # pairs without matches: the DD pairs' bandwidth

    def cb(user, Kc, p, s, want_jac, H, hb, g, cost):
        rc = L.glio_hf_evaluate_band(hf._h, Kc, p, s, want_jac, H, hb, g, cost)
        if rc != 0:
            return rc
        pz = np.ctypeslib.as_array(p, (Kc * 7,)).reshape(Kc, 7).copy()
        e = dr.dd_blocks(pz, f, sats, P["R"], P["anchor"])
        cost[0] = cost[0] + e["cost"]
        if want_jac:
            w = hb + 1
            band = np.ctypeslib.as_array(H, (Kc * nt * w,)).reshape(Kc * nt, w)
            gv = np.ctypeslib.as_array(g, (Kc * nt,))
            for k in range(Kc):
                for i in range(3):
                    for j in range(i + 1):
                        band[nt * k + i, j - i + hb] += e["Hdiag"][k, i, j]
                gv[nt * k:nt * k + 3] += e["g"][k, :3]
            for p_, (a, b) in enumerate(e["pairs"]):
                for x in range(3):
                    for y in range(3):
                        i, j = nt * b + y, nt * a + x
                        band[i, j - i + hb] += e["Hoff"][p_][x, y]
        return 0
    fn = api.HOST_FACTORS_BAND_FN(cb)
    opt = api.batch_solver_options(max_num_iterations=max_iter)
    summ = api.SolverSummary(); log = (api.Iteration * 64)(); n = K * nt; steps = np.zeros((64, n))
    ctx._chk(L.glio_batch_solve(ctx._h, C.c_int(K), api._ptr(pb), api._ptr(sbv), fn, None, C.byref(opt), C.byref(summ), log,
                                C.c_int(64), api._ptr(steps), C.c_int64(steps.size)))
    return dict(poses=pb, summary=summ, iterations=api.iterations_to_dicts(log, min(summ.num_iterations, 64)), steps=steps[:summ.num_valid_steps])


@pytest.mark.parametrize("with_sb,lidar,edges", [(False, False, False), (True, False, False), (False, True, True)])
def test_solve_with_dd_factors_matches_host_callback(api, with_sb, lidar, edges):
    """level 0 with the pose factors on the device in both arms; the DD blocks on the device in one, through the callback in the
    other"""
    K = 40
    P, pf, f, sats = _problem(api, K, lidar)
    hf = tp._host_factor_set(api, P["poses_true"], with_sb)
    sb = np.zeros((K, 9)) if with_sb else None
    a = tp._pairs_ctx(api, P, K, edges=edges); b = tp._pairs_ctx(api, P, K, edges=edges)
    try:
        for c in (a, b):
            c.batch_set_pose_factors(pf); c.batch_use_pose_factors(True)
        a.batch_set_dd_psr_factors(f, sats, P["R"], P["anchor"]); a.batch_use_dd_psr_factors(True)
        ra = a.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=8))
        rb = _solve_with_dd_callback(api, b, P, sb, hf, f, sats, 8)
        tp._compare(ra, rb, K, 15 if with_sb else 6)
        assert ra["summary"].final_cost < ra["summary"].initial_cost
    finally:
        a.close(); b.close()


def test_solve_with_dd_factors_and_no_other_pairs(api):
    """the DD pairs alone set the band (no LiDAR or pose pair) and the solve moves the trajectory toward the GNSS positions"""
    K = 30
    P, pf, f, sats = _problem(api, K)
    hf = tp._host_factor_set(api, P["poses_true"], False)
    ctx = api.Context(0)
    try:
        ctx.batch_set_dd_psr_factors(f, sats, P["R"], P["anchor"]); ctx.batch_use_dd_psr_factors(True)
        r = ctx.batch_solve(P["poses_init"], None, hf, api.batch_solver_options(max_num_iterations=10))
        assert r["summary"].num_iterations >= 2 and r["summary"].final_cost < r["summary"].initial_cost
    finally:
        ctx.close()


def test_switch_off_or_empty_list_changes_nothing(api):
    K = 40
    P, pf, f, sats = _problem(api, K, lidar=True)
    hf = tp._host_factor_set(api, P["poses_true"], False)

    def make():
        c = tp._pairs_ctx(api, P, K); c.batch_set_pose_factors(pf); c.batch_use_pose_factors(True)
        return c
    plain = make()
    off = make(); off.batch_set_dd_psr_factors(f, sats, P["R"], P["anchor"]); off.batch_use_dd_psr_factors(True); off.batch_use_dd_psr_factors(False)
    empty = make(); empty.batch_set_dd_psr_factors(f, sats, P["R"], P["anchor"]); empty.batch_set_dd_psr_factors(f[:0], sats[:0], P["R"], P["anchor"])
    empty.batch_use_dd_psr_factors(True)
    on = make(); on.batch_set_dd_psr_factors(f, sats, P["R"], P["anchor"]); on.batch_use_dd_psr_factors(True)
    try:
        opts = api.batch_solver_options(max_num_iterations=6)
        n0 = plain.launch_count
        r0 = plain.batch_solve(P["poses_init"], None, hf, opts)
        d0 = plain.launch_count - n0
        e0 = plain.eval_binary(P["poses_init"]); p0 = plain.eval_pose_factors(P["poses_init"])
        for c in (off, empty):
            n1 = c.launch_count
            r1 = c.batch_solve(P["poses_init"], None, hf, opts)
            assert c.launch_count - n1 == d0
            assert np.array_equal(r0["poses"], r1["poses"]) and np.array_equal(r0["steps"], r1["steps"])
        for c in (off, empty, on):                                           # the LiDAR and pose evaluations never add DD blocks
            e1 = c.eval_binary(P["poses_init"]); p1 = c.eval_pose_factors(P["poses_init"])
            assert all(np.array_equal(e0[k], e1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
            assert all(np.array_equal(p0[k], p1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
    finally:
        for c in (plain, off, empty, on):
            c.close()
