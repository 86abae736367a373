"""K2p on the device: glio_eval_pose_factors within the a-priori bound of the longdouble reference (tests/pose_factor_reference.py),
the argument checks of glio_batch_set_pose_factors, glio_batch_solve with the pose factors on against the same problem with the
pose blocks handed in through the band host callback, and what the switch must leave alone when it is off."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth
from tests import eval_reference as er
from tests import pose_factor_reference as pr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _exact_pairs_factors(api, rng, K, n_pairs, n, span):
    """n factors over exactly n_pairs distinct pairs (a, b), b - a <= span: each pair once, in random order and orientation,
    then the rest on random pairs of the same set"""
    cand = [(a, b) for a in range(K) for b in range(a + 1, min(K, a + span + 1))]
    assert len(cand) >= n_pairs and n >= n_pairs
    pick = np.array(cand)[rng.choice(len(cand), n_pairs, replace=False)]
    which = np.concatenate([np.arange(n_pairs), rng.integers(0, n_pairs, n - n_pairs)])
    ab = pick[which]
    flip = rng.random(n) < 0.5
    i = np.where(flip, ab[:, 1], ab[:, 0]); j = np.where(flip, ab[:, 0], ab[:, 1])
    dq = rng.normal(size=(n, 4)); dq[:, 0] += 4.0; dq /= np.linalg.norm(dq, axis=1)[:, None]
    return api.pose_factor_records(i, j, rng.choice([0, 1], n), dq, rng.normal(0, 1.5, (n, 3)))


def _random_factors(api, rng, K, n, kinds=(0, 1), span=None):
    i = rng.integers(0, K, n)
    if span is None:
        j = rng.integers(0, K - 1, n); j = np.where(j >= i, j + 1, j)
    else:
        d = rng.integers(1, span + 1, n) * rng.choice([-1, 1], n)
        j = np.clip(i + d, 0, K - 1); j = np.where(j == i, np.where(i > 0, i - 1, i + 1), j)
    dq = rng.normal(size=(n, 4)); dq[:, 0] += 4.0; dq /= np.linalg.norm(dq, axis=1)[:, None]
    return api.pose_factor_records(i, j, rng.choice(kinds, n), dq, rng.normal(0, 1.5, (n, 3)))


def _check(api, ctx, poses, f):
    ctx.batch_set_pose_factors(f)
    a, b = ctx.batch_pose_pair_list()
    R = pr.pose_blocks(poses, f)
    assert list(zip(a.tolist(), b.tolist())) == R["pairs"]
    d = ctx.eval_pose_factors(poses)
    er.assert_within(d["Hdiag"], R["Hdiag"], R["MHdiag"], "Hdiag")
    er.assert_within(d["g"], R["g"], R["Mg"], "g")
    if len(a):
        er.assert_within(d["Hoff"], R["Hoff"], R["MHoff"], "Hoff")
    er.assert_within(d["cost"], R["cost"], R["Mcost"], "cost")
    c = ctx.eval_pose_factors(poses, want_jac=False)                         # the cost-only kernel
    er.assert_within(c["cost"], R["cost"], R["Mcost"], "cost without Jacobians")
    return d


POSES = {"near": dict(offset=0.0), "3km": dict(offset=3000.0), "20km": dict(offset=20000.0),
         "q_nonunit": dict(qnorm=[0.5, 2.0, 1.3, 0.8]), "w_zero": dict(w_zero=True)}


@pytest.mark.parametrize("fx", list(POSES))
@pytest.mark.parametrize("K,n_pairs,n", [(2, 1, 1), (5, 7, 7), (9, 8, 8), (9, 9, 20), (20, 16, 16), (20, 17, 40), (64, 200, 300),
                                         (4096, 3000, 5000)])
def test_eval_matches_reference(api, fx, K, n_pairs, n):
    """exact pair counts around the kernel's 8 pairs per block (1, 7, 8, 9, 16, 17) and larger lists"""
    rng = np.random.default_rng(K * 31 + n)
    kw = dict(POSES[fx])
    if "qnorm" in kw:
        kw["qnorm"] = np.resize(kw["qnorm"], K)
    poses = er.make_poses(K, rng, **kw)
    f = _exact_pairs_factors(api, rng, K, n_pairs, n, span=6)
    ctx = api.Context(0)
    try:
        _check(api, ctx, poses, f)
        assert len(ctx.batch_pose_pair_list()[0]) == n_pairs
    finally:
        ctx.close()


def test_eval_duplicates_inactive_pairs_and_both_orders(api):
    rng = np.random.default_rng(5)
    K = 12
    poses = er.make_poses(K, rng, offset=3000.0, qnorm=np.resize([1.0, 1.7, 0.6], K))
    base = _random_factors(api, rng, K - 2, 40, span=4)                     # keyframes 0 .. 9
    dup = np.concatenate([base, base[:10], base[:10]])                       # the same factors repeated: long per-pair runs
    dup["i"][-5:], dup["j"][-5:] = dup["j"][-5:].copy(), dup["i"][-5:].copy()  # and some with i > j
    extra = api.pose_factor_records([10, 11], [11, 10], [0, 1], np.tile([1.0, 0, 0, 0], (2, 1)), active=[0, 0])
    f = np.concatenate([dup, extra])                                         # pair (10, 11) made only of inactive factors
    ctx = api.Context(0)
    try:
        d = _check(api, ctx, poses, f)
        a, b = ctx.batch_pose_pair_list()
        k = list(zip(a.tolist(), b.tolist())).index((10, 11))
        assert np.all(d["Hoff"][k] == 0.0)
        # the same pairs, factors in another order inside a pair: within the bound as well (the sum order only changes)
        _check(api, ctx, poses, f[::-1].copy())
    finally:
        ctx.close()


def test_eval_sample_run_size_and_empty_list(api):
    P = synth.pose_graph_problem(K=3457)
    f = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    ctx = api.Context(0)
    try:
        _check(api, ctx, P["poses_init"], f)
        ctx.batch_set_pose_factors(f[:0])
        assert len(ctx.batch_pose_pair_list()[0]) == 0
        d = ctx.eval_pose_factors(P["poses_init"][:1])                      # K = 1, nothing to evaluate
        assert np.all(d["Hdiag"] == 0) and d["cost"] == 0.0
    finally:
        ctx.close()


def test_argument_checks_keep_the_previous_list(api):
    rng = np.random.default_rng(9)
    K = 10
    poses = er.make_poses(K, rng)
    good = _random_factors(api, rng, K, 20, span=3)
    ctx = api.Context(0)
    try:
        ctx.batch_set_pose_factors(good)
        ref = ctx.eval_pose_factors(poses)
        pairs = ctx.batch_pose_pair_list()
        for field, val in (("i", -1), ("j", -3), ("kind", 2), ("kind", -1), ("i", api.POSE_MAX_KF), ("j", 2**31 - 1)):
            bad = good.copy(); bad[field][7] = val
            with pytest.raises(api.GlioError):
                ctx.batch_set_pose_factors(bad)
        bad = good.copy(); bad["j"][3] = bad["i"][3]
        with pytest.raises(api.GlioError):
            ctx.batch_set_pose_factors(bad)
        rc = ctx._lib.glio_batch_set_pose_factors(ctx._h, None, C.c_int64(3))
        assert rc != 0
        hi = good.copy(); hi["j"][0] = K                                     # accepted, but K keyframes are too few
        ctx.batch_set_pose_factors(hi)
        with pytest.raises(api.GlioError):
            ctx.eval_pose_factors(poses)
        ctx.batch_use_pose_factors(True)
        with pytest.raises(api.GlioError):
            ctx.batch_solve(poses, options=api.batch_solver_options(max_num_iterations=2))
        ctx.batch_set_pose_factors(good)
        assert all(np.array_equal(x, y) for x, y in zip(ctx.batch_pose_pair_list(), pairs))
        again = ctx.eval_pose_factors(poses)
        assert all(np.array_equal(ref[k], again[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
        ctx.batch_clear()
        assert len(ctx.batch_pose_pair_list()[0]) == 0
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the batch solve
# ---------------------------------------------------------------------------------------------------------------------------
def _host_factor_set(api, T, sb):
    hf = api.HostFactorSet(); rng = np.random.default_rng(7)
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0 if sb else 0.0)])
    hf.add_prior(0, T[0, :3], T[0, 3:], np.zeros(9) if sb else None, sw * 3)
    # noisy between factors: the pose factors alone are consistent, and a zero-residual optimum leaves no cost to compare
    for i in range(len(T) - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        hf.add_between(i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw)
    return hf


def _solve_with_pose_callback(api, ctx, poses, sb, hf, f, max_iter):
    """glio_batch_solve with host factors = hf + the reference's pose blocks (rounded to float64), written into the band"""
    L = ctx._lib
    pb = np.array(poses, np.float64).copy(); K = len(pb)
    sbv = None if sb is None else np.array(sb, np.float64).copy()
    nt = 15 if sbv is not None else 6
    pairs = np.array(pr.pair_table(f)[0], np.int32).reshape(-1, 2)
    ctx.batch_declare_pairs(pairs[:, 0], pairs[:, 1])                        # pairs without matches: zero blocks, the pose pairs' bandwidth

    def cb(user, Kc, p, s, want_jac, H, hb, g, cost):
        rc = L.glio_hf_evaluate_band(hf._h, Kc, p, s, want_jac, H, hb, g, cost)
        if rc != 0:
            return rc
        pz = np.ctypeslib.as_array(p, (Kc * 7,)).reshape(Kc, 7).copy()
        e = pr.pose_blocks(pz, f)
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
            for p_, (a, b) in enumerate(e["pairs"]):
                for x in range(6):
                    for y in range(6):
                        i, j = nt * b + y, nt * a + x                       # a < b: the entry lives in b's rows
                        band[i, j - i + hb] += e["Hoff"][p_][x, y]
        return 0
    fn = api.HOST_FACTORS_BAND_FN(cb)
    opt = api.batch_solver_options(max_num_iterations=max_iter)
    summ = api.SolverSummary(); log = (api.Iteration * 64)(); n = K * nt; steps = np.zeros((64, n))
    ctx._chk(L.glio_batch_solve(ctx._h, C.c_int(K), api._ptr(pb), api._ptr(sbv), fn, None, C.byref(opt), C.byref(summ), log,
                                C.c_int(64), api._ptr(steps), C.c_int64(steps.size)))
    return dict(poses=pb, summary=summ, iterations=api.iterations_to_dicts(log, min(summ.num_iterations, 64)), steps=steps[:summ.num_valid_steps])


def _pair_edges(rng, pose_c, pose_o, n, noise=0.02):
    """n binary edge correspondences of pair (cur, oth): cp in cur's body frame, the line points in oth's"""
    tc, qc, to, qo = pose_c[:3], pose_c[3:], pose_o[:3], pose_o[3:]
    a = tc + rng.uniform(-20, 20, (n, 3)); d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1)[:, None]
    b = a + d * rng.uniform(0.2, 1.0, (n, 1))
    pw = a + d * rng.uniform(-1, 2, (n, 1)) + rng.normal(0, noise, (n, 3))
    Rc, Ro = er.rot_poly(qc), er.rot_poly(qo)
    return dict(cp=((pw - tc) @ Rc).astype(np.float32), pa=((a - to) @ Ro).astype(np.float32), pb=((b - to) @ Ro).astype(np.float32),
                s=rng.uniform(0.5, 2.0, n).astype(np.float32).astype(np.float64))


def _pairs_ctx(api, P, K, rng_seed=3, edges=False):
    """a context with P's LiDAR pairs and synthetic plane matches (eval_reference.make_pair at the true poses), and with edges
    binary edge lists and glio_batch_use_edges on"""
    ctx = api.Context(0)
    if "pairs" in P:
        rng = np.random.default_rng(rng_seed)
        cur, oth = P["pairs"]
        ctx.batch_declare_pairs(cur, oth)
        for a, b in zip(cur, oth):
            m = er.make_pair(rng, P["poses_true"][a], P["poses_true"][b], 40, noise=0.02)
            ctx.batch_set_pair_matches(int(a), int(b), m["cp"], m["nc"], m["weight"])
            if edges:
                e = _pair_edges(rng, P["poses_true"][a], P["poses_true"][b], 20)
                ctx.batch_set_pair_edges(int(a), int(b), e["cp"], e["pa"], e["pb"], e["s"])
        if edges:
            ctx.batch_use_edges(True)
    return ctx


def _compare(ra, rb, K, nt):
    sa, sb_ = ra["summary"], rb["summary"]
    assert sa.num_iterations == sb_.num_iterations >= 2 and sa.num_valid_steps == sb_.num_valid_steps
    assert [it["step_is_successful"] for it in ra["iterations"]] == [it["step_is_successful"] for it in rb["iterations"]]
    for x, y in zip(ra["steps"], rb["steps"]):
        x = x.reshape(K, nt); y = y.reshape(K, nt)
        assert np.max(np.abs(x[:, :3] - y[:, :3])) <= 1e-6 and np.max(2 * np.linalg.norm(x[:, 3:6] - y[:, 3:6], axis=1)) <= 1e-8
    assert abs(sa.final_cost - sb_.final_cost) <= 1e-9 * abs(sb_.final_cost)


@pytest.mark.parametrize("level,with_sb,edges", [(0, False, False), (0, True, False), (1, False, False), (1, False, True)])
def test_solve_with_pose_factors_matches_host_callback(api, level, with_sb, edges):
    K = 40
    P = synth.pose_graph_problem(K=K, level=level)
    f = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    hf = _host_factor_set(api, P["poses_true"], with_sb)
    sb = np.zeros((K, 9)) if with_sb else None
    a = _pairs_ctx(api, P, K, edges=edges); b = _pairs_ctx(api, P, K, edges=edges)
    try:
        a.batch_set_pose_factors(f); a.batch_use_pose_factors(True)
        ra = a.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=8))
        rb = _solve_with_pose_callback(api, b, P["poses_init"], sb, hf, f, 8)
        _compare(ra, rb, K, 15 if with_sb else 6)
        if level == 0:
            err = lambda X: np.mean(np.linalg.norm(X[:, :3] - P["poses_true"][:, :3], axis=1))
            assert ra["summary"].final_cost < ra["summary"].initial_cost and err(ra["poses"]) < err(P["poses_init"])
    finally:
        a.close(); b.close()


def test_switch_off_or_empty_list_changes_nothing(api):
    K = 40
    P = synth.pose_graph_problem(K=K, level=1)
    f = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    hf = _host_factor_set(api, P["poses_true"], False)
    plain = _pairs_ctx(api, P, K)
    off = _pairs_ctx(api, P, K); off.batch_set_pose_factors(f); off.batch_use_pose_factors(True); off.batch_use_pose_factors(False)
    empty = _pairs_ctx(api, P, K); empty.batch_set_pose_factors(f); empty.batch_set_pose_factors(f[:0]); empty.batch_use_pose_factors(True)
    try:
        opts = api.batch_solver_options(max_num_iterations=6)
        n0 = plain.launch_count
        r0 = plain.batch_solve(P["poses_init"], None, hf, opts); e0 = plain.eval_binary(P["poses_init"])
        d0 = plain.launch_count - n0
        for c in (off, empty):
            n1 = c.launch_count
            r1 = c.batch_solve(P["poses_init"], None, hf, opts); e1 = c.eval_binary(P["poses_init"])
            assert c.launch_count - n1 == d0
            assert np.array_equal(r0["poses"], r1["poses"]) and np.array_equal(r0["steps"], r1["steps"])
            assert all(np.array_equal(e0[k], e1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
    finally:
        for c in (plain, off, empty):
            c.close()
