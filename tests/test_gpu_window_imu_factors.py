"""The window's IMU chain on the device (glio_window_set_imu_factors, glio_eval_window_imu_factors, glio_window_use_imu_factors):
the evaluation against the longdouble references (tangent columns: tests/imu_factor_reference.py; ambient columns:
tests/window_imu_reference.py), the dense and band window solves and the marginalisation against the same problems whose host
callbacks hand in the reference IMU blocks, a multi-step pipelined run, the refusals, and what the switch leaves alone when off."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth
from tests import eval_reference as er
from tests import imu_factor_reference as ir
from tests import window_imu_reference as wr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _quirky(P, seed):
    """P's initial states with non-unit and w < 0 quaternions, 20 km offsets and Bg_i away from linearized_bg; its IMU columns
    with every other factor's i and j swapped"""
    rng = np.random.default_rng(seed)
    W = len(P["poses_init"])
    poses = P["poses_init"].copy(); sb = P["sb_init"].copy()
    poses[:, 3:] *= rng.uniform(0.7, 1.4, (W, 1)); poses[1::3, 3:] *= -1.0
    poses[:, :3] += np.array([20_000.0, -12_000.0, 150.0])
    sb[:, 6:] += rng.normal(0.0, 0.01, (W, 3))
    cols = dict(P["imu"]); i, j = cols["i"].copy(), cols["j"].copy()
    cols["i"] = np.where(np.arange(len(i)) % 2 == 1, j, i); cols["j"] = np.where(np.arange(len(i)) % 2 == 1, i, j)
    return poses, sb, cols


def _check(ctx, poses, sb, f):
    ctx.window_set_imu_factors(f)
    a, b = ctx.window_imu_pair_list()
    for kind, ref in ((0, ir.imu_blocks(poses, sb, f)), (1, wr.imu_blocks(poses, sb, f))):
        assert list(zip(a.tolist(), b.tolist())) == ref["pairs"]
        d = ctx.eval_window_imu_factors(poses, sb, kind)
        er.assert_within(d["Hdiag"], ref["Hdiag"], ref["MHdiag"], f"Hdiag kind {kind}")
        er.assert_within(d["g"], ref["g"], ref["Mg"], f"g kind {kind}")
        if len(a):
            er.assert_within(d["Hoff"], ref["Hoff"], ref["MHoff"], f"Hoff kind {kind}")
        er.assert_within(d["cost"], ref["cost"], ref["Mcost"], f"cost kind {kind}")
        c = ctx.eval_window_imu_factors(poses, sb, kind, want_jac=False)
        er.assert_within(c["cost"], ref["cost"], ref["Mcost"], f"cost without Jacobians, kind {kind}")
    # kind 0 is glio_eval_imu_factors on the same records set as the batch list, bit for bit
    ctx.batch_set_imu_factors(f)
    t, u = ctx.eval_window_imu_factors(poses, sb, 0), ctx.eval_imu_factors(poses, sb)
    assert all(np.array_equal(t[k], u[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
    return d


@pytest.mark.parametrize("W", [2, 5, 20, 1000])
def test_eval_matches_reference(api, W):
    P = synth.window_imu_problem(W=W, Q=64, M=2000, seed=50 + W)
    ctx = api.Context(0)
    try:
        _check(ctx, P["poses_init"], P["sb_init"], api.imu_factor_records(**P["imu"]))
        poses, sb, cols = _quirky(P, W)
        _check(ctx, poses, sb, api.imu_factor_records(**cols))
        assert len(ctx.window_imu_pair_list()[0]) == W - 1
    finally:
        ctx.close()


def test_eval_duplicates_inactive_and_empty(api):
    W = 12
    P = synth.window_imu_problem(W=W, Q=64, M=2000, seed=61)
    poses, sb, cols = _quirky(P, 4)
    f = api.imu_factor_records(**cols)
    n0 = len(f)
    f = np.concatenate([f, f[:5], f[3:4], f[3:4]])
    f["i"][-1], f["j"][-1] = f["j"][-1], f["i"][-1]
    f["active"][[2, n0 + 2, len(f) - 2]] = 0                                   # pair 2 evaluates nothing
    ctx = api.Context(0)
    try:
        d = _check(ctx, poses, sb, f)
        assert np.all(d["Hoff"][2] == 0.0)
        _check(ctx, poses, sb, f[::-1].copy())
        ctx.window_set_imu_factors(f[:0])
        assert len(ctx.window_imu_pair_list()[0]) == 0
        for kind in (0, 1):
            e = ctx.eval_window_imu_factors(poses, sb, kind)
            assert np.all(e["Hdiag"] == 0) and np.all(e["g"] == 0) and e["cost"] == 0.0
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the window solve and the marginalisation
# ---------------------------------------------------------------------------------------------------------------------------
W5 = 5


@pytest.fixture(scope="module")
def problem():
    return (synth.window_imu_problem(W=W5, Q=3000, M=40000, seed=71),
            synth.window_edge_problem(W=W5, Q=1500, M=40000, seed=72))


def _ctx(api, P, E, lidar, edges):
    c = api.Context(0)
    if lidar:
        c.set_map(P["map_xyz"]); c.window_set_scans(P["scans"]); c.window_associate(P["poses_init"])
    if edges:
        c.set_edge_map(E["map_xyz"])
        for k in range(W5):
            c.window_set_edge_scan(k, E["scans"][k])
        assert c.window_associate_edges(P["poses_init"]).min() > 100
        c.window_use_edges(True)
    return c


def _prior_set(api, P):
    """the first window's speed-bias prior stand-in on KF0 (Estimator.cpp:2164-2176) fixes the gauge"""
    hf = api.HostFactorSet()
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)])
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], P["sb_true"][0], sw * 3)
    return hf


def _solve_ref(api, ctx, P, hf, f, band, opts):
    """glio_window_solve(_band) with host factors = hf + the reference's tangent IMU blocks (rounded to float64)"""
    L = ctx._lib
    pb = np.array(P["poses_init"], np.float64).copy(); W = len(pb)
    sbv = np.array(P["sb_init"], np.float64).copy()
    n = 15 * W

    def imu(p, s, W_):
        pz = np.ctypeslib.as_array(p, (W_ * 7,)).reshape(W_, 7).copy()
        sz = np.ctypeslib.as_array(s, (W_ * 9,)).reshape(W_, 9).copy()
        return ir.imu_blocks(pz, sz, f)

    def dense(user, W_, p, s, want_jac, H, g, cost):
        rc = L.glio_hf_evaluate(hf._h, W_, p, s, want_jac, H, g, cost)
        if rc != 0:
            return rc
        e = imu(p, s, W_)
        cost[0] = cost[0] + e["cost"]
        if want_jac:
            Hm = np.ctypeslib.as_array(H, (n * n,)).reshape(n, n); gv = np.ctypeslib.as_array(g, (n,))
            for k in range(W_):
                Hm[15 * k:15 * k + 15, 15 * k:15 * k + 15] += e["Hdiag"][k]
                gv[15 * k:15 * k + 15] += e["g"][k]
            for p_, (a, b) in enumerate(e["pairs"]):
                Hm[15 * a:15 * a + 15, 15 * b:15 * b + 15] += e["Hoff"][p_]
                Hm[15 * b:15 * b + 15, 15 * a:15 * a + 15] += e["Hoff"][p_].T
        return 0

    def banded(user, W_, p, s, want_jac, H, hb, g, cost):
        rc = L.glio_hf_evaluate_band(hf._h, W_, p, s, want_jac, H, hb, g, cost)
        if rc != 0:
            return rc
        e = imu(p, s, W_)
        cost[0] = cost[0] + e["cost"]
        if want_jac:
            w = hb + 1
            bm = np.ctypeslib.as_array(H, (n * w,)).reshape(n, w); gv = np.ctypeslib.as_array(g, (n,))
            for k in range(W_):
                for i in range(15):
                    bm[15 * k + i, hb - i:hb + 1] += e["Hdiag"][k, i, :i + 1]
                gv[15 * k:15 * k + 15] += e["g"][k]
            for p_, (a, b) in enumerate(e["pairs"]):
                for y in range(15):
                    i = 15 * b + y
                    bm[i, 15 * a - i + hb:15 * a + 15 - i + hb] += e["Hoff"][p_][:, y]
        return 0
    summ = api.SolverSummary(); log = (api.Iteration * 64)(); steps = np.zeros((64, n))
    if band:
        fn = api.HOST_FACTORS_BAND_FN(banded)
        ctx._chk(L.glio_window_solve_band(ctx._h, C.c_int(W), api._ptr(pb), api._ptr(sbv), fn, C.c_int(29), None, C.byref(opts),
                                          C.byref(summ), log, C.c_int(64), api._ptr(steps), C.c_int64(steps.size)))
    else:
        fn = api.HOST_FACTORS_FN(dense)
        ctx._chk(L.glio_window_solve(ctx._h, C.c_int(W), api._ptr(pb), api._ptr(sbv), fn, None, C.byref(opts), C.byref(summ), log,
                                     C.c_int(64), api._ptr(steps), C.c_int64(steps.size)))
    return dict(poses=pb, speed_bias=sbv, summary=summ)


@pytest.mark.parametrize("lidar,edges", [(True, False), (True, True), (False, False)])
@pytest.mark.parametrize("band", [False, True])
def test_solve_matches_host_callback(api, problem, lidar, edges, band):
    P, E = problem
    f = api.imu_factor_records(**P["imu"])
    hf = _prior_set(api, P)
    opts = api.default_solver_options()
    a, b = _ctx(api, P, E, lidar, edges), _ctx(api, P, E, lidar, edges)
    try:
        a.window_set_imu_factors(f); a.window_use_imu_factors(True)
        ra = a.window_solve(P["poses_init"], P["sb_init"], hf, opts, band=29 if band else None)
        rb = _solve_ref(api, b, P, hf, f, band, opts)
        sa, sb_ = ra["summary"], rb["summary"]
        assert sa.num_iterations == sb_.num_iterations >= 2 and sa.termination == sb_.termination
        # without LiDAR the chain and the prior can be met exactly and the final cost sits at the rounding level (about 1e-14),
        # where only an absolute floor far below it makes sense
        assert abs(sa.final_cost - sb_.final_cost) <= 1e-12 * abs(sb_.final_cost) + 1e-18
        assert np.max(np.abs(ra["poses"] - rb["poses"])) <= 1e-9
        assert np.max(np.abs(ra["speed_bias"] - rb["speed_bias"])) <= 1e-9
        assert sa.final_cost < sa.initial_cost
        if band:                                               # a smaller half_bandwidth hint still covers the chain
            rc = a.window_solve(P["poses_init"], P["sb_init"], hf, opts, band=5)
            assert np.array_equal(rc["poses"], ra["poses"]) and np.array_equal(rc["speed_bias"], ra["speed_bias"])
    finally:
        a.close(); b.close()


def _marg_ref_fn(api, ctx, hf, f, captured):
    """glio_host_marg_fn: hf's marginalisation factors plus the reference ambient blocks of the IMU factors on pair {0, 1}"""
    L = ctx._lib

    def cb(user, W_, p, s, A, b):
        rc = L.glio_hf_marg_evaluate(hf._h, W_, p, s, A, b)
        if rc != 0:
            return rc
        N = 6 * W_ + 18
        pz = np.ctypeslib.as_array(p, (W_ * 7,)).reshape(W_, 7).copy()
        sz = np.ctypeslib.as_array(s, (W_ * 9,)).reshape(W_, 9).copy()
        Ai, _, bi, _ = wr.marg_pair01(pz, sz, f, N)
        Am = np.ctypeslib.as_array(A, (N * N,)).reshape(N, N); bm = np.ctypeslib.as_array(b, (N,))
        Am += Ai; bm += bi
        captured["A"] = Am.copy(); captured["b"] = bm.copy()
        return 0
    return api.HOST_MARG_FN(cb)


def _marg_raw(api, ctx, poses, sb, fn, asynchronous):
    L = ctx._lib
    pb = np.ascontiguousarray(poses, np.float64); sv = np.ascontiguousarray(sb, np.float64); W = len(pb)
    out = C.c_void_p()
    if asynchronous:
        job = C.c_void_p()
        ctx._chk(L.glio_window_marginalize_async(ctx._h, C.c_int(W), api._ptr(pb), api._ptr(sv), fn, None, C.c_double(1e-8), C.byref(job)))
        return api.MargJob(ctx, job, (pb, sv, fn)).wait()
    ctx._chk(L.glio_window_marginalize(ctx._h, C.c_int(W), api._ptr(pb), api._ptr(sv), fn, None, C.c_double(1e-8), C.byref(out)))
    return api.MargPrior(out, L)


@pytest.mark.parametrize("lidar,edges", [(True, False), (True, True), (False, False)])
def test_marginalisation_matches_host_callback(api, problem, lidar, edges):
    P, E = problem
    W = W5; N = 6 * W + 18
    f = api.imu_factor_records(**P["imu"])
    hf = _prior_set(api, P)
    poses, sb = P["poses_init"], P["sb_init"]
    a, b = _ctx(api, P, E, lidar, edges), _ctx(api, P, E, lidar, edges)
    try:
        a.window_set_imu_factors(f); a.window_use_imu_factors(True)
        pa = a.window_marginalize(poses, sb, hf).arrays()
        pq = a.window_marginalize_async(poses, sb, hf).wait().arrays()
        assert all(np.array_equal(pa[k], pq[k]) for k in pa)                 # sync = async, bit for bit
        cap = {}
        rb = _marg_raw(api, b, poses, sb, _marg_ref_fn(api, b, hf, f, cap), False).arrays()
        rq = _marg_raw(api, b, poses, sb, _marg_ref_fn(api, b, hf, f, {}), True).arrays()
        assert all(np.array_equal(rb[k], rq[k]) for k in rb)
        # Tolerance: the device's IMU sums and the reference's agree to KAPPA 2^-53 of their magnitudes (<= 2^-44 max|A|, the
        # eval tests above).  The prior is the Schur complement S = A_kk - A_km A_mm^-1 A_mk, whose change under a change dA of A is
        # bounded by |dA| (1 + |A_km A_mm^-1|)^2 to first order; A_info is S restricted to eigenvalues > 1e-8, none of which sit
        # near the threshold here.  2^-40 leaves a factor 16 over 2^-44 for the decomposition's own rounding.
        A = cap["A"].copy()
        H = b.eval_unary(poses, jac_kind=1)["H"] if lidar else np.zeros((W, 6, 6))
        for k in range(W):
            base = 0 if k == 0 else (15 if k == 1 else 30 + 6 * (k - 2))
            A[base:base + 6, base:base + 6] += H[k]
        if edges:
            He = b.eval_edge_kind(poses, 1)["H"]
            for k in range(W):
                base = 0 if k == 0 else (15 if k == 1 else 30 + 6 * (k - 2))
                A[base:base + 6, base:base + 6] += He[k]
        kappa = (1.0 + np.linalg.norm(A[15:, :15] @ np.linalg.inv(A[:15, :15]), 2)) ** 2
        tol = 2.0 ** -40 * np.max(np.abs(A)) * kappa
        assert np.max(np.abs(pa["A_info"] - rb["A_info"])) <= tol
        assert np.max(np.abs(pa["b_info"] - rb["b_info"])) <= 2.0 ** -40 * (np.max(np.abs(cap["b"])) + np.max(np.abs(A))) * kappa
        assert A.shape == (N, N)
    finally:
        a.close(); b.close()


def test_multi_step_pipelined_run_matches_synchronous(api):
    """W = 20: association, solve, marginalisation and the prior consumed by the next window, three windows; the pipelined run
    (asynchronous marginalisation, the next window's association queued before the wait) equals the synchronous one bit for bit"""
    W, steps = 20, 3
    P = synth.window_imu_problem(W=W + steps - 1, Q=3000, M=60000, seed=81)
    f_all = api.imu_factor_records(**P["imu"])

    def run(pipelined):
        c = api.Context(0); c.set_map(P["map_xyz"]); c.window_use_imu_factors(True)
        hf = _prior_set(api, P)
        poses = P["poses_init"][:W].copy(); sb = P["sb_init"][:W].copy()
        out = []
        c.window_set_scans(P["scans"][:W]); c.window_associate(poses)
        try:
            for s in range(steps):
                f = f_all[s:s + W - 1].copy(); f["i"] -= s; f["j"] -= s
                c.window_set_imu_factors(f)
                r = c.window_solve(poses, sb, hf, band=max(29, hf.marg_half_bandwidth()))
                out += [r["poses"], r["speed_bias"]]
                nxt = np.concatenate([r["poses"][1:], P["poses_init"][s + W:s + W + 1]]) if s + 1 < steps else None
                nsb = np.concatenate([r["speed_bias"][1:], P["sb_init"][s + W:s + W + 1]]) if s + 1 < steps else None
                if pipelined:
                    job = c.window_marginalize_async(r["poses"], r["speed_bias"], hf)
                    if nxt is not None:
                        c.window_set_scans(P["scans"][s + 1:s + 1 + W]); c.window_associate(nxt)
                    prior = job.wait()
                else:
                    prior = c.window_marginalize(r["poses"], r["speed_bias"], hf)
                    if nxt is not None:
                        c.window_set_scans(P["scans"][s + 1:s + 1 + W]); c.window_associate(nxt)
                pr = prior.arrays(); out += [pr[k] for k in sorted(pr)]
                hf = api.HostFactorSet(); hf.set_marg_prior(prior)
                poses, sb = nxt, nsb
        finally:
            c.close()
        return out
    a, b = run(False), run(True)
    assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------------------------
# refusals, and what the switch leaves alone
# ---------------------------------------------------------------------------------------------------------------------------
def test_refusals_and_independent_lists(api, problem):
    P, E = problem
    W = W5
    good = api.imu_factor_records(**P["imu"])
    ctx = _ctx(api, P, E, True, False)
    try:
        ctx.window_set_imu_factors(good)
        ref = ctx.eval_window_imu_factors(P["poses_init"], P["sb_init"], 1)
        pairs = ctx.window_imu_pair_list()
        for field, k, val in [("i", 0, -1), ("j", 3, -2), ("i", 2, 4096), ("j", 2, 2), ("sum_dt", 1, np.nan), ("sqrt_info", 3, np.inf),
                              ("g_vec", 0, -np.inf)]:
            bad = good.copy()
            if bad[field].ndim == 1:
                bad[field][k] = val
            else:
                bad[field][k].flat[-1] = val
            with pytest.raises(api.GlioError):
                ctx.window_set_imu_factors(bad)
        assert ctx._lib.glio_window_set_imu_factors(ctx._h, None, C.c_int64(2)) != 0
        assert all(np.array_equal(x, y) for x, y in zip(ctx.window_imu_pair_list(), pairs))
        again = ctx.eval_window_imu_factors(P["poses_init"], P["sb_init"], 1)
        assert all(np.array_equal(ref[k], again[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
        with pytest.raises(api.GlioError):
            ctx.eval_window_imu_factors(P["poses_init"], P["sb_init"], 2)
        # the batch list and the window list are independent
        assert len(ctx.batch_imu_pair_list()[0]) == 0
        ctx.batch_set_imu_factors(good[:2]); ctx.batch_clear()
        assert all(np.array_equal(x, y) for x, y in zip(ctx.window_imu_pair_list(), pairs))
        ctx.batch_set_imu_factors(good[:2])
        ctx.window_set_imu_factors(good[:1])
        assert len(ctx.batch_imu_pair_list()[0]) == 2 and len(ctx.window_imu_pair_list()[0]) == 1
        ctx.window_slide(W)
        assert len(ctx.window_imu_pair_list()[0]) == 1
        ctx.window_set_imu_factors(good)
        # speed_bias == NULL; a slot >= W
        ctx.window_use_imu_factors(True)
        hf = _prior_set(api, P)
        with pytest.raises(api.GlioError):
            ctx.window_solve(P["poses_init"], None)
        hi = good.copy(); hi["j"][-1] = W                                    # accepted, but W slots are too few
        ctx.window_set_imu_factors(hi)
        for call in (lambda: ctx.eval_window_imu_factors(P["poses_init"], P["sb_init"], 0),
                     lambda: ctx.window_solve(P["poses_init"], P["sb_init"], hf),
                     lambda: ctx.window_solve(P["poses_init"], P["sb_init"], hf, band=29)):
            with pytest.raises(api.GlioError):
                call()
        # a (0, k != 1) factor in the marginalisation; inactive, it takes no part
        odd = good.copy(); odd["j"][0] = 2
        ctx.window_set_imu_factors(odd)
        with pytest.raises(api.GlioError):
            ctx.window_marginalize(P["poses_init"], P["sb_init"], hf)
        with pytest.raises(api.GlioError):
            ctx.window_marginalize_async(P["poses_init"], P["sb_init"], hf)
        odd["active"][0] = 0
        ctx.window_set_imu_factors(odd)
        ctx.window_marginalize(P["poses_init"], P["sb_init"], hf)
    finally:
        ctx.close()


def test_switch_off_or_empty_list_changes_nothing(api, problem):
    P, E = problem
    f = api.imu_factor_records(**P["imu"])
    hf = _prior_set(api, P)
    plain = _ctx(api, P, E, True, True)
    off = _ctx(api, P, E, True, True); off.window_set_imu_factors(f); off.window_use_imu_factors(True); off.window_use_imu_factors(False)
    empty = _ctx(api, P, E, True, True); empty.window_set_imu_factors(f); empty.window_set_imu_factors(f[:0]); empty.window_use_imu_factors(True)
    try:
        def run(c):
            c.lib_profile(True)
            n0 = c.launch_count
            r = c.window_solve(P["poses_init"], P["sb_init"], hf)
            rb = c.window_solve(P["poses_init"], P["sb_init"], hf, band=29)
            m = c.window_marginalize(r["poses"], r["speed_bias"], hf).arrays()
            q = c.window_marginalize_async(r["poses"], r["speed_bias"], hf).wait().arrays()
            n = c.launch_count - n0
            prof = {k: v[1] for k, v in c.lib_profile_read().items()}
            c.lib_profile(False)
            return [r["poses"], r["speed_bias"], r["steps"], rb["poses"], rb["speed_bias"]] + [m[k] for k in sorted(m)] + [q[k] for k in sorted(q)], n, prof
        o0, n0, p0 = run(plain)
        assert not any(k.startswith("k_imu") for k in p0)
        for c in (off, empty):
            o1, n1, p1 = run(c)
            assert n1 == n0 and p1 == p0
            assert all(np.array_equal(x, y) for x, y in zip(o0, o1))
    finally:
        for c in (plain, off, empty):
            c.close()
