"""K2i on the device: glio_eval_imu_factors within the a-priori bound of the longdouble reference (tests/imu_factor_reference.py),
the argument checks of glio_batch_set_imu_factors, glio_batch_solve with the IMU factors on against the same problem with the IMU
blocks handed in through the band host callback, and what the switch must leave alone when it is off."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth
from tests import eval_reference as er
from tests import imu_factor_reference as ir
from tests import test_gpu_pose_factors as tp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _quirky(P, seed):
    """P's initial states with non-unit and w < 0 quaternions, 20 km offsets, Bg_i away from linearized_bg, and its IMU columns with
    every other factor's i and j swapped"""
    rng = np.random.default_rng(seed)
    K = len(P["poses_init"])
    poses = P["poses_init"].copy(); sb = P["sb_init"].copy()
    poses[:, 3:] *= rng.uniform(0.7, 1.4, (K, 1)); poses[1::3, 3:] *= -1.0
    poses[:, :3] += np.array([20_000.0, -12_000.0, 150.0])
    sb[:, 6:] += rng.normal(0.0, 0.01, (K, 3))
    cols = dict(P["imu"]); i, j = cols["i"].copy(), cols["j"].copy()
    cols["i"] = np.where(np.arange(len(i)) % 2 == 1, j, i); cols["j"] = np.where(np.arange(len(i)) % 2 == 1, i, j)
    return poses, sb, cols


def _check(ctx, poses, sb, f):
    ctx.batch_set_imu_factors(f)
    a, b = ctx.batch_imu_pair_list()
    ref = ir.imu_blocks(poses, sb, f)
    assert list(zip(a.tolist(), b.tolist())) == ref["pairs"]
    d = ctx.eval_imu_factors(poses, sb)
    er.assert_within(d["Hdiag"], ref["Hdiag"], ref["MHdiag"], "Hdiag")
    er.assert_within(d["g"], ref["g"], ref["Mg"], "g")
    if len(a):
        er.assert_within(d["Hoff"], ref["Hoff"], ref["MHoff"], "Hoff")
    er.assert_within(d["cost"], ref["cost"], ref["Mcost"], "cost")
    c = ctx.eval_imu_factors(poses, sb, want_jac=False)                       # the cost-only kernel
    er.assert_within(c["cost"], ref["cost"], ref["Mcost"], "cost without Jacobians")
    return d


@pytest.mark.parametrize("K", [2, 7, 40, 200, 3457])
def test_eval_matches_reference(api, K):
    P = synth.imu_problem(K=K)
    ctx = api.Context(0)
    try:
        _check(ctx, P["poses_init"], P["sb_init"], api.imu_factor_records(**P["imu"]))
        poses, sb, cols = _quirky(P, K)
        _check(ctx, poses, sb, api.imu_factor_records(**cols))
        assert len(ctx.batch_imu_pair_list()[0]) == K - 1
    finally:
        ctx.close()


def test_eval_duplicates_inactive_and_empty(api):
    K = 12
    P = synth.imu_problem(K=K, seed=11)
    poses, sb, cols = _quirky(P, 4)
    f = api.imu_factor_records(**cols)
    n0 = len(f)
    f = np.concatenate([f, f[:5], f[3:4], f[3:4]])                             # several factors on one pair, in two orientations
    f["i"][-1], f["j"][-1] = f["j"][-1], f["i"][-1]
    f["active"][[2, n0 + 2, len(f) - 2]] = 0                                   # inactive factors; pair 2 evaluates nothing
    ctx = api.Context(0)
    try:
        d = _check(ctx, poses, sb, f)
        assert np.all(d["Hoff"][2] == 0.0)
        _check(ctx, poses, sb, f[::-1].copy())                                 # another order inside the pairs
        ctx.batch_set_imu_factors(f[:0])
        assert len(ctx.batch_imu_pair_list()[0]) == 0
        e = ctx.eval_imu_factors(poses, sb)
        assert np.all(e["Hdiag"] == 0) and np.all(e["g"] == 0) and e["cost"] == 0.0
    finally:
        ctx.close()


def test_argument_checks_keep_the_previous_list(api):
    K = 10
    P = synth.imu_problem(K=K, seed=12)
    good = api.imu_factor_records(**P["imu"])
    ctx = api.Context(0)
    try:
        ctx.batch_set_imu_factors(good)
        ref = ctx.eval_imu_factors(P["poses_init"], P["sb_init"])
        pairs = ctx.batch_imu_pair_list()
        bads = [("i", 0, -1), ("j", 3, -2), ("i", 7, api.IMU_MAX_KF), ("j", 2, 2), ("sum_dt", 1, np.nan), ("sum_dt", 4, np.inf),
                ("sqrt_info", 5, np.nan), ("delta_q", 6, -np.inf), ("dv_dbg", 8, np.nan), ("g_vec", 0, np.inf)]
        for field, k, val in bads:
            bad = good.copy()
            if bad[field].ndim == 1:
                bad[field][k] = val
            else:
                bad[field][k].flat[-1] = val
            with pytest.raises(api.GlioError):
                ctx.batch_set_imu_factors(bad)
        assert ctx._lib.glio_batch_set_imu_factors(ctx._h, None, C.c_int64(3)) != 0
        assert all(np.array_equal(x, y) for x, y in zip(ctx.batch_imu_pair_list(), pairs))
        again = ctx.eval_imu_factors(P["poses_init"], P["sb_init"])
        assert all(np.array_equal(ref[k], again[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
        # speed_bias is required by the evaluation and, with the switch on, by the solve
        pb = np.ascontiguousarray(P["poses_init"])
        assert ctx._lib.glio_eval_imu_factors(ctx._h, C.c_int(K), api._ptr(pb), None, None, None, None, None) != 0
        ctx.batch_use_imu_factors(True)
        with pytest.raises(api.GlioError):
            ctx.batch_solve(P["poses_init"], None, options=api.batch_solver_options(max_num_iterations=2))
        hi = good.copy(); hi["j"][-1] = K                                      # accepted, but K keyframes are too few
        ctx.batch_set_imu_factors(hi)
        with pytest.raises(api.GlioError):
            ctx.eval_imu_factors(P["poses_init"], P["sb_init"])
        with pytest.raises(api.GlioError):
            ctx.batch_solve(P["poses_init"], P["sb_init"], options=api.batch_solver_options(max_num_iterations=2))
        ctx.batch_clear()
        assert len(ctx.batch_imu_pair_list()[0]) == 0
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the batch solve
# ---------------------------------------------------------------------------------------------------------------------------
def _host_factor_set(api, P):
    """a prior on keyframe 0 (pose and speed-bias) fixes the gauge"""
    hf = api.HostFactorSet()
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)])
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], P["sb_true"][0], sw * 3)
    return hf


def _solve_with_imu_callback(api, ctx, P, hf, f, max_iter):
    """glio_batch_solve with host factors = hf + the reference's IMU blocks (rounded to float64), written into the 15-column band"""
    L = ctx._lib
    pb = np.array(P["poses_init"], np.float64).copy(); K = len(pb)
    sbv = np.array(P["sb_init"], np.float64).copy()
    nt = 15
    pairs = np.array(ir.pair_table(f)[0], np.int32).reshape(-1, 2)
    ctx.batch_declare_pairs(pairs[:, 0], pairs[:, 1])                        # pairs without matches: the IMU pairs' bandwidth

    def cb(user, Kc, p, s, want_jac, H, hb, g, cost):
        rc = L.glio_hf_evaluate_band(hf._h, Kc, p, s, want_jac, H, hb, g, cost)
        if rc != 0:
            return rc
        pz = np.ctypeslib.as_array(p, (Kc * 7,)).reshape(Kc, 7).copy()
        sz = np.ctypeslib.as_array(s, (Kc * 9,)).reshape(Kc, 9).copy()
        e = ir.imu_blocks(pz, sz, f)
        cost[0] = cost[0] + e["cost"]
        if want_jac:
            w = hb + 1
            band = np.ctypeslib.as_array(H, (Kc * nt * w,)).reshape(Kc * nt, w)
            gv = np.ctypeslib.as_array(g, (Kc * nt,))
            for k in range(Kc):
                for i in range(15):
                    band[nt * k + i, hb - i:hb + 1] += e["Hdiag"][k, i, :i + 1]
                gv[nt * k:nt * k + 15] += e["g"][k]
            for p_, (a, b) in enumerate(e["pairs"]):
                for y in range(15):
                    i = nt * b + y
                    band[i, nt * a - i + hb:nt * a + 15 - i + hb] += e["Hoff"][p_][:, y]
        return 0
    fn = api.HOST_FACTORS_BAND_FN(cb)
    opt = api.batch_solver_options(max_num_iterations=max_iter)
    summ = api.SolverSummary(); log = (api.Iteration * 64)(); n = K * nt; steps = np.zeros((64, n))
    ctx._chk(L.glio_batch_solve(ctx._h, C.c_int(K), api._ptr(pb), api._ptr(sbv), fn, None, C.byref(opt), C.byref(summ), log,
                                C.c_int(64), api._ptr(steps), C.c_int64(steps.size)))
    return dict(poses=pb, speed_bias=sbv, summary=summ, iterations=api.iterations_to_dicts(log, min(summ.num_iterations, 64)))


def _compare(ra, rb):
    sa, sb_ = ra["summary"], rb["summary"]
    assert sa.num_iterations == sb_.num_iterations >= 2 and sa.termination == sb_.termination
    assert [it["step_is_successful"] for it in ra["iterations"]] == [it["step_is_successful"] for it in rb["iterations"]]
    assert abs(sa.final_cost - sb_.final_cost) <= 1e-9 * abs(sb_.final_cost)
    assert np.max(np.abs(ra["poses"][:, :3] - rb["poses"][:, :3])) <= 1e-7
    assert sa.final_cost < sa.initial_cost


@pytest.mark.parametrize("pose,lidar,dd", [(True, True, False), (False, True, False), (True, False, False), (True, False, True)])
def test_solve_with_imu_factors_matches_host_callback(api, pose, lidar, dd):
    K = 40
    P = synth.imu_problem(K=K)
    if not lidar:
        del P["pairs"]
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    f = api.imu_factor_records(**P["imu"])
    hf = _host_factor_set(api, P)
    a = tp._pairs_ctx(api, P, K); b = tp._pairs_ctx(api, P, K)
    try:
        for c in (a, b):
            if pose:
                c.batch_set_pose_factors(pf); c.batch_use_pose_factors(True)
            if dd:
                D = synth.dd_psr_problem(K=K, seed=synth.SEED0 + 18)             # imu_problem's trajectory
                c.batch_set_dd_psr_factors(api.dd_psr_factor_records(**D["dd"]), api.dd_psr_sat_records(**D["dd_sats"]), D["R"], D["anchor"])
                c.batch_use_dd_psr_factors(True)
        a.batch_set_imu_factors(f); a.batch_use_imu_factors(True)
        ra = a.batch_solve(P["poses_init"], P["sb_init"], hf, api.batch_solver_options(max_num_iterations=8))
        rb = _solve_with_imu_callback(api, b, P, hf, f, 8)
        _compare(ra, rb)
    finally:
        a.close(); b.close()


def test_switch_off_or_empty_list_changes_nothing(api):
    K = 40
    P = synth.imu_problem(K=K)
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    f = api.imu_factor_records(**P["imu"])
    hf = _host_factor_set(api, P)

    def make():
        c = tp._pairs_ctx(api, P, K); c.batch_set_pose_factors(pf); c.batch_use_pose_factors(True)
        return c
    plain = make()
    off = make(); off.batch_set_imu_factors(f); off.batch_use_imu_factors(True); off.batch_use_imu_factors(False)
    empty = make(); empty.batch_set_imu_factors(f); empty.batch_set_imu_factors(f[:0]); empty.batch_use_imu_factors(True)
    try:
        opts = api.batch_solver_options(max_num_iterations=6)
        for sb in (None, P["sb_init"]):
            n0 = plain.launch_count
            r0 = plain.batch_solve(P["poses_init"], sb, hf, opts)
            d0 = plain.launch_count - n0
            for c in (off, empty):
                c.lib_profile(True)
                n1 = c.launch_count
                r1 = c.batch_solve(P["poses_init"], sb, hf, opts)
                assert c.launch_count - n1 == d0
                assert not any(k.startswith("k_imu") for k in c.lib_profile_read())
                c.lib_profile(False)
                assert np.array_equal(r0["poses"], r1["poses"]) and np.array_equal(r0["steps"], r1["steps"])
        e0 = plain.eval_binary(P["poses_init"]); p0 = plain.eval_pose_factors(P["poses_init"])
        on = make(); on.batch_set_imu_factors(f); on.batch_use_imu_factors(True)
        try:
            for c in (off, empty, on):                                       # the LiDAR and pose evaluations never add IMU blocks
                e1 = c.eval_binary(P["poses_init"]); p1 = c.eval_pose_factors(P["poses_init"])
                assert all(np.array_equal(e0[k], e1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
                assert all(np.array_equal(p0[k], p1[k]) for k in ("Hdiag", "Hoff", "g", "cost"))
        finally:
            on.close()
    finally:
        for c in (plain, off, empty):
            c.close()
