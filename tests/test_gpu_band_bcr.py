"""The band solve by block cyclic reduction: glio_band_solve_bcr against tests/band_bcr_reference.py over one to many blocks, half
bandwidths 0 to 256 and sizes around block multiples (x within 1e-11 of the reference on well-conditioned bands, the normwise
backward error within 1e-14 on all, the same failures, the same bits from call to call and context to context, argument checks);
and the device minimizer with GLIO_FACTOR_BCR against the host path under tests/test_gpu_imu_factors.py's _compare criteria, up to
the 3 457-keyframe sample run and at the half bandwidth 194 that K4 refuses."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth
from tests import band_bcr_reference as bcr
from tests import band_solve_reference as br
from tests import test_gpu_device_solve as ds
from tests import test_gpu_imu_factors as ti
from tests import test_gpu_pose_factors as tp
from tests.test_band_bcr_reference import HBS, sizes

pytestmark = pytest.mark.gpu
XTOL = 1e-11
BOUND = 1e-14


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


@pytest.fixture(scope="module")
def ctx(api):
    c = api.Context(0)
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _check(ctx, band, rhs, well_conditioned):
    x, ok = ctx.band_solve_bcr(band, rhs)
    xr, okr = bcr.bcr_solve(band, rhs)
    assert ok and okr
    assert bcr.backward_error(band, x, rhs) <= BOUND
    if well_conditioned:
        assert np.max(np.abs(x - xr)) <= XTOL * np.max(np.abs(xr))
    return x


@pytest.mark.parametrize("scale_exp", [0.0, 6.0])
@pytest.mark.parametrize("hb", HBS)
def test_band_solve_bcr_matches_reference(ctx, hb, scale_exp):
    rng = np.random.default_rng([hb, int(scale_exp), 7])
    for n in sizes(hb):
        band = br.random_spd_band(n, hb, rng, scale_exp=scale_exp)
        _check(ctx, band, rng.normal(size=n), scale_exp == 0.0)


@pytest.mark.parametrize("nt,span", [(6, 6), (15, 6), (15, 12), (15, 16)])
def test_band_solve_bcr_on_block_bands(ctx, nt, span):
    rng = np.random.default_rng([nt, span, 7])
    for K in (span + 1, 3 * (span + 1) + 1, 40, 200):
        band = br.block_band(K, nt, span, rng)
        _check(ctx, band, rng.normal(size=band.shape[0]), True)


@pytest.mark.parametrize("hb", [41, 104, 194, 256])
def test_band_solve_bcr_at_full_size(ctx, hb):
    rng = np.random.default_rng([hb, 51855])
    n = 20742 if hb == 41 else 51855
    band = br.random_spd_band(n, hb, rng)
    _check(ctx, band, rng.normal(size=n), True)


@pytest.mark.parametrize("hb", [5, 41, 194])
def test_failures_match_reference_and_leave_the_context_usable(api, ctx, hb):
    rng = np.random.default_rng(hb + 11)
    b = bcr.block_size(hb)
    n = 5 * b + 3
    band = br.random_spd_band(n, hb, rng)
    rhs = rng.normal(size=n)
    fresh = api.Context(0)
    try:
        for row in (0, 2 * b + 7, n - 1):
            for val in (-abs(band[row, hb]) * 1e3, np.nan):
                bad = band.copy(); bad[row, hb] = val
                assert ctx.band_solve_bcr(bad, rhs)[1] == bcr.bcr_solve(bad, rhs)[1] == False   # noqa: E712
        x, ok = ctx.band_solve_bcr(band, rhs)
        xf, okf = fresh.band_solve_bcr(band, rhs)
        assert ok and okf and np.array_equal(_bits(x), _bits(xf))
    finally:
        fresh.close()


def test_bit_identical_across_calls_and_contexts(api, ctx):
    rng = np.random.default_rng(3)
    other = api.Context(0)
    try:
        for hb, n in ((41, 20742), (194, 9000), (256, 3000)):
            band = br.random_spd_band(n, hb, rng); rhs = rng.normal(size=n)
            x1, _ = ctx.band_solve_bcr(band, rhs); x2, _ = ctx.band_solve_bcr(band, rhs); x3, _ = other.band_solve_bcr(band, rhs)
            assert np.array_equal(_bits(x1), _bits(x2)) and np.array_equal(_bits(x1), _bits(x3))
    finally:
        other.close()


def test_bad_arguments_are_refused(api, ctx):
    L = api.lib()
    x = np.zeros(600); ok = C.c_int(0)
    band = np.ones((600, 258)); rhs = np.ones(600)
    assert L.glio_band_solve_bcr(ctx._h, C.c_int(600), C.c_int(257), api._ptr(band), api._ptr(rhs), api._ptr(x), C.byref(ok)) == -3
    assert L.glio_band_solve_bcr(ctx._h, C.c_int(0), C.c_int(5), api._ptr(band), api._ptr(rhs), api._ptr(x), C.byref(ok)) == -3
    assert L.glio_band_solve_bcr(ctx._h, C.c_int(600), C.c_int(-1), api._ptr(band), api._ptr(rhs), api._ptr(x), C.byref(ok)) == -3
    assert L.glio_batch_device_factorization(ctx._h, C.c_int(2)) == -3
    band = br.random_spd_band(600, 20, np.random.default_rng(0))
    assert ctx.band_solve_bcr(band, rhs)[1]


def test_kernel_names_are_profiled(api, ctx):
    ctx.lib_profile(True)
    try:
        ctx.band_solve_bcr(br.random_spd_band(500, 41, np.random.default_rng(1)), np.ones(500))
        prof = ctx.lib_profile_read()
    finally:
        ctx.lib_profile(False)
    for k in ("k_bcr_gather", "k_bcr_potrf", "k_bcr_trsm", "k_bcr_update", "k_bcr_back", "k_bcr_finish"):
        assert k in prof and prof[k][1] > 0, k


# ---- the device minimizer with GLIO_FACTOR_BCR

def _solve(api, c, P, sb, hf, on, bcr_kind=True, **opt):
    c.batch_use_device_solver(on)
    c.batch_device_factorization(api.FACTOR_BCR if bcr_kind else api.FACTOR_SEQUENTIAL)
    return c.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(**opt))


def _level1_all_pairs(api, K):
    """synth.imu_problem with all of its LiDAR pairs (up to 12 keyframes apart: hb = 13 * 15 - 1 = 194)"""
    P = synth.imu_problem(K=K)
    c = tp._pairs_ctx(api, P, K)
    c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
    c.batch_set_imu_factors(api.imu_factor_records(**P["imu"])); c.batch_use_imu_factors(True)
    return c, P, P["sb_init"], ti._host_factor_set(api, P)


@pytest.mark.parametrize("fuse", [0, 1])
@pytest.mark.parametrize("strategy", ["dogleg", "subspace", "lm"])
@pytest.mark.parametrize("level,K", [(0, 40), (0, 200), (1, 40), (1, 200)])
def test_bcr_solve_matches_host(api, level, K, strategy, fuse):
    opt = dict(max_num_iterations=10, fuse_candidate_jacobian=fuse,
               trust_region_strategy=1 if strategy == "lm" else 0, dogleg_type=1 if strategy == "subspace" else 0)
    c, P, sb, hf = (ds._level0 if level == 0 else ds._level1)(api, K)
    try:
        rh = _solve(api, c, P, sb, hf, False, **opt)
        rd = _solve(api, c, P, sb, hf, True, **opt)
        ti._compare(rd, rh)
    finally:
        c.close()


@pytest.mark.parametrize("level", [0, 1])
def test_bcr_solve_full_size(api, level):
    c, P, sb, hf = (ds._level0 if level == 0 else ds._level1)(api, 3457)
    try:
        rh = _solve(api, c, P, sb, hf, False, max_num_iterations=10)
        rd = _solve(api, c, P, sb, hf, True, max_num_iterations=10)
        ti._compare(rd, rh)
    finally:
        c.close()


def test_bcr_solve_with_wide_attitude_factor(api):
    """an attitude factor 12 keyframes apart at level 1: hb = 194, which K4 refuses"""
    K = 40
    c, P, sb, hf = ds._level1(api, K)
    try:
        pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
        wide = np.concatenate([pf, pf[:1]])
        wide["i"][-1], wide["j"][-1] = 3, 15
        c.batch_set_pose_factors(wide)
        assert c.batch_normal_equations(P["poses_init"], sb, hf)[0].shape[1] - 1 == 194
        rh = _solve(api, c, P, sb, hf, False, max_num_iterations=10)
        rd = _solve(api, c, P, sb, hf, True, max_num_iterations=10)
        ti._compare(rd, rh)
    finally:
        c.close()


def test_bcr_solve_with_all_lidar_pairs(api):
    c, P, sb, hf = _level1_all_pairs(api, 200)
    try:
        assert c.batch_normal_equations(P["poses_init"], sb, hf)[0].shape[1] - 1 == 194
        rh = _solve(api, c, P, sb, hf, False, max_num_iterations=10)
        rd = _solve(api, c, P, sb, hf, True, max_num_iterations=10)
        ti._compare(rd, rh)
    finally:
        c.close()


def test_bcr_solve_without_gauge_prior(api):
    """no prior: the normal equations are singular up to the shift; poses stay finite and no accepted step raises the cost"""
    c, P, sb, _ = ds._level0(api, 40)
    try:
        r = _solve(api, c, P, sb, None, True, max_num_iterations=8, use_nonmonotonic_steps=0)
        assert np.all(np.isfinite(r["poses"])) and r["summary"].final_cost <= r["summary"].initial_cost
        accepted = [it["cost"] for it in r["iterations"] if it["iteration"] == 0 or it["step_is_successful"]]
        assert all(b <= a for a, b in zip(accepted, accepted[1:])), accepted
    finally:
        c.close()


def test_bcr_solve_is_deterministic(api):
    c, P, sb, hf = ds._level1(api, 200)
    try:
        r1 = _solve(api, c, P, sb, hf, True, max_num_iterations=6)
        r2 = _solve(api, c, P, sb, hf, True, max_num_iterations=6)
        assert np.array_equal(_bits(r1["poses"]), _bits(r2["poses"])) and np.array_equal(_bits(r1["steps"]), _bits(r2["steps"]))
    finally:
        c.close()


def test_kind_round_trip_and_switch_off_change_nothing(api):
    """BCR and back to sequential: the launches and results of a fresh context; with the device solver off the kind is ignored"""
    a, P, sb, hf = ds._level1(api, 40)
    b, _, _, _ = ds._level1(api, 40)
    try:
        opt = api.batch_solver_options(max_num_iterations=6)
        b.batch_device_factorization(api.FACTOR_BCR); b.batch_device_factorization(api.FACTOR_SEQUENTIAL)
        for on in (True, False):
            a.batch_use_device_solver(on); b.batch_use_device_solver(on)
            la, lb = a.launch_count, b.launch_count
            ra = a.batch_solve(P["poses_init"], sb, hf, opt); rb = b.batch_solve(P["poses_init"], sb, hf, opt)
            assert a.launch_count - la == b.launch_count - lb
            assert np.array_equal(_bits(ra["poses"]), _bits(rb["poses"])) and np.array_equal(_bits(ra["steps"]), _bits(rb["steps"]))
        b.batch_device_factorization(api.FACTOR_BCR)       # device solver off: the host path whatever the kind
        la, lb = a.launch_count, b.launch_count
        ra = a.batch_solve(P["poses_init"], sb, hf, opt); rb = b.batch_solve(P["poses_init"], sb, hf, opt)
        assert a.launch_count - la == b.launch_count - lb
        assert np.array_equal(_bits(ra["poses"]), _bits(rb["poses"])) and np.array_equal(_bits(ra["steps"]), _bits(rb["steps"]))
    finally:
        a.close(); b.close()


def test_minimizer_profiles_bcr_kernels(api):
    c, P, sb, hf = ds._level0(api, 40)
    try:
        c.lib_profile(True)
        _solve(api, c, P, sb, hf, True, max_num_iterations=2)
        prof = c.lib_profile_read(); c.lib_profile(False)
        assert "k_bcr_potrf" in prof and "k_band_chol_solve" not in prof and "k_band_shift" not in prof
    finally:
        c.close()
