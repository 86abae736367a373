"""glio_batch_use_device_solver: the batch minimizer's band algebra on the device.  glio_batch_normal_equations on the device equals
the host path bit for bit (band, g, cost); glio_batch_solve with the switch on meets tests/test_gpu_imu_factors.py's _compare
criteria against the host path over the three strategies and both fuse_candidate_jacobian settings; two device solves are
bit-identical; with the switch off a context launches and returns exactly what a context that never turned it on does."""
import numpy as np
import pytest

from glio_b200 import synth
from tests import test_gpu_imu_factors as ti
from tests import test_gpu_pose_factors as tp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _level0(api, K, pairs=True):
    P = synth.dd_psr_problem(K=K)
    c = api.Context(0)
    c.batch_set_dd_psr_factors(api.dd_psr_factor_records(**P["dd"]), api.dd_psr_sat_records(**P["dd_sats"]), P["R"], P["anchor"])
    c.batch_use_dd_psr_factors(True)
    c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
    hf = api.HostFactorSet()
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], None, np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.zeros(9)]))
    return c, P, None, hf


def _level1(api, K, pairs=True, edges=False):
    P = synth.imu_problem(K=K)
    if not pairs:
        del P["pairs"]
    else:
        # the generator's LiDAR pairs reach 12 keyframes; the device factorisation takes a half bandwidth up to 160, so keep the
        # pairs within the attitude factors' search range of 6 (half bandwidth 104 at 15 columns per keyframe)
        cur, oth = (np.asarray(v) for v in P["pairs"])
        keep = np.abs(cur - oth) <= 6
        P["pairs"] = (cur[keep], oth[keep])
    c = tp._pairs_ctx(api, P, K, edges=edges)
    c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
    c.batch_set_imu_factors(api.imu_factor_records(**P["imu"])); c.batch_use_imu_factors(True)
    return c, P, P["sb_init"], ti._host_factor_set(api, P)


def with_pose_factor(api, made, i, j):
    """made = (c, P, sb, hf) with one more pose factor, a copy of the first, between keyframes i and j: it sets the half bandwidth
    to (j - i + 1) nt - 1"""
    c, P, sb, hf = made
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    wide = np.concatenate([pf, pf[:1]])
    wide["i"][-1], wide["j"][-1] = i, j
    c.batch_set_pose_factors(wide)
    return c, P, sb, hf


CASES = {"level0": lambda api: _level0(api, 40), "level1": lambda api: _level1(api, 40),
         "level1_edges": lambda api: _level1(api, 40, edges=True), "level1_no_pairs": lambda api: _level1(api, 40, pairs=False),
         # half bandwidths the device minimizer takes only with GLIO_FACTOR_BCR: 251 at level 0 (a pose factor 41 keyframes apart),
         # 194 and 254 at level 1 (12 and 16 apart)
         "level0_hb251": lambda api: with_pose_factor(api, _level0(api, 200), 3, 44),
         "level1_hb194": lambda api: with_pose_factor(api, _level1(api, 40), 3, 15),
         "level1_hb254": lambda api: with_pose_factor(api, _level1(api, 40), 3, 19)}


@pytest.mark.parametrize("callback", [True, False])
@pytest.mark.parametrize("case", list(CASES))
def test_normal_equations_on_device_equal_host(api, case, callback):
    c, P, sb, hf = CASES[case](api)
    try:
        rng = np.random.default_rng(1)
        for x in (P["poses_init"], P["poses_init"] + np.concatenate([rng.normal(0, 0.01, (len(P["poses_init"]), 3)),
                                                                    np.zeros((len(P["poses_init"]), 4))], axis=1)):
            h = c.batch_normal_equations(x, sb, hf if callback else None, on_device=False)
            d = c.batch_normal_equations(x, sb, hf if callback else None, on_device=True)
            assert np.array_equal(_bits(h[0]), _bits(d[0])) and np.array_equal(_bits(h[1]), _bits(d[1])) and h[2] == d[2]
    finally:
        c.close()


def _solve(api, c, P, sb, hf, on, **opt):
    c.batch_use_device_solver(on)
    return c.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(**opt))


@pytest.mark.parametrize("fuse", [0, 1])
@pytest.mark.parametrize("strategy", ["dogleg", "subspace", "lm"])
@pytest.mark.parametrize("level,K", [(0, 40), (0, 200), (1, 40), (1, 200)])
def test_device_solve_matches_host(api, level, K, strategy, fuse):
    opt = dict(max_num_iterations=10, fuse_candidate_jacobian=fuse,
               trust_region_strategy=1 if strategy == "lm" else 0, dogleg_type=1 if strategy == "subspace" else 0)
    c, P, sb, hf = (_level0 if level == 0 else _level1)(api, K)
    try:
        rh = _solve(api, c, P, sb, hf, False, **opt)
        rd = _solve(api, c, P, sb, hf, True, **opt)
        ti._compare(rd, rh)
    finally:
        c.close()


def test_device_solve_without_gauge_prior_escalates_like_host(api):
    c, P, sb, _ = _level0(api, 40)
    try:
        opt = dict(max_num_iterations=5)
        rh = _solve(api, c, P, sb, None, False, **opt); rd = _solve(api, c, P, sb, None, True, **opt)
        assert rh["summary"].num_linear_solves == rd["summary"].num_linear_solves
        assert [it["mu"] for it in rh["iterations"]] == [it["mu"] for it in rd["iterations"]]
        assert rh["summary"].num_iterations == rd["summary"].num_iterations
    finally:
        c.close()


@pytest.mark.parametrize("level", [0, 1])
def test_device_solve_full_size(api, level):
    c, P, sb, hf = (_level0 if level == 0 else _level1)(api, 3457)
    try:
        rh = _solve(api, c, P, sb, hf, False, max_num_iterations=10)
        rd = _solve(api, c, P, sb, hf, True, max_num_iterations=10)
        ti._compare(rd, rh)
    finally:
        c.close()


def test_device_solve_is_deterministic(api):
    c, P, sb, hf = _level1(api, 200)
    try:
        r1 = _solve(api, c, P, sb, hf, True, max_num_iterations=6)
        r2 = _solve(api, c, P, sb, hf, True, max_num_iterations=6)
        assert np.array_equal(_bits(r1["poses"]), _bits(r2["poses"])) and np.array_equal(_bits(r1["steps"]), _bits(r2["steps"]))
    finally:
        c.close()


def test_switch_off_changes_nothing(api):
    a, P, sb, hf = _level1(api, 40)
    b, _, _, _ = _level1(api, 40)
    try:
        b.batch_use_device_solver(True); b.batch_use_device_solver(False)
        la, lb = a.launch_count, b.launch_count
        ra = a.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=6))
        rb = b.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=6))
        assert a.launch_count - la == b.launch_count - lb
        assert np.array_equal(_bits(ra["poses"]), _bits(rb["poses"])) and np.array_equal(_bits(ra["steps"]), _bits(rb["steps"]))
    finally:
        a.close(); b.close()
