"""Edges of the device minimizer (glio_batch_use_device_solver, band.cu):
- glio_band_ops, the scale, shift and product kernels alone, bit-identical to tests/band_solve_reference.py over sizes around the
  launch blocks and up to the level-1 problem, half bandwidths up to GLIO_BAND_BCR_MAX_HB, and scales and vectors spanning 1e+-150;
- K4 at the edges of its shared-memory ring (n from hb+1 to hb+18 and around 2R), with pivot failures in the prologue's rows and
  the last rows, and on the Jacobi-scaled, shifted normal equations the minimizer hands it;
- device solves against host solves (tests/test_gpu_imu_factors.py's _compare) at the shipped options, without Jacobi scaling,
  at K = 2 and 3, with speed-bias at level 0, with edges and with every factor kind at level 1; a host callback that fails
  inside a solve; the refusal of a band wider than GLIO_BAND_MAX_HB; one context reused across shapes."""
import ctypes as C

import numpy as np
import pytest

from glio_b200 import synth
from tests import band_solve_reference as br
from tests.band_refined_reference import backward_error
from tests import eval_reference as er
from tests import test_gpu_device_solve as ds
from tests import test_gpu_imu_factors as ti

pytestmark = pytest.mark.gpu


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


def _differs(a, b):
    return np.argwhere(_bits(a) != _bits(b))[:5].tolist()


# ---------------------------------------------------------------------------------------------------------------------------
# glio_band_ops: k_band_scale, k_band_shift, k_band_symv
# ---------------------------------------------------------------------------------------------------------------------------
HBS = [0, 1, 5, 104, 160, 161, 193, 224, 255, 256]


def _ops_cases():
    out = []
    for hb in HBS:
        for n in sorted({1, 2, 3, hb, hb + 1, 255, 256, 257, 20742, 51855}):
            if n >= 1:
                out.append((n, hb))
    return out


@pytest.mark.parametrize("n,hb", _ops_cases())
def test_band_ops_bit_identical_to_reference(ctx, n, hb):
    rng = np.random.default_rng([n, hb, 3])
    H = br.random_spd_band(n, hb, rng)                       # slots with j < 0 hold NaN
    H[:, :hb] *= rng.uniform(0.0, 1.0, (n, hb)) < 0.8           # some exact zeros inside the band
    s = 10.0 ** rng.uniform(-150, 150, n)
    v = rng.uniform(-1.0, 1.0, n) * 10.0 ** rng.uniform(-150, 150, n)
    x = rng.uniform(-1.0, 1.0, n) * 10.0 ** rng.uniform(-3, 3, n) / s          # spans 1e-150 .. 1e150; Hs x stays finite
    Hs_ref, hd_ref = br.band_scale(H, s)
    A_ref = br.band_shift(Hs_ref, v)
    y_ref = br.band_symv(Hs_ref, x)
    Hs, hd, A, y = ctx.band_ops(H, s, v, x)
    _, _, inside = br._offsets(n, hb)
    assert np.all(np.isfinite(Hs[inside])) and np.all(np.isfinite(A[inside])) and np.all(np.isfinite(hd)) and np.all(np.isfinite(y))
    assert np.array_equal(_bits(Hs[inside]), _bits(Hs_ref[inside])), f"Hs differs at {np.argwhere(inside & (_bits(Hs) != _bits(Hs_ref)))[:5].tolist()}"
    assert np.array_equal(_bits(A[inside]), _bits(A_ref[inside])), f"A differs at {np.argwhere(inside & (_bits(A) != _bits(A_ref)))[:5].tolist()}"
    assert np.array_equal(_bits(hd), _bits(hd_ref)), f"hs_diag differs at {_differs(hd, hd_ref)}"
    assert np.array_equal(_bits(y), _bits(y_ref)), f"y differs at {_differs(y, y_ref)}"


def test_band_ops_launches_and_is_profiled(api, ctx):
    rng = np.random.default_rng(4)
    n, hb = 300, 20
    H = br.random_spd_band(n, hb, rng)
    ctx.lib_profile(True)
    before = ctx.launch_count
    ctx.band_ops(H, np.ones(n), np.ones(n), np.ones(n))
    prof = ctx.lib_profile_read()
    ctx.lib_profile(False)
    assert ctx.launch_count == before + 3
    for k in ("k_band_scale", "k_band_shift", "k_band_symv"):
        assert prof[k][1] == 1 and prof[k][0] > 0.0, k


def test_band_ops_arguments_up_to_bcr_max_hb(api, ctx):
    rng = np.random.default_rng(5)
    with pytest.raises(api.GlioError, match="GLIO_BAND_BCR_MAX_HB"):
        ctx.band_ops(br.random_spd_band(400, api.BAND_BCR_MAX_HB + 1, rng), np.ones(400), np.ones(400), np.ones(400))
    with pytest.raises(api.GlioError, match="n > 0"):
        ctx.band_ops(np.zeros((0, 5)), np.zeros(0), np.zeros(0), np.zeros(0))
    d = np.zeros(40 * 6); p = api._ptr(d)
    assert ctx._lib.glio_band_ops(ctx._h, C.c_int(40), C.c_int(5), p, p, p, None, p, p, p, p) == -3
    assert ctx._lib.glio_band_ops(ctx._h, C.c_int(40), C.c_int(-1), p, p, p, p, p, p, p, p) == -3
    assert ctx._lib.glio_band_ops(None, C.c_int(40), C.c_int(5), p, p, p, p, p, p, p, p) == -3


# ---------------------------------------------------------------------------------------------------------------------------
# K4 at the edges of its ring
# ---------------------------------------------------------------------------------------------------------------------------
def _check_solve(ctx, band, b, what):
    L_ref, _, x_ref, ok_ref = br.band_cholesky_solve(band, b)
    assert ok_ref, what
    L, x, ok = ctx.band_solve(band, b)
    assert ok, what
    assert np.array_equal(_bits(L), _bits(L_ref)), f"{what}: L differs at {_differs(L, L_ref)}"
    assert np.array_equal(_bits(x), _bits(x_ref)), f"{what}: x differs at {_differs(x, x_ref)}"


@pytest.mark.parametrize("hb", [0, 1, 7, 8, 9, 41, 104, 160])
def test_band_solve_at_the_ring_edges(ctx, hb):
    for n in br.ring_edge_sizes(hb):
        rng = np.random.default_rng([hb, n, 1])
        band = br.random_spd_band(n, hb, rng, 6)
        b = rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)
        _check_solve(ctx, band, b, f"hb={hb} n={n}")


@pytest.mark.parametrize("hb", [0, 8, 41, 160])
@pytest.mark.parametrize("where", ["first", "prologue", "last_rows", "last"])
def test_band_solve_pivot_failure_then_recovery(ctx, hb, where):
    R = hb + 1 + br.PREFETCH
    n = 2 * R + 5
    row = {"first": 0, "prologue": 5, "last_rows": n - 5, "last": n - 1}[where]
    rng = np.random.default_rng([hb, row])
    band = br.random_spd_band(n, hb, rng, 3)
    band[row, hb] = -band[row, hb]                 # diagonally dominant: the pivots before `row` stay positive, row's is negative
    b = rng.standard_normal(n)
    L_ref, y_ref, _, ok_ref = br.band_cholesky_solve(band, b)
    assert not ok_ref and np.all(L_ref[:row, hb] > 0)
    L, x, ok = ctx.band_solve(band, b)
    assert not ok
    # the rows before the failing one are final: written back, with y in x
    assert np.array_equal(_bits(L[:row]), _bits(L_ref[:row])) and np.array_equal(_bits(x[:row]), _bits(y_ref[:row]))
    ok_band = br.random_spd_band(n, hb, rng, 6)
    _check_solve(ctx, ok_band, rng.standard_normal(n), f"after a failure at row {row}")


# ---------------------------------------------------------------------------------------------------------------------------
# K4 on the minimizer's own systems
# ---------------------------------------------------------------------------------------------------------------------------
MIN_LM_DIAGONAL, MAX_LM_DIAGONAL, RADIUS = 1e-6, 1e32, 1e4      # glio_default_solver_options, initial_trust_region_radius


def _minimizer_systems(band, g):
    """(name, A, rhs): the band scaled as solve() scales it and shifted as the dogleg (mu from its first 1e-8 to its last 1) and
    LM shift it"""
    s = 1.0 / (1.0 + np.sqrt(band[:, -1]))
    Hs, hd = br.band_scale(band, s)
    gs = g * s
    clamped = np.minimum(np.maximum(hd, MIN_LM_DIAGONAL), MAX_LM_DIAGONAL)
    out = [(f"dogleg mu={mu:g}", br.band_shift(Hs, np.sqrt(clamped) * np.sqrt(mu)), gs) for mu in (1e-8, 1e-4, 1e-1, 1.0)]
    out.append(("lm", br.band_shift(Hs, np.sqrt(clamped / RADIUS)), gs))
    return out


@pytest.mark.parametrize("prior", [True, False])
@pytest.mark.parametrize("level,K", [(0, 40), (0, 200), (0, 3457), (1, 40), (1, 200)])
def test_band_solve_on_the_minimizers_systems(api, ctx, level, K, prior):
    c, P, sb, hf = (ds._level0 if level == 0 else ds._level1)(api, K)
    try:
        band, g, _ = c.batch_normal_equations(P["poses_init"], sb, hf if prior else None, on_device=False)
    finally:
        c.close()
    hb = band.shape[1] - 1
    band[~br._offsets(len(band), hb)[2]] = np.nan             # slots with j < 0: never read
    n_ok = 0
    for name, A, rhs in _minimizer_systems(band, g):
        L_ref, _, x_ref, ok_ref = br.band_cholesky_solve(A, rhs)
        L, x, ok = ctx.band_solve(A, rhs)
        assert ok == ok_ref, name
        if not ok_ref:
            continue
        n_ok += 1
        assert np.array_equal(_bits(L), _bits(L_ref)), f"{name}: L differs at {_differs(L, L_ref)}"
        assert np.array_equal(_bits(x), _bits(x_ref)), f"{name}: x differs at {_differs(x, x_ref)}"
        assert backward_error(A, x_ref, rhs) <= 4 * (hb + 2) * np.finfo(float).eps, name
    assert n_ok >= (3 if prior else 1)


# ---------------------------------------------------------------------------------------------------------------------------
# device solves against host solves
# ---------------------------------------------------------------------------------------------------------------------------
def _raw_solve(api, c, K, poses, sb, fn, user, options, max_log=256):
    """glio_batch_solve as api.Context.batch_solve calls it, but with any callback and options (None: the shipped defaults)"""
    pb = np.array(poses, np.float64).reshape(K, 7).copy()
    sbv = None if sb is None else np.array(sb, np.float64).reshape(K, 9).copy()
    n = K * (15 if sb is not None else 6)
    summ = api.SolverSummary(); log = (api.Iteration * max_log)(); steps = np.zeros((max_log, n))
    rc = c._lib.glio_batch_solve(c._h, C.c_int(K), api._ptr(pb), api._ptr(sbv), fn, user, None if options is None else C.byref(options),
                                 C.byref(summ), log, C.c_int(max_log), api._ptr(steps), C.c_int64(steps.size))
    return rc, dict(poses=pb, speed_bias=sbv, summary=summ, iterations=api.iterations_to_dicts(log, min(summ.num_iterations, max_log)),
                    steps=steps[:summ.num_valid_steps])


def _hf_fn(api, hf):
    return (C.cast(None, api.HOST_FACTORS_BAND_FN), None) if hf is None else (C.cast(api.lib().glio_hf_evaluate_band, api.HOST_FACTORS_BAND_FN), hf._h)


def _both(api, c, P, sb, hf, options):
    out = []
    for on in (False, True):
        c.batch_use_device_solver(on)
        rc, r = _raw_solve(api, c, len(P["poses_init"]), P["poses_init"], sb, *_hf_fn(api, hf), options)
        assert rc == 0, c._lib.glio_last_error(c._h)
        out.append(r)
    return out


def _level0_sb(api, K):
    c, P, _, _ = ds._level0(api, K)
    hf = api.HostFactorSet()
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], np.zeros(9), np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.ones(9)]))
    return c, P, np.zeros((K, 9)), hf


def _level0_small(api, K):
    """level 0 at K = 2 or 3: no DD factor reaches so few keyframes, and the pose factors alone fit the prior exactly (the final cost
    is rounding).  A second prior 5 cm off on the last keyframe keeps a cost that the relative criterion can compare."""
    c, P, sb, hf = ds._level0(api, K)
    hf.add_prior(K - 1, P["poses_true"][K - 1, :3] + 0.05, P["poses_true"][K - 1, 3:], None,
                 np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.zeros(9)]))
    return c, P, sb, hf


def _level1_all(api, K):
    """level 1 with LiDAR pairs, attitude, DD pseudorange and IMU factors"""
    c, P, sb, hf = ds._level1(api, K)
    D = synth.dd_psr_problem(K=K, seed=synth.SEED0 + 18)          # imu_problem's trajectory
    c.batch_set_dd_psr_factors(api.dd_psr_factor_records(**D["dd"]), api.dd_psr_sat_records(**D["dd_sats"]), D["R"], D["anchor"])
    c.batch_use_dd_psr_factors(True)
    return c, P, sb, hf


SOLVES = {
    "defaults_level0": (lambda api: ds._level0(api, 40), None),
    "defaults_level1": (lambda api: ds._level1(api, 40), None),
    "no_jacobi_level0": (lambda api: ds._level0(api, 40), dict(jacobi_scaling=0, max_num_iterations=10)),
    "no_jacobi_level1": (lambda api: ds._level1(api, 40), dict(jacobi_scaling=0, max_num_iterations=10)),
    "K2_level0": (lambda api: _level0_small(api, 2), dict(max_num_iterations=10)),
    "K3_level0": (lambda api: _level0_small(api, 3), dict(max_num_iterations=10)),
    "K2_level1": (lambda api: ds._level1(api, 2), dict(max_num_iterations=10)),
    "K3_level1": (lambda api: ds._level1(api, 3), dict(max_num_iterations=10)),
    "speed_bias_level0": (lambda api: _level0_sb(api, 40), dict(max_num_iterations=10)),
    "edges_level1": (lambda api: ds._level1(api, 40, edges=True), dict(max_num_iterations=10)),
    "pose_dd_imu_level1": (lambda api: _level1_all(api, 40), dict(max_num_iterations=10)),
}


@pytest.mark.parametrize("case", list(SOLVES))
def test_device_solve_matches_host(api, case):
    make, opt = SOLVES[case]
    c, P, sb, hf = make(api)
    try:
        K = len(P["poses_init"])
        if case.startswith("K"):           # the whole system inside K4's ring: hb = n - 1
            band = c.batch_normal_equations(P["poses_init"], sb, hf)[0]
            assert band.shape[1] == band.shape[0] == K * (15 if sb is not None else 6)
        rh, rd = _both(api, c, P, sb, hf, None if opt is None else api.batch_solver_options(**opt))
        ti._compare(rd, rh)
        if opt is None:
            assert rh["summary"].num_iterations <= 100
    finally:
        c.close()


class _FailingCallback:
    """glio_hf_evaluate_band behind a HOST_FACTORS_BAND_FN that returns -1 at its fail_at-th call (1-based; 0: never) and records
    every call's want_jac"""

    def __init__(self, api, hf, fail_at=0):
        self.hf, self.fail_at, self.calls = hf, fail_at, []
        lib = api.lib()

        def cb(user, K, p, s, want_jac, H, hb, g, cost):
            self.calls.append(int(want_jac))
            if len(self.calls) == self.fail_at:
                return -1
            return lib.glio_hf_evaluate_band(self.hf._h, K, p, s, want_jac, H, hb, g, cost)
        self.fn = api.HOST_FACTORS_BAND_FN(cb)


@pytest.mark.parametrize("where", ["candidate", "accepted_point"])
def test_failing_callback_ends_both_paths_alike(api, where):
    fuse = 1 if where == "candidate" else 0
    opt = api.batch_solver_options(max_num_iterations=10, fuse_candidate_jacobian=fuse)
    c, P, sb, hf = ds._level0(api, 40)
    try:
        K = len(P["poses_init"])
        probe = _FailingCallback(api, hf)
        rc, r0 = _raw_solve(api, c, K, P["poses_init"], sb, probe.fn, None, opt)
        assert rc == 0 and r0["summary"].termination != 2 and len(probe.calls) >= 3
        if where == "candidate":
            fail_at = 3                                         # the second candidate (fused: every call evaluates Jacobians)
        else:
            jac = [k + 1 for k, w in enumerate(probe.calls) if w]
            assert len(jac) >= 3 and probe.calls[1] == 0
            fail_at = jac[2]                                    # the re-evaluation of the second accepted point
        out = []
        for on in (False, True):
            c.batch_use_device_solver(on)
            cb = _FailingCallback(api, hf, fail_at)
            rc, r = _raw_solve(api, c, K, P["poses_init"], sb, cb.fn, None, opt)
            assert rc == 0 and len(cb.calls) >= fail_at
            out.append(r)
        rh, rd = out
        sh, sd = rh["summary"], rd["summary"]
        assert sh.termination == sd.termination == (2 if where == "accepted_point" else sh.termination)
        if where == "candidate":
            assert sh.termination != 2
            # the failed candidate is a rejected step with cost = max
            assert any(not it["step_is_successful"] and it["cost"] == np.finfo(float).max for it in rh["iterations"])
            assert any(not it["step_is_successful"] and it["cost"] == np.finfo(float).max for it in rd["iterations"])
        assert sh.num_iterations == sd.num_iterations >= 1
        assert [it["step_is_successful"] for it in rh["iterations"]] == [it["step_is_successful"] for it in rd["iterations"]]
        assert abs(sh.final_cost - sd.final_cost) <= 1e-9 * abs(sh.final_cost)
        assert np.max(np.abs(rh["poses"][:, :3] - rd["poses"][:, :3])) <= 1e-7
        assert np.max(np.abs(rh["poses"][:, 3:] - rd["poses"][:, 3:])) <= 1e-8
        assert not np.array_equal(rh["poses"], P["poses_init"])
    finally:
        c.close()


def test_too_wide_band_is_refused_and_leaves_the_context_usable(api):
    """an attitude factor 12 keyframes apart at level 1: hb = 13 * 15 - 1 = 194 > GLIO_BAND_MAX_HB"""
    K = 40
    c, P, sb, hf = ds._level1(api, K)
    fresh, _, _, _ = ds._level1(api, K)
    try:
        pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
        wide = np.concatenate([pf, pf[:1]])
        wide["i"][-1], wide["j"][-1] = 3, 15
        c.batch_set_pose_factors(wide)
        assert c.batch_normal_equations(P["poses_init"], sb, hf)[0].shape[1] - 1 == 194
        c.batch_use_device_solver(True)
        poses = np.array(P["poses_init"], np.float64).copy(); sbv = np.array(sb, np.float64).copy()
        summ = api.SolverSummary(); log = (api.Iteration * 16)(); steps = np.zeros((16, K * 15))
        rc = c._lib.glio_batch_solve(c._h, C.c_int(K), api._ptr(poses), api._ptr(sbv), *_hf_fn(api, hf),
                                     C.byref(api.batch_solver_options(max_num_iterations=6)), C.byref(summ), log, C.c_int(16),
                                     api._ptr(steps), C.c_int64(steps.size))
        assert rc == -3 and b"GLIO_BAND_MAX_HB" in c._lib.glio_last_error(c._h)
        assert np.array_equal(_bits(poses), _bits(P["poses_init"])) and np.array_equal(_bits(sbv), _bits(sb))
        c.batch_set_pose_factors(pf)
        fresh.batch_use_device_solver(True)
        opt = api.batch_solver_options(max_num_iterations=6)
        ra = c.batch_solve(P["poses_init"], sb, hf, opt)
        rb = fresh.batch_solve(P["poses_init"], sb, hf, opt)
        _bit_identical(ra, rb)
    finally:
        c.close(); fresh.close()


def _bit_identical(ra, rb):
    assert np.array_equal(_bits(ra["poses"]), _bits(rb["poses"])) and np.array_equal(_bits(ra["steps"]), _bits(rb["steps"]))
    assert ra["summary"].num_iterations == rb["summary"].num_iterations and ra["summary"].termination == rb["summary"].termination
    log = lambda r: np.array([[float(v) for v in it.values()] for it in r["iterations"]])
    assert np.array_equal(_bits(log(ra)), _bits(log(rb)))
    if ra["speed_bias"] is not None:
        assert np.array_equal(_bits(ra["speed_bias"]), _bits(rb["speed_bias"]))


def _configure(api, c, level, K):
    """c cleared and given the problem ds._level0 / ds._level1 build on a fresh context (same lists, matches and switches)"""
    c.batch_clear(); c.batch_use_edges(False)
    if level == 0:
        P = synth.dd_psr_problem(K=K)
        c.batch_set_dd_psr_factors(api.dd_psr_factor_records(**P["dd"]), api.dd_psr_sat_records(**P["dd_sats"]), P["R"], P["anchor"])
        c.batch_use_dd_psr_factors(True)
        c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
        hf = api.HostFactorSet()
        hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], None, np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.zeros(9)]))
        return P, None, hf
    P = synth.imu_problem(K=K)
    cur, oth = (np.asarray(v) for v in P["pairs"])
    keep = np.abs(cur - oth) <= 6
    cur, oth = cur[keep], oth[keep]
    rng = np.random.default_rng(3)                               # tp._pairs_ctx's matches
    c.batch_declare_pairs(cur, oth)
    for a, b in zip(cur, oth):
        m = er.make_pair(rng, P["poses_true"][a], P["poses_true"][b], 40, noise=0.02)
        c.batch_set_pair_matches(int(a), int(b), m["cp"], m["nc"], m["weight"])
    c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
    c.batch_set_imu_factors(api.imu_factor_records(**P["imu"])); c.batch_use_imu_factors(True)
    return P, P["sb_init"], ti._host_factor_set(api, P)


def test_one_context_across_shapes_equals_fresh_contexts(api):
    c = api.Context(0)
    try:
        c.batch_use_device_solver(True)
        opt = api.batch_solver_options(max_num_iterations=5)
        for level, K in ((0, 200), (1, 40), (0, 2), (1, 200), (0, 200)):
            P, sb, hf = _configure(api, c, level, K)
            ra = c.batch_solve(P["poses_init"], sb, hf, opt)
            f = api.Context(0)
            try:
                f.batch_use_device_solver(True)
                Pf, sbf, hff = _configure(api, f, level, K)
                rb = f.batch_solve(Pf["poses_init"], sbf, hff, opt)
            finally:
                f.close()
            assert ra["summary"].num_iterations >= 1, (level, K)
            _bit_identical(ra, rb)
    finally:
        c.close()
