"""Edges of the band solve by block cyclic reduction (glio_band_solve_bcr, GLIO_FACTOR_BCR; bcr.cu) on the systems it is given,
held to tests/band_refined_reference.py's extended-precision solution.  With eps = 2^-53 and b BCR's block size, every solve that
reports ok meets the backward-error bar ||b - A x||_inf / (||A||_inf ||x||_inf + ||b||_inf) <= 4 (b + 2) eps and the forward-error
bar ||x - x_ref||_inf / ||x_ref||_inf <= 4 (b + 2) eps kappa, kappa = cond_estimate (tests/test_band_refined_reference.py
calibrates both on the numpy restatement):
- a. ill-conditioned bands that are not diagonally dominant (factor_band, gauge_band) at kappa 1 .. 1e12, half bandwidths on
  either side of every tile multiple up to 256, n from 1 to 16 b + 1; K4 on the same bands up to hb 160, and the two agree;
- b. indefinite bands whose diagonal blocks are all positive definite: BCR, K4 and the restatement all fail, and the context's
  next solve is a fresh context's bit for bit;
- c. the minimizer's own Jacobi-scaled, shifted normal equations, levels 0 and 1 up to K = 3 457, with and without the gauge
  prior, at half bandwidths 194 and 254;
- d. the device minimizer's BCR step bit for bit against glio_band_solve_bcr on the shifted band (k_bcr_gather's v * v term,
  at the default trust-region radius and at radius 1);
- f. the minimizer's refusal of a band wider than GLIO_BAND_BCR_MAX_HB;
- g. more blocks than one launch can take along y (m > 2 * 65 535);
- h. one context across block counts, half bandwidths and a minimizer solve, equal to fresh contexts bit for bit.
The device normal equations and glio_band_ops at half bandwidths 161 .. 256 are in tests/test_gpu_device_solve.py and
tests/test_gpu_band_device_edges.py.  Each group's largest error over its bar is printed at the end of the module (pytest -s)."""
import ctypes as C
import time

import numpy as np
import pytest

from tests import band_bcr_reference as bcr
from tests import band_refined_reference as rr
from tests import band_solve_reference as br
from tests import test_gpu_device_solve as ds
from tests.test_band_bcr_reference import sizes
from tests.test_band_refined_reference import make
from tests.test_gpu_band_bcr import _level1_all_pairs
from tests.test_gpu_band_device_edges import _bit_identical, _hf_fn, _minimizer_systems

pytestmark = pytest.mark.gpu
EPS = rr.EPS
HBS = [0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 160, 161, 193, 194, 223, 224, 225, 255, 256]
KAPPAS = [1.0, 1e4, 1e8, 1e12]
WORST = {}                                          # group -> [largest backward error / bar, largest forward error / bar]


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


@pytest.fixture(scope="module")
def ctx(api):
    c = api.Context(0)
    yield c
    c.close()
    for g, (be, fe) in sorted(WORST.items()):
        print(f"\n[bcr edges] group {g}: largest backward error {be:.3g} of its bar, forward error {fe:.3g} of its bar")


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _bar(hb):
    return 4 * (bcr.block_size(hb) + 2) * EPS


def _meets_bars(group, A, rhs, x, x_ref, kappa, what):
    """x's backward error against A, and its forward error against x_ref (when given), within the bars; records the ratios"""
    hb = A.shape[1] - 1
    be = rr.backward_error(A, x, rhs) / _bar(hb)
    w = WORST.setdefault(group, [0.0, 0.0])
    w[0] = max(w[0], be)
    assert be <= 1.0, f"{what}: backward error {be:.3g} of the bar"
    if x_ref is not None:
        fe = np.max(np.abs(x - x_ref)) / np.max(np.abs(x_ref)) / (_bar(hb) * kappa)
        w[1] = max(w[1], fe)
        assert fe <= 1.0, f"{what}: forward error {fe:.3g} of the bar (kappa {kappa:.3g})"


# ---------------------------------------------------------------------------------------------------------------------------
# a. ill-conditioned bands
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["factor", "gauge"])
@pytest.mark.parametrize("hb", HBS)
def test_ill_conditioned_bands(ctx, hb, kind):
    rng = np.random.default_rng([hb, len(kind), 41])
    for n in sorted({1, 2, max(hb, 1), hb + 1} | set(sizes(hb))):
        for kappa in KAPPAS:
            what = f"{kind} hb={hb} n={n} kappa={kappa:g}"
            A = make(kind, n, hb, rng, kappa)
            rhs = rng.normal(size=n)
            x_ref, conv = rr.refined_solve(A, rhs)
            k = rr.cond_estimate(A)
            assert conv, what
            x, ok = ctx.band_solve_bcr(A, rhs)
            assert ok, what
            _meets_bars("a", A, rhs, x, x_ref, k, what)
            if hb <= 160:
                _, x4, ok4 = ctx.band_solve(A, rhs)
                assert ok4, what
                _meets_bars("a", A, rhs, x4, x_ref, k, what + " (K4)")
                assert np.max(np.abs(x - x4)) <= _bar(hb) * k * np.max(np.abs(x_ref)), what


# ---------------------------------------------------------------------------------------------------------------------------
# b. failures
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", rr.SCHUR_WHERE)
@pytest.mark.parametrize("hb", [1, 33, 129, 194, 256])
def test_indefinite_bands_fail_everywhere(api, ctx, hb, where):
    rng = np.random.default_rng([hb, len(where), 43])
    b = bcr.block_size(hb)
    fresh = api.Context(0)
    try:
        for n in (5 * b + 1, 8 * b - 1):
            A = rr.schur_indefinite_band(n, hb, rng, where)
            rhs = rng.normal(size=n)
            lam = np.linalg.eigvalsh(br.band_to_dense(np.nan_to_num(A)))[0]
            near = abs(lam) <= 100 * n * EPS * rr.norm1(A)
            x, ok = ctx.band_solve_bcr(A, rhs)
            assert not bcr.bcr_solve(A, rhs)[1] or near
            if ok:
                assert near, f"n={n}: BCR reports ok on a band with lambda_min = {lam:.3g}"
                _meets_bars("b", A, rhs, x, None, np.inf, f"n={n}")
            if hb <= 160:
                _, x4, ok4 = ctx.band_solve(A, rhs)
                assert not ok4 or near
            good = make("factor", n, hb, rng, 1e8)
            x1, ok1 = ctx.band_solve_bcr(good, rhs)
            xf, okf = fresh.band_solve_bcr(good, rhs)
            assert ok1 and okf and np.array_equal(_bits(x1), _bits(xf))
    finally:
        fresh.close()


# ---------------------------------------------------------------------------------------------------------------------------
# c. the minimizer's own systems
# ---------------------------------------------------------------------------------------------------------------------------
def _level1_hb254(api, K):
    """level 1 with a pose factor 16 keyframes apart: hb = 17 * 15 - 1 = 254"""
    return ds.with_pose_factor(api, ds._level1(api, K), 3, 19)


PROBLEMS = {f"level{lv}_K{K}": (lambda api, lv=lv, K=K: (ds._level0 if lv == 0 else ds._level1)(api, K))
            for lv in (0, 1) for K in (40, 200, 3457)}
PROBLEMS["level1_all_pairs_hb194"] = lambda api: _level1_all_pairs(api, 200)
PROBLEMS["level1_hb254"] = lambda api: _level1_hb254(api, 40)


@pytest.mark.parametrize("prior", [True, False])
@pytest.mark.parametrize("problem", list(PROBLEMS))
def test_minimizers_systems(api, ctx, problem, prior):
    c, P, sb, hf = PROBLEMS[problem](api)
    try:
        band, g, _ = c.batch_normal_equations(P["poses_init"], sb, hf if prior else None, on_device=False)
    finally:
        c.close()
    hb = band.shape[1] - 1
    assert hb == {"level1_all_pairs_hb194": 194, "level1_hb254": 254}.get(problem, hb)
    band[~br._offsets(len(band), hb)[2]] = np.nan
    n_ok = 0
    for name, A, rhs in _minimizer_systems(band, g):
        what = f"{problem} prior={prior} {name}"
        k = rr.cond_estimate(A)
        x, ok = ctx.band_solve_bcr(A, rhs)
        assert ok or k * EPS >= 1e-3, f"{what}: BCR fails at kappa {k:.3g}"
        if not ok:
            continue
        n_ok += 1
        x_ref, conv = rr.refined_solve(A, rhs) if k * EPS < 1e-3 else (None, False)
        _meets_bars("c", A, rhs, x, x_ref if conv else None, k, what)
        if hb <= 160 and conv:
            _, x4, ok4 = ctx.band_solve(A, rhs)
            assert ok4, what
            assert np.max(np.abs(x - x4)) <= _bar(hb) * k * np.max(np.abs(x_ref)), what
    assert n_ok >= (4 if prior else 1)


# ---------------------------------------------------------------------------------------------------------------------------
# d. the minimizer's BCR path, bit for bit
# ---------------------------------------------------------------------------------------------------------------------------
LM_PROBLEMS = {"level0_hb41": (lambda api: ds._level0(api, 40), 41),
               "level1_hb104": (lambda api: ds._level1(api, 40), 104),
               "level1_hb194": (lambda api: ds.with_pose_factor(api, ds._level1(api, 40), 3, 15), 194),
               "level1_hb254": (lambda api: _level1_hb254(api, 40), 254)}


@pytest.mark.parametrize("radius", [1e4, 1.0])
@pytest.mark.parametrize("problem", list(LM_PROBLEMS))
def test_minimizer_lm_step_is_the_shifted_bcr_solve(api, ctx, problem, radius):
    """one LM iteration's logged step is (-x) * s, x = glio_band_solve_bcr(band_shift(band_scale(H, s), v), g * s),
    s = 1 / (1 + sqrt(diag H)), v = sqrt(clamp(diag Hs) / radius): lm_compute_step and the step log (solver.cpp).  At the
    default radius v * v is 1e-4 of the diagonal it shifts, so its rounding rarely reaches the sum; at radius 1 it is as large as
    the diagonal, and a shift rounded once (a fused multiply-add) changes x."""
    make_problem, hb_want = LM_PROBLEMS[problem]
    c, P, sb, hf = make_problem(api)
    try:
        H, g, _ = c.batch_normal_equations(P["poses_init"], sb, hf, on_device=False)
        assert H.shape[1] - 1 == hb_want
        opt = api.batch_solver_options(trust_region_strategy=1, max_num_iterations=1, initial_trust_region_radius=radius)
        s = 1.0 / (1.0 + np.sqrt(H[:, -1]))
        Hs, hd = br.band_scale(H, s)
        v = np.sqrt(np.minimum(np.maximum(hd, opt.min_lm_diagonal), opt.max_lm_diagonal) / opt.initial_trust_region_radius)
        x, ok = ctx.band_solve_bcr(br.band_shift(Hs, v), g * s)
        assert ok
        c.batch_use_device_solver(True)
        c.batch_device_factorization(api.FACTOR_BCR)
        r = c.batch_solve(P["poses_init"], sb, hf, opt)
        assert r["iterations"][1]["step_is_valid"] == 1 and len(r["steps"]) == 1
        want = (-x) * s
        assert np.array_equal(_bits(r["steps"][0]), _bits(want)), np.argwhere(_bits(r["steps"][0]) != _bits(want))[:5].tolist()
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------------
# f. refusal above GLIO_BAND_BCR_MAX_HB
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level,K,i,j,hb", [(0, 200, 3, 45, 257), (1, 40, 3, 20, 269)])
def test_minimizer_refuses_bands_wider_than_bcr_takes(api, level, K, i, j, hb):
    make_problem = ds._level0 if level == 0 else ds._level1
    c, P, sb, hf = ds.with_pose_factor(api, make_problem(api, K), i, j)
    fresh, _, _, _ = make_problem(api, K)
    try:
        assert c.batch_normal_equations(P["poses_init"], sb, hf)[0].shape[1] - 1 == hb
        c.batch_use_device_solver(True)
        c.batch_device_factorization(api.FACTOR_BCR)
        poses = np.array(P["poses_init"], np.float64).copy()
        sbv = None if sb is None else np.array(sb, np.float64).copy()
        n = K * (15 if sb is not None else 6)
        summ = api.SolverSummary(); log = (api.Iteration * 16)(); steps = np.zeros((16, n))
        rc = c._lib.glio_batch_solve(c._h, C.c_int(K), api._ptr(poses), api._ptr(sbv), *_hf_fn(api, hf),
                                     C.byref(api.batch_solver_options(max_num_iterations=6)), C.byref(summ), log, C.c_int(16),
                                     api._ptr(steps), C.c_int64(steps.size))
        assert rc == -3 and b"GLIO_BAND_BCR_MAX_HB" in c._lib.glio_last_error(c._h)
        assert np.array_equal(_bits(poses), _bits(P["poses_init"]))
        if sb is not None:
            assert np.array_equal(_bits(sbv), _bits(sb))
        c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"]))
        fresh.batch_use_device_solver(True)
        fresh.batch_device_factorization(api.FACTOR_BCR)
        opt = api.batch_solver_options(max_num_iterations=6)
        _bit_identical(c.batch_solve(P["poses_init"], sb, hf, opt), fresh.batch_solve(P["poses_init"], sb, hf, opt))
    finally:
        c.close(); fresh.close()


# ---------------------------------------------------------------------------------------------------------------------------
# g. more blocks than one launch takes along y
# ---------------------------------------------------------------------------------------------------------------------------
def _launches(m):
    """glio_band_solve_bcr's launches for m blocks: the gather; per level (L = ceil(log2 m) of them) k_bcr_potrf, then k_bcr_trsm
    and k_bcr_update in one launch per 65 535 blocks along y; the last block's potrf and trsm; L + 1 back-substitutions; the finish"""
    out, s = 1, 1
    while s < m:
        ml = -(-m // s)
        out += 1 + -(-(ml // 2) // 65535) + -(-((ml + 1) // 2) // 65535)
        s *= 2
    return out + 2 + (s.bit_length()) + 1


@pytest.mark.parametrize("hb", [1, 5])
def test_more_blocks_than_one_launch_takes(api, hb):
    """n = 4 227 073, b = 32: m = 132 097 blocks, so level 0 eliminates 66 048 and updates 66 049 (> 65 535 CTAs along y).  About
    3.3 GB of workspace.  A small solve on the same context afterwards equals a fresh context's."""
    n = 4227073
    assert -(-n // bcr.block_size(hb)) == 132097
    rng = np.random.default_rng([hb, 47])
    A = make("factor", n, hb, rng, 1e4)
    rhs = rng.normal(size=n)
    c = api.Context(0)
    fresh = api.Context(0)
    try:
        l0, t0 = c.launch_count, time.perf_counter()
        x, ok = c.band_solve_bcr(A, rhs)
        t1 = time.perf_counter()
        assert ok and c.launch_count - l0 == _launches(132097) == 4 * 18 + 5 + 2
        l0 = c.launch_count
        assert c.band_solve_bcr(A[:320], rhs[:320])[1] and c.launch_count - l0 == _launches(10) == 4 * 4 + 5
        x_ref, conv = rr.refined_solve(A, rhs)
        assert conv
        _meets_bars("g", A, rhs, x, x_ref, rr.cond_estimate(A), f"hb={hb} n={n}")
        print(f"\n[bcr edges] hb={hb} n={n}: glio_band_solve_bcr {t1 - t0:.2f} s (with the band's upload)")
        small = make("factor", 300, hb, rng, 1e8)
        xs, oks = c.band_solve_bcr(small, rhs[:300])
        xf, okf = fresh.band_solve_bcr(small, rhs[:300])
        assert oks and okf and np.array_equal(_bits(xs), _bits(xf))
    finally:
        c.close(); fresh.close()


# ---------------------------------------------------------------------------------------------------------------------------
# h. one context across shapes
# ---------------------------------------------------------------------------------------------------------------------------
def test_one_context_across_shapes_equals_fresh_contexts(api):
    """glio_band_solve_bcr at many blocks, few blocks, other half bandwidths and many blocks again, with a BCR minimizer solve in
    between, all on one context (one BCR workspace): every result equals a fresh context's bit for bit"""
    rng = np.random.default_rng(53)
    cases = [(200001, 5), (100, 5), (3000, 194), (300000, 33), (70, 256)]
    bands = [(make("factor", n, hb, rng, 1e6), rng.normal(size=n)) for n, hb in cases]
    c, P, sb, hf = ds._level1(api, 40)
    f, _, _, _ = ds._level1(api, 40)
    try:
        opt = api.batch_solver_options(max_num_iterations=5)
        for ctx_ in (c, f):
            ctx_.batch_use_device_solver(True); ctx_.batch_device_factorization(api.FACTOR_BCR)
        rb = f.batch_solve(P["poses_init"], sb, hf, opt)
        for k, (A, rhs) in enumerate(bands):
            x, ok = c.band_solve_bcr(A, rhs)
            g = api.Context(0)
            try:
                xf, okf = g.band_solve_bcr(A, rhs)
            finally:
                g.close()
            assert ok and okf and np.array_equal(_bits(x), _bits(xf)), cases[k]
            if k in (1, 3):                         # the minimizer after a small and after a large block count
                _bit_identical(c.batch_solve(P["poses_init"], sb, hf, opt), rb)
    finally:
        c.close(); f.close()
