"""The device edge selection (glio_select_random_edges, glio_batch_select_random_edges) against the plane rules of
tests/select_reference.py at Philox domains 3, 4 and 5, bit for bit; what the evaluation, solve and marginalisation make of it
(equal to a second context given the copied-out subsets); its independence from the plane selection; and its argument checks."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch  # noqa: F401  (first: torch binds its bundled CUDA runtime before libglio_b200.so loads)

from glio_b200 import dist, synth
from tests import edge_select_reference as es

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "workers", "batch_edge_select_shard_worker.py")

# F - 1 .. F + 2 at F = 100, around the R' clamp (n - F < R': n up to F + R = 400), R' = n - 1 for small n
WINDOW_SIZES = [0, 1, 2, 99, 100, 101, 102, 103, 299, 300, 301, 302, 399, 400, 401, 402, 1000, 4096, 4097, 4098, 20_000]
# B - 1 .. B + 2 at B = 25, 49 / 50 / 51 (start/end), around the BR' clamp (n - B < BR': n up to B + BR = 425)
BATCH_SIZES = [0, 1, 24, 25, 26, 27, 49, 50, 51, 52, 400, 424, 425, 426, 427, 3000]


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


def _fake_edges(rng, n):
    return (rng.normal(size=(n, 3)).astype(np.float32), rng.normal(size=(n, 3)).astype(np.float32),
            rng.normal(size=(n, 3)).astype(np.float32), rng.uniform(0.5, 1.0, n))


def _window_edge_ctx(api, sizes, seed=0):
    ctx = api.Context(0)
    rng = np.random.default_rng(seed)
    big = _fake_edges(rng, max(sizes))
    for k, n in enumerate(sizes):
        if n > 0:
            ctx.set_edges(k, *(a[:n] for a in big))
    return ctx


def _check_window(ctx, counts, ids, opt, na):
    for k, n in enumerate(counts):
        keep, _ = es.window_select(int(n), int(ids[k]), opt.seed, opt.nonce, F=opt.feature_res_num, R=opt.rand_set_num,
                                   random_select=bool(opt.random_select))
        got = ctx.get_edge_selection(k)
        if keep is None:
            assert got is None and na[k] == n, (k, n)
        else:
            assert got is not None and got.tolist() == keep, (k, n)
            assert na[k] == len(keep)


@pytest.mark.parametrize("W", [1, 20, 64])
def test_window_edge_selection_bit_exact(api, W):
    sizes = [WINDOW_SIZES[(k * 7 + W) % len(WINDOW_SIZES)] for k in range(W)] if W > 1 else [20_000]
    ctx = _window_edge_ctx(api, sizes, seed=W)
    ids = np.arange(W, dtype=np.int64) + 1000
    for opt in (api.select_default_options(seed=11, nonce=3), api.select_default_options(feature_res_num=7, rand_set_num=2, seed=5),
                api.select_default_options(feature_res_num=4096, seed=1), api.select_default_options(random_select=0),
                api.select_default_options(feature_res_num=300, rand_set_num=90, seed=2**64 - 1, nonce=2**40 + 7)):
        l0 = ctx.launch_count
        na = ctx.select_random_edges(ids, opt)
        assert ctx.launch_count - l0 <= 1
        _check_window(ctx, sizes, ids, opt, na)
        assert [ctx.get_edges(k)["n"] for k in range(W)] == sizes           # the full list stays readable
    ctx.close()


def test_window_every_size_once_and_the_gathered_records(api):
    ctx = _window_edge_ctx(api, WINDOW_SIZES, seed=3)
    ids = np.arange(len(WINDOW_SIZES), dtype=np.int64) * 3 + 5
    opt = api.select_default_options(seed=9, nonce=4)
    na = ctx.select_random_edges(ids, opt)
    _check_window(ctx, WINDOW_SIZES, ids, opt, na)
    # the evaluation reads exactly the selected records in draw order: a context given them as its lists agrees bit for bit
    W = len(WINDOW_SIZES)
    poses = np.tile(np.array([0.1, -0.2, 0.3, 1.0, 0.0, 0.0, 0.0]), (W, 1))
    ref = api.Context(0)
    for k in range(W):
        _upload_subset(ctx, ref, k, ctx.get_edge_selection(k))
    for kind in (0, 1):
        a, b = ctx.eval_edge_kind(poses, kind), ref.eval_edge_kind(poses, kind)
        assert all(np.array_equal(a[x], b[x]) for x in ("H", "g", "cost"))
    ctx.close(); ref.close()


def test_window_real_association_at_bench_shape(api):
    E = synth.window_edge_problem(W=20, Q=10_000, M=200_000)
    ctx = api.Context(0)
    ctx.set_edge_map(E["map_xyz"])
    for k in range(20):
        ctx.window_set_edge_scan(k, E["scans"][k])
    ne = ctx.window_associate_edges(E["poses_init"])
    assert ne.min() > 101
    ids = np.arange(20, dtype=np.int64) + 77
    for opt in (api.select_default_options(seed=5, nonce=1), api.select_default_options(feature_res_num=4096, seed=6)):
        na = ctx.select_random_edges(ids, opt)
        _check_window(ctx, ne, ids, opt, na)
    assert (ctx.select_random_edges(ids, seed=1) == 100).all()
    ctx.close()


def _batch_edge_ctx(api, cur, oth, sizes, seed=0):
    ctx = api.Context(0)
    rng = np.random.default_rng(seed)
    big = _fake_edges(rng, int(max(sizes)))
    for c, o, n in zip(cur, oth, sizes):
        ctx.batch_set_pair_edges(int(c), int(o), *(a[:n] for a in big))
    return ctx


@pytest.fixture(scope="module")
def cfg3(api):
    """cfg 3's pair list (200 keyframes, search range 6: 2 400 pairs) with about 9 000 edges per pair and every threshold size"""
    cur, oth = dist.batch_pairs(200, 6)
    rng = np.random.default_rng(23)
    sizes = rng.integers(8000, 10_000, len(cur))
    sizes[::7] = np.array(BATCH_SIZES)[rng.integers(0, len(BATCH_SIZES), len(sizes[::7]))]
    ctx = _batch_edge_ctx(api, cur, oth, sizes, seed=4)
    yield ctx, cur, oth, sizes
    ctx.close()


def _check_batch(ctx, cur, oth, sizes, mode, opt, na):
    ref = es.batch_select(list(zip(cur.tolist(), oth.tolist())), list(sizes), mode, opt.seed, opt.nonce,
                          B=opt.batch_feature_res_num, BR=opt.batch_rand_set_num)
    for i, (c, o) in enumerate(zip(cur, oth)):
        keep, _ = ref[i]
        got = ctx.batch_get_edge_selection(int(c), int(o))
        if keep is None:
            assert got is None and na[i] == sizes[i], (i, sizes[i])
        else:
            assert got.tolist() == keep, (i, sizes[i])
            assert na[i] == len(keep)
    return ref


@pytest.mark.parametrize("mode", [0, 1])
def test_cfg3_pairs_in_one_launch_bit_exact(api, cfg3, mode):
    ctx, cur, oth, sizes = cfg3
    for opt in (api.select_default_options(seed=7, nonce=mode * 4 + 1),
                api.select_default_options(batch_feature_res_num=50, batch_rand_set_num=60, seed=3)):
        l0 = ctx.launch_count
        na = ctx.batch_select_random_edges(cur, oth, mode, opt)
        assert ctx.launch_count - l0 == 1
        ref = _check_batch(ctx, cur, oth, sizes, mode, opt, na)
        assert sum(k is not None for k, _ in ref) > 800
        if mode == 0 and opt.batch_feature_res_num == 25:
            assert any(u for _, u in ref), "the undefined size n = 50 is among the pairs"
            assert any(k is None and n >= 50 for (k, _), n in zip(ref, sizes)), "a `return` reaches later pairs of its keyframe"


def test_batch_threshold_sizes_each_alone(api):
    cur = np.zeros(len(BATCH_SIZES), np.int32) + np.arange(len(BATCH_SIZES), dtype=np.int32)
    oth = cur + 100
    ctx = _batch_edge_ctx(api, cur, oth, BATCH_SIZES, seed=6)
    for mode in (0, 1):
        opt = api.select_default_options(seed=12, nonce=mode)
        na = ctx.batch_select_random_edges(cur, oth, mode, opt)
        _check_batch(ctx, cur, oth, BATCH_SIZES, mode, opt, na)
    ctx.close()


# ---- evaluation and solves read the selected subset ---------------------------------------------------------------------------

def _upload_subset(src, dst, k, keep):
    e = src.get_edges(k)
    idx = np.arange(e["n"]) if keep is None else keep
    if len(idx):
        dst.set_edges(k, e["cp"][idx], e["pa"][idx], e["pb"][idx], e["s"][idx])
    else:
        dst.set_edges(k, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros(0))


W = 4


@pytest.fixture(scope="module")
def window(api):
    P = synth.window_problem(W=W, Q=3000, M=40000, seed=31)
    E = synth.window_edge_problem(W=W, Q=1500, M=40000, seed=32)
    ctxs = []
    for edges in (True, False):
        c = api.Context(0)
        c.set_map(P["map_xyz"]); c.window_set_scans(P["scans"]); c.window_associate(P["poses_init"])
        if edges:
            c.set_edge_map(E["map_xyz"])
            for k in range(W):
                c.window_set_edge_scan(k, E["scans"][k])
            assert c.window_associate_edges(P["poses_init"]).min() > 100
        ctxs.append(c)
    a, b = ctxs
    ids = np.array([40, 41, 42, 43], np.int64)
    popt = api.select_default_options(seed=21, nonce=6)
    eopt = api.select_default_options(feature_res_num=60, seed=21, nonce=6)
    assert (a.select_random(ids, popt) == 100).all()
    assert (a.select_random_edges(ids, eopt) == 60).all()
    for k in range(W):
        b.select(k, a.get_selection(k))
        _upload_subset(a, b, k, a.get_edge_selection(k))
    yield P, E, a, b, ids
    for c in ctxs:
        c.close()


def test_window_eval_solve_marginalize_equal_subset_input(api, window):
    P, _, a, b, _ = window
    for kind in (0, 1):
        ea, eb = a.eval_edge_kind(P["poses_init"], kind), b.eval_edge_kind(P["poses_init"], kind)
        assert all(np.array_equal(ea[x], eb[x]) for x in ("H", "g", "cost"))
    ea, eb = a.eval_edge(P["poses_init"]), b.eval_edge(P["poses_init"])
    assert all(np.array_equal(ea[x], eb[x]) for x in ("H", "g", "cost"))
    try:
        for c in (a, b):
            c.window_use_edges(True)
        ra, rb = a.window_solve(P["poses_init"]), b.window_solve(P["poses_init"])
        assert ra["summary"].num_iterations > 1
        assert np.array_equal(ra["poses"], rb["poses"]) and np.array_equal(ra["steps"], rb["steps"])
        assert ra["summary"].initial_cost == rb["summary"].initial_cost
        sb = np.zeros((W, 9))
        pa, pb = a.window_marginalize(ra["poses"], sb).arrays(), b.window_marginalize(rb["poses"], sb).arrays()
        qa, qb = a.window_marginalize_async(ra["poses"], sb).wait().arrays(), b.window_marginalize_async(rb["poses"], sb).wait().arrays()
        for x in ("lin_jac", "lin_res", "x0_pose", "A_info", "b_info"):
            assert np.array_equal(pa[x], pb[x]) and np.array_equal(qa[x], pa[x]) and np.array_equal(qb[x], pb[x])
    finally:
        for c in (a, b):
            c.window_use_edges(False)


def test_window_selection_independence_and_drops(api, window):
    P, E, a, _, ids = window
    poses = P["poses_init"]
    sel = [a.get_edge_selection(k) for k in range(W)]
    psel = [a.get_selection(k) for k in range(W)]
    eu = a.eval_unary(poses)
    # plane selection again: the same plane lists, the edge lists untouched
    a.select_random(ids, seed=21, nonce=6)
    assert all(np.array_equal(x, a.get_edge_selection(k)) for k, x in enumerate(sel))
    assert all(np.array_equal(x, a.get_selection(k)) for k, x in enumerate(psel))
    # edge selection again leaves the plane lists and K2 alone, and reproduces its lists
    a.select_random_edges(ids, feature_res_num=60, seed=21, nonce=6)
    assert all(np.array_equal(x, a.get_selection(k)) for k, x in enumerate(psel))
    assert all(np.array_equal(x, a.get_edge_selection(k)) for k, x in enumerate(sel))
    eu2 = a.eval_unary(poses)
    assert all(np.array_equal(eu[x], eu2[x]) for x in ("H", "g", "cost"))
    # a fresh context: the plane lists are the same whether edge selection never ran (here), ran after (a) or before (below)
    f = api.Context(0)
    try:
        f.set_map(P["map_xyz"]); f.window_set_scans(P["scans"]); f.window_associate(poses)
        f.select_random(ids, seed=21, nonce=6)
        assert all(np.array_equal(x, f.get_selection(k)) for k, x in enumerate(psel))
        f.set_edge_map(E["map_xyz"])
        for k in range(W):
            f.window_set_edge_scan(k, E["scans"][k])
        full = f.window_associate_edges(poses)
        e_all = f.eval_edge(poses)
        f.select_random_edges(ids, feature_res_num=60, seed=21, nonce=6)
        f.select_random(ids, seed=21, nonce=6)
        assert all(np.array_equal(x, f.get_selection(k)) for k, x in enumerate(psel))
        assert all(np.array_equal(x, f.get_edge_selection(k)) for k, x in enumerate(sel))
        e_sel = f.eval_edge(poses)
        assert not np.array_equal(e_sel["cost"], e_all["cost"])
        # re-association drops every slot's selection: all edges are evaluated again, the full lists stay readable
        assert np.array_equal(f.window_associate_edges(poses), full)
        assert all(f.get_edge_selection(k) is None for k in range(W))
        assert all(np.array_equal(e_all[x], f.eval_edge(poses)[x]) for x in ("H", "g", "cost"))
        f.select_random_edges(ids, feature_res_num=60, seed=21, nonce=6)
        assert all(np.array_equal(e_sel[x], f.eval_edge(poses)[x]) for x in ("H", "g", "cost"))
        assert [f.get_edges(k)["n"] for k in range(W)] == full.tolist()
        # glio_set_edges drops the slot's selection
        e0 = f.get_edges(0)
        f.set_edges(0, e0["cp"], e0["pa"], e0["pb"], e0["s"])
        assert f.get_edge_selection(0) is None and np.array_equal(f.get_edge_selection(1), sel[1])
        assert f.eval_edge(poses)["cost"][0] == e_all["cost"][0]
        # a slide moves each selection with its slot; the recycled slot has none
        f.select_random_edges(ids, feature_res_num=60, seed=21, nonce=6)
        f.window_slide(W)
        for k in range(W - 1):
            assert np.array_equal(f.get_edge_selection(k), sel[k + 1])
        assert f.get_edge_selection(W - 1) is None and f.get_edges(W - 1)["n"] == 0
    finally:
        f.close()


@pytest.fixture(scope="module")
def batch(api):
    K, srng = 10, 2
    B = synth.batch_problem(K=K, Q=4000, seed=47, search_range=srng, rng_range=8.0)
    E = synth.batch_edge_problem(K=K, Q=3000, seed=47, search_range=srng, rng_range=8.0)
    cur, oth = dist.batch_pairs(K, srng)
    ctxs = []
    for edges in (True, False):
        c = api.Context(0)
        for k in range(K):
            c.batch_set_frame(k, B["scans"][k], B["poses_init"][k])
            if edges:
                c.batch_set_edge_frame(k, E["corner_scans"][k])
        c.batch_declare_pairs(cur, oth)
        c.batch_associate_pairs(cur, oth)
        if edges:
            c.batch_associate_edges_pairs(cur, oth)
        ctxs.append(c)
    yield B, cur, oth, ctxs[0], ctxs[1]
    for c in ctxs:
        c.close()


def _host_factor_set(api, B, sb):
    hf = api.HostFactorSet(); T = B["poses_true"]; rng = np.random.default_rng(7)
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0 if sb else 0.0)])
    hf.add_prior(0, T[0, :3], T[0, 3:], np.zeros(9) if sb else None, sw * 3)
    for i in range(B["K"] - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        hf.add_between(i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw)
    return hf


def _copy_pair_subsets(a, b, cur, oth):
    for c, o in zip(cur, oth):
        e = a.batch_get_edges(int(c), int(o))
        keep = a.batch_get_edge_selection(int(c), int(o))
        idx = np.arange(e["n"]) if keep is None else keep
        b.batch_set_pair_edges(int(c), int(o), e["cp"][idx], e["pa"][idx], e["pb"][idx], e["s"][idx])


@pytest.mark.parametrize("mode", [0, 1])
def test_batch_eval_and_solve_equal_subset_input(api, batch, mode):
    B, cur, oth, a, b = batch
    opt = api.select_default_options(batch_feature_res_num=30, batch_rand_set_num=400, seed=8, nonce=mode)
    na = a.batch_select_random_edges(cur, oth, mode, opt)
    assert (na == 30).any()
    a.batch_select_random(cur, oth, mode, seed=8, nonce=mode)
    for c, o in zip(cur, oth):
        b.batch_select(int(c), int(o), a.batch_get_selection(int(c), int(o)))
    _copy_pair_subsets(a, b, cur, oth)
    ea, eb = a.eval_binary_edge(B["poses_init"]), b.eval_binary_edge(B["poses_init"])
    assert all(np.array_equal(ea[x], eb[x]) for x in ("Hdiag", "Hoff", "g")) and ea["cost"] == eb["cost"]
    try:
        for c in (a, b):
            c.batch_use_edges(True)
        for with_sb in (False, True):
            hf = _host_factor_set(api, B, with_sb)
            sb = np.zeros((B["K"], 9)) if with_sb else None
            opts = api.batch_solver_options(max_num_iterations=8)
            ra, rb = a.batch_solve(B["poses_init"], sb, hf, opts), b.batch_solve(B["poses_init"], sb, hf, opts)
            assert ra["summary"].num_iterations == rb["summary"].num_iterations >= 3
            assert np.array_equal(ra["poses"], rb["poses"]) and ra["summary"].final_cost == rb["summary"].final_cost
    finally:
        for c in (a, b):
            c.batch_use_edges(False)


def test_batch_independence_and_drops(api, batch):
    B, cur, oth, a, _ = batch
    poses = B["poses_init"]
    pl = lambda: [a.batch_get_selection(int(c), int(o)) for c, o in zip(cur, oth)]           # noqa: E731
    el = lambda: [a.batch_get_edge_selection(int(c), int(o)) for c, o in zip(cur, oth)]      # noqa: E731
    same = lambda x, y: all((p is None and q is None) or np.array_equal(p, q) for p, q in zip(x, y))   # noqa: E731
    a.batch_select_random(cur, oth, 1, seed=4, nonce=2); p0 = pl()
    a.batch_select_random_edges(cur, oth, 1, seed=4, nonce=2); e0 = el()
    assert not same(p0, e0)                                                    # independent draws
    eb = a.eval_binary(poses)
    a.batch_select_random(cur, oth, 1, seed=4, nonce=2)                        # plane selection after: edge lists untouched
    assert same(el(), e0) and same(pl(), p0)
    a.batch_select_random_edges(cur, oth, 0, seed=9, nonce=1)                  # edge selection: plane lists and K2b untouched
    assert same(pl(), p0)
    eb2 = a.eval_binary(poses)
    assert all(np.array_equal(eb[x], eb2[x]) for x in ("Hdiag", "Hoff", "g")) and eb["cost"] == eb2["cost"]
    # re-association and glio_batch_set_pair_edges drop the selection: all edges are evaluated again
    a.batch_select_random_edges(cur, oth, 1, seed=4, nonce=2)
    full = a.batch_associate_edges_pairs(cur, oth)
    assert all(x is None for x in el())
    e_all = a.eval_binary_edge(poses)
    a.batch_select_random_edges(cur, oth, 1, seed=4, nonce=2)
    assert same(el(), e0)
    c0, o0 = int(cur[0]), int(oth[0])
    e = a.batch_get_edges(c0, o0)
    assert e["n"] == full[0]                                                   # the full list stays readable
    a.batch_set_pair_edges(c0, o0, e["cp"], e["pa"], e["pb"], e["s"])
    assert a.batch_get_edge_selection(c0, o0) is None and a.batch_get_edge_selection(int(cur[1]), int(oth[1])) is not None


def test_batch_clear_drops_the_edge_selection(api):
    cur, oth = np.array([0, 0, 1], np.int32), np.array([1, 2, 0], np.int32)
    ctx = _batch_edge_ctx(api, cur, oth, [300, 400, 500], seed=1)
    ctx.batch_select_random_edges(cur, oth, 1)
    assert ctx.batch_get_edge_selection(0, 1) is not None
    ctx.batch_clear()
    with pytest.raises(api.GlioError):
        ctx.batch_get_edge_selection(0, 1)                                     # the pair is gone
    ctx.close()
    ctx = _batch_edge_ctx(api, cur, oth, [300, 400, 500], seed=1)
    assert all(ctx.batch_get_edge_selection(int(c), int(o)) is None for c, o in zip(cur, oth))
    ctx.close()


def test_argument_errors_change_nothing(api, cfg3):
    ctx, cur, oth, sizes = cfg3
    opt = api.select_default_options(seed=3)
    ctx.batch_select_random_edges(cur, oth, 1, opt)
    before = [ctx.batch_get_edge_selection(int(c), int(o)) for c, o in zip(cur, oth)]
    bad = [
        (np.r_[cur[:12], cur[24:36], cur[:1]], np.r_[oth[:12], oth[24:36], oth[1:2]], 1, opt),          # not grouped by cur
        (cur[:3], np.r_[oth[:2], 199].astype(np.int32), 1, opt),                                       # not on the pair list
        (cur[:3], np.r_[oth[:2], cur[2]].astype(np.int32), 1, opt),                                    # cur == oth
        (np.r_[cur[:3], cur[2]], np.r_[oth[:3], oth[2]], 1, opt),                                      # listed twice
        (cur, oth, 2, opt),                                                                            # mode
        (cur, oth, -1, opt),
        (cur, oth, 0, api.select_default_options(batch_feature_res_num=0)),
        (cur, oth, 0, api.select_default_options(batch_feature_res_num=4097, batch_rand_set_num=5000)),
        (cur, oth, 0, api.select_default_options(batch_rand_set_num=24)),
        (cur, oth, 0, api.select_default_options(rand_set_num=0)),
        (cur, oth, 0, api.select_default_options(feature_res_num=4097)),
    ]
    for c, o, mode, op in bad:
        with pytest.raises(api.GlioError):
            ctx.batch_select_random_edges(c, o, mode, op)
    after = [ctx.batch_get_edge_selection(int(c), int(o)) for c, o in zip(cur, oth)]
    assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(before, after))
    assert all(ctx.batch_get_selection(int(c), int(o)) is None for c, o in zip(cur[:50], oth[:50]))   # no plane selection appeared
    with pytest.raises(api.GlioError):
        ctx.batch_get_edge_selection(0, 199)
    wctx = _window_edge_ctx(api, [500, 5000], seed=2)
    wctx.select_random_edges([0, 1], seed=4)
    w0 = [wctx.get_edge_selection(k) for k in range(2)]
    for kw in (dict(feature_res_num=0), dict(feature_res_num=4097), dict(rand_set_num=0), dict(batch_rand_set_num=1)):
        with pytest.raises(api.GlioError):
            wctx.select_random_edges([0, 1], **kw)
    with pytest.raises(api.GlioError):
        wctx.select_random_edges(np.zeros(0, np.int64))
    with pytest.raises(api.GlioError):
        wctx.select_random_edges(np.zeros(4097, np.int64))
    assert all(np.array_equal(x, wctx.get_edge_selection(k)) for k, x in enumerate(w0))
    assert wctx.get_selection(0) is None
    wctx.close()


# ---- sharding -------------------------------------------------------------------------------------------------------------------

def _run(tmp_path, world, tag):
    out = str(tmp_path / tag)
    env = dict(os.environ); env["OMP_NUM_THREADS"] = "4"
    if world == 1:
        subprocess.check_call([sys.executable, WORKER, out], env=env, timeout=600)
    else:
        subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                               "--master-port", "29637", WORKER, out], env=env, timeout=600)
    return [json.load(open(out + f".rank{r}.json")) for r in range(world)]


def test_sharded_edge_selection_and_solve_equal_single_rank(tmp_path):
    one = _run(tmp_path, 1, "one")[0]
    two = _run(tmp_path, 2, "two")
    assert two[0]["hook_calls"] > 0 and two[0]["hook_calls"] == two[1]["hook_calls"]
    assert 0 < two[0]["n_edge_active"] < one["n_edge_active"] < one["n_edge_own"]
    assert two[0]["n_edge_active"] + two[1]["n_edge_active"] == one["n_edge_active"]
    sel_one = {tuple(k): v for k, v in one["edge_selection"]}
    for r in two:
        for k, v in r["edge_selection"]:
            assert sel_one[tuple(k)] == v
        assert r["iterations"] == one["iterations"] >= 3
        assert abs(r["final_cost"] - one["final_cost"]) <= 1e-9 * abs(one["final_cost"])
        assert np.max(np.abs(np.array(r["poses"])[:, :3] - np.array(one["poses"])[:, :3])) <= 1e-7
        assert np.max(np.abs(np.array(r["poses"])[:, 3:] - np.array(one["poses"])[:, 3:])) <= 1e-8
    assert np.array_equal(np.array(two[0]["poses"]), np.array(two[1]["poses"]))
