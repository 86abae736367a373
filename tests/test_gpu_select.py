"""The device feature selection (glio_select_random, glio_batch_select_random) against tests/select_reference.py, bit for bit, and
what the evaluation, solve and marginalisation make of it."""
import numpy as np
import pytest
import torch  # noqa: F401  (first: torch binds its bundled CUDA runtime before libglio_b200.so loads)

from glio_b200 import dist, synth
from tests import select_reference as sr

pytestmark = pytest.mark.gpu

WINDOW_SIZES = [0, 1, 2, 99, 100, 101, 102, 103, 299, 300, 301, 302, 1000, 4096, 100_000]
BATCH_SIZES = [0, 1, 24, 25, 26, 27, 49, 50, 51, 52, 400, 425, 426, 427, 3000]


def _fake_matches(rng, n):
    cp = rng.normal(size=(n, 3)).astype(np.float32)
    nsd = rng.normal(size=(n, 4)).astype(np.float32)
    w = rng.uniform(0.5, 1.0, n).astype(np.float32)
    return cp, nsd, w


def _window_ctx(api, sizes, seed=0):
    ctx = api.Context(0)
    rng = np.random.default_rng(seed)
    data = []
    for k, n in enumerate(sizes):
        cp, nsd, w = _fake_matches(rng, n)
        ctx.set_matches(k, cp, nsd, w)
        data.append((cp, nsd, w))
    return ctx, data


def _check_window(ctx, sizes, ids, opt, na):
    for k, n in enumerate(sizes):
        keep, undef = sr.window_select(n, int(ids[k]), opt.seed, opt.nonce, F=opt.feature_res_num, R=opt.rand_set_num,
                                       random_select=bool(opt.random_select))
        got = ctx.get_selection(k)
        if keep is None:
            assert got is None and na[k] == n, (k, n)
        else:
            assert got is not None and got.tolist() == keep, (k, n)
            assert na[k] == len(keep)


@pytest.mark.parametrize("W", [1, 20, 64])
def test_window_selection_bit_exact(W):
    from glio_b200 import api
    sizes = [WINDOW_SIZES[(k * 7 + W) % len(WINDOW_SIZES)] for k in range(W)]
    if W == 1:
        sizes = [100_000]
    ctx, _ = _window_ctx(api, sizes, seed=W)
    ids = np.arange(W, dtype=np.int64) + 1000
    for opt in (api.select_default_options(seed=11, nonce=3), api.select_default_options(feature_res_num=7, rand_set_num=2, seed=5),
                api.select_default_options(feature_res_num=4096, seed=1), api.select_default_options(random_select=0)):
        na = ctx.select_random(ids, opt)
        _check_window(ctx, sizes, ids, opt, na)
        assert np.array_equal(ctx.get_match_counts(W), na)
    ctx.close()


def test_window_threshold_sizes_every_size_once():
    from glio_b200 import api
    ctx, data = _window_ctx(api, WINDOW_SIZES, seed=3)
    ids = np.array([5, 9, 4, 1, 2, 3, 6, 7, 8, 10, 11, 12, 13, 14, 15], np.int64)
    opt = api.select_default_options(seed=2**64 - 1, nonce=2**40 + 7)
    na = ctx.select_random(ids, opt)
    _check_window(ctx, WINDOW_SIZES, ids, opt, na)
    # the gathered records are the selected matches, in draw order
    r = ctx.eval_unary_residuals(12, np.array([0, 0, 0, 1, 0, 0, 0.0]), 200)[0]
    cp, nsd, w = data[12]
    keep = ctx.get_selection(12)
    ctx.select(12, keep)
    assert np.array_equal(ctx.eval_unary_residuals(12, np.array([0, 0, 0, 1, 0, 0, 0.0]), 200)[0], r)
    ctx.close()


def _batch_ctx(api, cur, oth, sizes, seed=0):
    ctx = api.Context(0)
    rng = np.random.default_rng(seed)
    for c, o, n in zip(cur, oth, sizes):
        cp = rng.normal(size=(n, 3)).astype(np.float32)
        nc = rng.normal(size=(n, 6))
        w = rng.uniform(0.5, 1.0, n).astype(np.float32)
        ctx.batch_set_pair_matches(int(c), int(o), cp, nc, w)
    return ctx


@pytest.fixture(scope="module")
def cfg3():
    from glio_b200 import api
    cur, oth = dist.batch_pairs(200, 6)
    rng = np.random.default_rng(17)
    sizes = rng.integers(0, 2000, len(cur))
    sizes[::11] = np.array(BATCH_SIZES)[rng.integers(0, len(BATCH_SIZES), len(sizes[::11]))]
    ctx = _batch_ctx(api, cur, oth, sizes, seed=4)
    yield ctx, cur, oth, sizes
    ctx.close()


def _check_batch(ctx, cur, oth, sizes, mode, opt, na):
    ref = sr.batch_select(list(zip(cur.tolist(), oth.tolist())), list(sizes), mode, opt.seed, opt.nonce,
                          B=opt.batch_feature_res_num, BR=opt.batch_rand_set_num)
    for i, (c, o) in enumerate(zip(cur, oth)):
        keep, _ = ref[i]
        got = ctx.batch_get_selection(int(c), int(o))
        if keep is None:
            assert got is None and na[i] == sizes[i], (i, sizes[i])
        else:
            assert got.tolist() == keep, (i, sizes[i])
            assert na[i] == len(keep)
    return ref


@pytest.mark.parametrize("mode", [0, 1])
def test_cfg3_pairs_in_one_call_bit_exact(cfg3, mode):
    from glio_b200 import api
    ctx, cur, oth, sizes = cfg3
    opt = api.select_default_options(seed=7, nonce=mode * 4 + 1)
    l0 = ctx.launch_count
    na = ctx.batch_select_random(cur, oth, mode, opt)
    assert ctx.launch_count - l0 == 1
    ref = _check_batch(ctx, cur, oth, sizes, mode, opt, na)
    assert sum(k is not None for k, _ in ref) > 1000
    if mode == 0:
        assert any(u for _, u in ref), "the undefined size n = 50 is among the pairs"
        assert any(k is None and n >= 50 for (k, _), n in zip(ref, sizes)), "a `return` reaches later pairs of its keyframe"


def test_seed_stream_nonce_each_change_the_lists(cfg3):
    from glio_b200 import api
    ctx, cur, oth, sizes = cfg3
    big = np.nonzero(sizes > 500)[0]
    i = int(big[0])
    c, o = cur[i:i + 1], oth[i:i + 1]

    def lst(**kw):
        ctx.batch_select_random(c, o, 1, api.select_default_options(**kw))
        return ctx.batch_get_selection(int(c[0]), int(o[0])).tolist()
    base = lst(seed=1, nonce=2)
    assert lst(seed=1, nonce=2) == base
    assert lst(seed=2, nonce=2) != base and lst(seed=1, nonce=3) != base
    ctx.batch_select_random(c, o, 0, api.select_default_options(seed=1, nonce=2))
    assert ctx.batch_get_selection(int(c[0]), int(o[0])).tolist() != base                  # the domain
    wctx, _ = _window_ctx(api, [5000], seed=1)
    wctx.select_random([3], seed=1, nonce=2); a = wctx.get_selection(0).tolist()
    wctx.select_random([3], seed=1, nonce=2); assert wctx.get_selection(0).tolist() == a
    wctx.select_random([4], seed=1, nonce=2); assert wctx.get_selection(0).tolist() != a     # the stream
    wctx.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_sharded_selection_equals_single(cfg3, mode):
    from glio_b200 import api
    ctx, cur, oth, sizes = cfg3
    opt = api.select_default_options(seed=99, nonce=5)
    ctx.batch_select_random(cur, oth, mode, opt)
    own = dist.owner_of(cur, 200, 4) == 2                    # the pairs rank 2 of 4 would select
    part = _batch_ctx(api, cur[own], oth[own], sizes[own], seed=0)
    part.batch_select_random(cur[own], oth[own], mode, opt)
    for c, o in zip(cur[own], oth[own]):
        a = ctx.batch_get_selection(int(c), int(o)); b = part.batch_get_selection(int(c), int(o))
        assert (a is None and b is None) or np.array_equal(a, b)
    part.close()


def test_argument_errors_change_nothing(cfg3):
    from glio_b200 import api
    ctx, cur, oth, sizes = cfg3
    opt = api.select_default_options(seed=3)
    ctx.batch_select_random(cur, oth, 1, opt)
    before = [ctx.batch_get_selection(int(c), int(o)) for c, o in zip(cur, oth)]
    bad = [
        (np.r_[cur[:12], cur[24:36], cur[:1]], np.r_[oth[:12], oth[24:36], oth[1:2]], 1, opt),          # not grouped by cur
        (cur[:3], np.r_[oth[:2], 199].astype(np.int32), 1, opt),                                       # never associated
        (cur[:3], np.r_[oth[:2], cur[2]].astype(np.int32), 1, opt),                                    # cur == oth
        (np.r_[cur[:3], cur[2]], np.r_[oth[:3], oth[2]], 1, opt),                                      # listed twice
        (cur, oth, 2, opt),                                                                            # mode
        (cur, oth, 0, api.select_default_options(batch_feature_res_num=0)),
        (cur, oth, 0, api.select_default_options(batch_feature_res_num=4097, batch_rand_set_num=5000)),
        (cur, oth, 0, api.select_default_options(batch_rand_set_num=24)),
        (cur, oth, 0, api.select_default_options(rand_set_num=0)),
        (cur, oth, 0, api.select_default_options(feature_res_num=4097)),
    ]
    for c, o, mode, op in bad:
        with pytest.raises(api.GlioError):
            ctx.batch_select_random(c, o, mode, op)
    after = [ctx.batch_get_selection(int(c), int(o)) for c, o in zip(cur, oth)]
    assert all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(before, after))
    wctx, _ = _window_ctx(api, [500, 5000], seed=2)
    wctx.select_random([0, 1], seed=4)
    w0 = [wctx.get_selection(k) for k in range(2)]
    for kw in (dict(feature_res_num=0), dict(feature_res_num=4097), dict(rand_set_num=0), dict(batch_rand_set_num=1)):
        with pytest.raises(api.GlioError):
            wctx.select_random([0, 1], **kw)
    with pytest.raises(api.GlioError):
        wctx.select_random(np.zeros(0, np.int64))
    assert all(np.array_equal(a, wctx.get_selection(k)) for k, a in enumerate(w0))
    assert np.array_equal(wctx.get_match_counts(2), [100, 100])
    wctx.close()


def test_one_launch_and_no_stream_synchronisation():
    import torch
    from glio_b200 import api
    ctx, _ = _window_ctx(api, [100_000] * 20, seed=5)
    ctx.select_random(np.arange(20), seed=1)                 # buffers and the staging table exist now
    ctx.synchronize()
    st = torch.cuda.ExternalStream(ctx.stream)
    with torch.cuda.stream(st):
        torch.cuda._sleep(200_000_000)                        # keeps the context's stream busy for a while (order 0.1 s)
    l0 = ctx.launch_count
    ctx.select_random(np.arange(20), seed=2)
    busy = not st.query()
    assert ctx.launch_count - l0 == 1
    assert busy, "glio_select_random waited for the stream"
    ctx.synchronize()
    assert ctx.get_selection(0).tolist() == sr.window_select(100_000, 0, 2, 0)[0]
    ctx.close()


# ---- what the rest of the pipeline makes of the selection -------------------------------------------------------------------

@pytest.fixture(scope="module")
def window():
    from glio_b200 import api
    W, Q, M = 4, 3000, 40000
    P = synth.window_problem(W=W, Q=Q, M=M, seed=13)
    ctxs = []
    for _ in range(2):
        c = api.Context(0)
        c.set_map(P["map_xyz"]); c.window_set_scans(P["scans"]); c.window_associate(P["poses_init"])
        ctxs.append(c)
    ids = np.array([40, 41, 42, 43], np.int64)
    opt = api.select_default_options(seed=21, nonce=6)
    na = ctxs[0].select_random(ids, opt)
    assert (na == 100).all()
    for k in range(W):
        ctxs[1].select(k, ctxs[0].get_selection(k))          # the list-input path with the copied-out lists
    yield P, ctxs, ids, opt
    for c in ctxs:
        c.close()


def test_window_eval_solve_marginalize_equal_list_input(window):
    P, (a, b), _, _ = window
    for jac in (0, 1):
        ea, eb = a.eval_unary(P["poses_init"], jac_kind=jac), b.eval_unary(P["poses_init"], jac_kind=jac)
        for key in ("H", "g", "cost"):
            assert np.array_equal(ea[key], eb[key])
    ra, rb = a.window_solve(P["poses_init"]), b.window_solve(P["poses_init"])
    assert np.array_equal(ra["poses"], rb["poses"]) and np.array_equal(ra["steps"], rb["steps"])
    sb = np.zeros((len(P["poses_init"]), 9))
    pa, pb = a.window_marginalize(ra["poses"], sb).arrays(), b.window_marginalize(rb["poses"], sb).arrays()
    for key in ("lin_jac", "lin_res", "x0_pose", "A_info", "b_info"):
        assert np.array_equal(pa[key], pb[key])


def test_window_solve_with_selection_against_oracle(window, oracle):
    po = oracle
    P, (a, _), ids, opt = window
    W = len(P["poses_init"])
    tree = po.KdTree(P["map_xyz"])
    prob = po.WindowProblem(P["poses_init"], None, P["q_lb"], P["t_lb"], huber_delta=1.0)
    kf, cp, nsd, score = [], [], [], []
    for k in range(W):
        t2, q2 = a.lidar_pose(P["poses_init"][k])
        o = po.assoc_scan_to_map(P["map_xyz"], P["scans"][k], t2, q2, tree=tree)
        v = o["status"] == po.GO_VALID
        keep, _ = sr.window_select(int(v.sum()), int(ids[k]), opt.seed, opt.nonce)
        assert a.get_selection(k).tolist() == keep
        kf.append(np.full(len(keep), k, np.int32)); cp.append(P["scans"][k][v][keep]); nsd.append(o["nsd"][v][keep]); score.append(o["score"][v][keep])
    prob.add_unary(*map(np.concatenate, (kf, cp, nsd, score)))
    ro = prob.solve(po.solver_options())
    rg = a.window_solve(P["poses_init"])
    assert rg["summary"].num_iterations == ro["summary"].num_iterations
    for x, y in zip(rg["steps"], ro["steps"]):
        x = x.reshape(W, 6); y = y.reshape(W, 6)
        assert np.max(np.abs(x[:, :3] - y[:, :3])) <= 1e-6 and np.max(2 * np.linalg.norm(x[:, 3:] - y[:, 3:], axis=1)) <= 1e-8


def test_eval_binary_equal_list_input():
    from glio_b200 import api
    K, Q, srng = 6, 4000, 2
    B = synth.batch_problem(K=K, Q=Q, seed=31, search_range=srng, rng_range=5.0)
    cur, oth = dist.batch_pairs(K, srng)
    ctxs = []
    for _ in range(2):
        c = api.Context(0)
        for k in range(K):
            c.batch_set_frame(k, B["scans"][k], B["poses_init"][k])
        c.batch_associate_pairs(cur, oth)
        ctxs.append(c)
    a, b = ctxs
    for mode in (0, 1):
        na = a.batch_select_random(cur, oth, mode, seed=8, nonce=mode)
        assert (na == 25).sum() > len(cur) // 2
        for c, o in zip(cur, oth):
            b.batch_select(int(c), int(o), a.batch_get_selection(int(c), int(o)))
        ea, eb = a.eval_binary(B["poses_init"]), b.eval_binary(B["poses_init"])
        for key in ("Hdiag", "Hoff", "g"):
            assert np.array_equal(ea[key], eb[key])
        assert ea["cost"] == eb["cost"]
    for c in ctxs:
        c.close()


def test_list_input_selection_is_kept_per_slot_and_pair():
    from glio_b200 import api
    ctx, _ = _window_ctx(api, [50, 60], seed=8)
    assert ctx.get_selection(0) is None
    ctx.select(0, [3, 1, 4]); ctx.select(1, [])
    assert ctx.get_selection(0).tolist() == [3, 1, 4] and ctx.get_selection(1).tolist() == []
    ctx.select(0, None)
    assert ctx.get_selection(0) is None
    ctx.close()
