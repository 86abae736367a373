"""K1e: scan-to-map edge association on the device (glio_window_associate_edges) against the sequential reference
(tests/edge_reference.py on the CPU oracle's 5-NN), bit for bit; state the edge calls must leave alone; sliding, errors, launches."""
import numpy as np
import pytest

from glio_b200 import synth
from tests import edge_reference as er

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from glio_b200 import api as a
    return a


@pytest.fixture(scope="module")
def ctx(api):
    c = api.Context(0, keep_debug=1)
    yield c
    c.close()


def _check(ctx, oracle, corner_map, scans, poses, opts=None, tree=None, brute=False):
    """Associate slots 0..W-1 (scans already set) and compare every slot with the reference; returns the reference results."""
    ne = ctx.window_associate_edges(poses, **(opts or {}))
    if tree is None and not brute:
        tree = oracle.KdTree(corner_map)
    refs = []
    for k, s in enumerate(scans):
        t2, q2 = ctx.lidar_pose(poses[k])
        o = er.associate_edges(oracle, corner_map, s, t2, q2, opts, tree=None if brute else tree)
        Q = len(s)
        d = ctx.get_edge_debug(k, Q)
        assert np.array_equal(d["pm"], o["pm"]), "transformed corner points differ"
        assert np.array_equal(d["status"], o["status"]), f"status differs at {np.nonzero(d['status'] != o['status'])[0][:10]}"
        ok = o["status"] != er.FAIL_RADIUS
        assert np.array_equal(d["idx5"][ok], o["idx5"][ok]) and np.array_equal(d["sqd5"][ok], o["sqd5"][ok])
        assert np.array_equal(d["eig"], o["eig"]), "eigenvalues differ (bit-exact expected)"
        e = ctx.get_edges(k)
        assert e["n"] == ne[k] == o["n"]
        for key in ("cp", "pa", "pb", "s", "src"):
            assert np.array_equal(e[key], o[key]), key
        refs.append(o)
    return refs


@pytest.mark.parametrize("W,Q,M,seed,offset", [(1, 1, 5000, 1, 0.0), (1, 50000, 200000, 2, 0.0), (20, 600, 100000, 3, 0.0),
                                               (3, 2000, 60000, 4, 3000.0), (2, 2000, 60000, 5, 20000.0)])
def test_parity_window(ctx, oracle, W, Q, M, seed, offset):
    P = synth.window_edge_problem(W=W, Q=Q, M=M, seed=seed)
    cmap = P["map_xyz"] + np.float32(offset)
    poses = P["poses_init"].copy(); poses[:, :3] += offset
    ctx.set_edge_map(cmap)
    for k in range(W):
        ctx.window_set_edge_scan(k, P["scans"][k])
    refs = _check(ctx, oracle, cmap, P["scans"], poses)
    st = np.concatenate([r["status"] for r in refs])
    assert (st == er.VALID).any()
    if Q > 1:
        assert (st == er.FAIL_LINE).any()


def test_parity_stride8_host_and_device_and_radius_gate(ctx, oracle):
    import torch
    P = synth.window_edge_problem(W=2, Q=3000, M=50000, seed=6)
    poses = P["poses_init"].copy(); poses[1, :3] += [0.8, -0.6, 0.4]           # far corners fail the radius gate
    rng = np.random.default_rng(6)
    s8 = [np.concatenate([s, rng.standard_normal((len(s), 5)).astype(np.float32)], axis=1) for s in P["scans"]]
    ctx.set_edge_map(P["map_xyz"])
    ctx.window_set_edge_scan(0, s8[0])
    dev = torch.from_numpy(s8[1]).cuda()
    ctx.window_set_edge_scan(1, dev)
    refs = _check(ctx, oracle, P["map_xyz"], s8, poses)
    st = np.concatenate([r["status"] for r in refs])
    assert (st == er.FAIL_RADIUS).any() and (st == er.VALID).any() and (st == er.FAIL_LINE).any()
    # a gate equal to a query's 5th squared distance rejects that query (the comparison is strict)
    r0 = refs[0]
    i = int(np.nonzero(r0["status"] == er.VALID)[0][0])
    gate = float(r0["sqd5"][i, 4])
    refs = _check(ctx, oracle, P["map_xyz"], s8, poses, dict(max_sqdist=gate))
    assert refs[0]["status"][i] == er.FAIL_RADIUS
    del dev


def test_ties_and_brute_force(ctx, oracle):
    """every corner-map point twice: neighbours come in equal-distance pairs, the lower index first"""
    P = synth.window_edge_problem(W=1, Q=2000, M=6000, seed=7)
    m = np.concatenate([P["map_xyz"], P["map_xyz"]])
    ctx.set_edge_map(m)
    ctx.window_set_edge_scan(0, P["scans"][0])
    r = _check(ctx, oracle, m, P["scans"], P["poses_init"], brute=True)[0]
    ok = r["status"] != er.FAIL_RADIUS
    assert np.all(r["sqd5"][ok, 0] == r["sqd5"][ok, 1]) and np.all(r["idx5"][ok, 0] + 6000 == r["idx5"][ok, 1])


@pytest.mark.parametrize("offset", [0.0, 3000.0, 20000.0])
def test_degenerate_neighbourhoods_on_the_device(ctx, oracle, offset):
    """identical, exactly collinear, isotropic in-plane and dyadic lambda_2 = 3 lambda_1 clusters (50 m apart), a corner map of
    exactly these points; queries at the cluster centres with the identity lidar pose"""
    base = np.array([[0.0, 0.0, 0.0], [50.0, 0.0, 0.0], [0.0, 50.0, 0.0], [50.0, 50.0, 0.0]]) + offset
    same = np.zeros((5, 3))
    line = np.outer([0.0, 0.25, -0.25, 0.5, -0.5], [1.0, 0.0, 0.0])
    square = np.array([[0, 0, 0], [0.5, 0, 0], [-0.5, 0, 0], [0, 0.5, 0], [0, -0.5, 0]], float)
    dy = 0.125 * np.array([[2, 0, 0], [-1, 1, 0], [-1, -1, 0], [0, 0, 0], [0, 0, 0]], float)
    m = np.concatenate([b + c for b, c in zip(base, (same, line, square, dy))]).astype(np.float32)
    q = base.astype(np.float32)
    pose = np.array([[0, 0, 0.28, 1, 0, 0, 0]])                               # T2 = 0, Q2 = identity: p_m = p
    ctx.set_edge_map(m)
    ctx.window_set_edge_scan(0, q)
    r = _check(ctx, oracle, m, [q], pose, brute=True)[0]
    assert list(r["status"]) == [er.FAIL_LINE, er.VALID, er.FAIL_LINE, er.FAIL_LINE]
    assert r["eig"][3, 2] == 3 * r["eig"][3, 1]
    r = _check(ctx, oracle, m, [q], pose, dict(min_ratio=2.5), brute=True)[0]
    assert list(r["status"]) == [er.FAIL_LINE, er.VALID, er.FAIL_LINE, er.VALID]


def test_five_point_map_and_too_small_map(api, oracle):
    c = api.Context(0, keep_debug=1)
    try:
        m5 = (np.array([[0, 0, 0], [0.1, 0, 0], [0.2, 0, 0], [0.3, 0.01, 0], [0.4, 0, 0]]) + [5, 1, 2]).astype(np.float32)
        c.set_edge_map(m5)
        q = np.array([[5.2, 1.0, 2.0], [9.0, 9.0, 9.0]], np.float32)
        c.window_set_edge_scan(0, q)
        pose = np.array([[0, 0, 0.28, 1, 0, 0, 0]])                           # T2 = 0, Q2 = identity: p_m = p
        r = _check(c, oracle, m5, [q], pose, brute=True)[0]
        assert list(r["status"]) == [er.VALID, er.FAIL_RADIUS]
        before = c.get_edges(0)
        with pytest.raises(api.GlioError, match="error -3"):
            c.set_edge_map(m5[:4])
        r2 = _check(c, oracle, m5, [q], pose, brute=True)[0]                  # the 5-point map is still the corner map
        assert np.array_equal(r2["status"], r["status"])
        assert all(np.array_equal(before[k], c.get_edges(0)[k]) for k in ("cp", "pa", "pb", "s", "src"))
    finally:
        c.close()


def test_edge_calls_leave_surf_state_alone(api):
    """a context that also runs every edge call gives the surf association, selection, evaluation, solve and marginalisation of
    one that never touched edges, bit for bit"""
    P = synth.window_problem(W=4, Q=3000, M=40000, seed=13)
    E = synth.window_edge_problem(W=4, Q=1500, M=30000, seed=14)
    a, b = api.Context(0, keep_debug=1), api.Context(0, keep_debug=1)
    try:
        for c in (a, b):
            c.set_map(P["map_xyz"]); c.window_set_scans(P["scans"])
        b.set_edge_map(E["map_xyz"])
        for k in range(4):
            b.window_set_edge_scan(k, E["scans"][k])
        ne = b.window_associate_edges(P["poses_init"])
        assert ne.sum() > 0
        na, nb = a.window_associate(P["poses_init"]), b.window_associate(P["poses_init"])
        b.window_associate_edges(P["poses_init"])
        assert np.array_equal(na, nb)
        for k in range(4):
            for key, x in a.get_assoc_debug(k, 3000).items():
                assert np.array_equal(x, b.get_assoc_debug(k, 3000)[key])
            for key, x in a.get_matches(k, 3000).items():
                assert np.array_equal(x, b.get_matches(k, 3000)[key])
        assert np.array_equal(a.get_map(), b.get_map())
        ids = np.arange(4, dtype=np.int64)
        assert np.array_equal(a.select_random(ids), b.select_random(ids))
        for jac in (0, 1):
            ea, eb = a.eval_unary(P["poses_init"], jac_kind=jac), b.eval_unary(P["poses_init"], jac_kind=jac)
            assert all(np.array_equal(ea[key], eb[key]) for key in ("H", "g", "cost"))
        ra, rb = a.window_solve(P["poses_init"]), b.window_solve(P["poses_init"])
        assert np.array_equal(ra["poses"], rb["poses"]) and np.array_equal(ra["steps"], rb["steps"])
        sb = np.zeros((4, 9))
        pa, pb = a.window_marginalize(ra["poses"], sb).arrays(), b.window_marginalize(rb["poses"], sb).arrays()
        assert all(np.array_equal(pa[key], pb[key]) for key in ("lin_jac", "lin_res", "x0_pose", "A_info", "b_info"))
    finally:
        a.close(); b.close()


def test_associated_edges_feed_k2e(ctx, oracle):
    """glio_eval_edge evaluates the associated lists as the oracle's LidarEdgeFactor does"""
    P = synth.window_edge_problem(W=3, Q=2000, M=40000, seed=15)
    ctx.set_edge_map(P["map_xyz"])
    for k in range(3):
        ctx.window_set_edge_scan(k, P["scans"][k])
    ne = ctx.window_associate_edges(P["poses_init"])
    es = [ctx.get_edges(k) for k in range(3)]
    kf = np.concatenate([np.full(ne[k], k, np.int32) for k in range(3)])
    cat = {key: np.concatenate([e[key] for e in es]) for key in ("cp", "pa", "pb", "s")}
    o = oracle.eval_edge(P["poses_init"], P["q_lb"], P["t_lb"], kf, cat["cp"], cat["pa"], cat["pb"], cat["s"], huber_delta=1.0)
    g = ctx.eval_edge(P["poses_init"])
    for k in range(3):
        Hk = o["H"][6 * k:6 * k + 6, 6 * k:6 * k + 6]
        assert np.max(np.abs(g["H"][k] - Hk)) <= 1e-11 * np.max(np.abs(Hk))
        assert abs(g["cost"][k] - o["cost"][kf == k].sum()) <= 1e-11 * abs(g["cost"][k])


def test_slide_carries_corner_scans_and_edges(api, oracle):
    W = 4
    E = synth.window_edge_problem(W=W + 1, Q=1500, M=40000, seed=16)
    a = api.Context(0, keep_debug=1)
    try:
        a.set_edge_map(E["map_xyz"])
        for k in range(W):
            a.window_set_edge_scan(k, E["scans"][k])
        a.window_associate_edges(E["poses_init"][:W])
        before = [a.get_edges(k) for k in range(W)]
        a.window_slide(W)
        for k in range(W - 1):
            assert all(np.array_equal(before[k + 1][key], a.get_edges(k)[key]) for key in ("cp", "pa", "pb", "s", "src"))
        assert a.get_edges(W - 1)["n"] == 0                                     # the dropped keyframe's edges left with it
        with pytest.raises(api.GlioError, match="error -4"):                     # and so did its corner scan
            a.window_associate_edges(E["poses_init"][1:W + 1])
        a.window_set_edge_scan(W - 1, E["scans"][W])
        _check(a, oracle, E["map_xyz"], E["scans"][1:W + 1], E["poses_init"][1:W + 1])
    finally:
        a.close()


def test_argument_errors_change_nothing(api, ctx):
    fresh = api.Context(0, keep_debug=1)
    try:
        fresh.window_set_edge_scan(0, np.zeros((10, 3), np.float32))
        pose = np.array([[0, 0, 0, 1, 0, 0, 0.0]])
        with pytest.raises(api.GlioError, match="error -4"):                     # no corner map
            fresh.window_associate_edges(pose)
        fresh.set_edge_map(np.random.default_rng(0).random((100, 3)).astype(np.float32))
        with pytest.raises(api.GlioError, match="error -4"):                     # slot 1 has no corner scan
            fresh.window_associate_edges(np.concatenate([pose, pose]))
        assert fresh.get_edges(0)["n"] == 0
        assert fresh.window_associate_edges(pose).shape == (1,)
    finally:
        fresh.close()
    P = synth.window_edge_problem(W=2, Q=800, M=20000, seed=17)
    ctx.set_edge_map(P["map_xyz"])
    for k in range(2):
        ctx.window_set_edge_scan(k, P["scans"][k])
    ne = ctx.window_associate_edges(P["poses_init"])
    snap = [ctx.get_edges(k) for k in range(2)]
    for bad in (dict(max_sqdist=0.0), dict(max_sqdist=float("nan")), dict(min_ratio=-1.0), dict(half_length=0.0),
                dict(score=float("inf"))):
        with pytest.raises(api.GlioError, match="error -3"):
            ctx.window_associate_edges(P["poses_init"], **bad)
    with pytest.raises(api.GlioError, match="error -3"):
        ctx.window_associate_edges(np.zeros((0, 7)))
    with pytest.raises(api.GlioError, match="error -3"):
        ctx.window_set_edge_scan(0, np.zeros((0, 3), np.float32))
    with pytest.raises(api.GlioError, match="error -3"):
        ctx.window_set_edge_scan(-1, P["scans"][0])
    for k in range(2):
        e = ctx.get_edges(k)
        assert e["n"] == ne[k] and all(np.array_equal(snap[k][key], e[key]) for key in ("cp", "pa", "pb", "s", "src"))


def test_launches_constant_in_W(api):
    """the same corner map and the same corner points as 2 and as 20 keyframes"""
    E = synth.window_edge_problem(W=20, Q=600, M=30000, seed=18)
    c = api.Context(0)
    try:
        c.set_edge_map(E["map_xyz"])
        counts = []
        for W in (2, 20):
            per = 20 // W
            poses = E["poses_init"][::per][:W]
            for k in range(W):
                c.window_set_edge_scan(k, np.concatenate(E["scans"][k * per:(k + 1) * per]))
            c.window_associate_edges(poses)
            n0 = c.launch_count
            c.window_associate_edges(poses)
            counts.append(c.launch_count - n0)
        assert counts[0] == counts[1]
    finally:
        c.close()


def test_edge_localmap_equals_uploaded_concatenation(api, oracle):
    """the corner local map (push, pop_front, build without a filter) is the corner map the same concatenation uploads"""
    E = synth.window_edge_problem(W=3, Q=1500, M=9000, seed=19)
    parts = [E["map_xyz"][i * 3000:(i + 1) * 3000] for i in range(3)]
    ts = [np.array([0.5 * i, -0.2 * i, 0.1]) for i in range(3)]
    qs = [synth.quat_from_rpy(0.0, 0.0, 0.01 * i) for i in range(3)]
    a, b = api.Context(0, keep_debug=1), api.Context(0, keep_debug=1)
    try:
        a.edge_localmap_push(np.zeros((10, 3), np.float32), ts[0], qs[0])
        for p, t, q in zip(parts, ts, qs):
            a.edge_localmap_push(p, t, q)
        a.edge_localmap_pop_front()
        assert a.edge_localmap_build(leaf=0.0) == 9000
        cat = np.concatenate([oracle.transform_points(p, t, q) for p, t, q in zip(parts, ts, qs)])
        b.set_edge_map(cat)
        for c in (a, b):
            for k in range(3):
                c.window_set_edge_scan(k, E["scans"][k])
        _check(a, oracle, cat, E["scans"], E["poses_init"])
        _check(b, oracle, cat, E["scans"], E["poses_init"])
        a.edge_localmap_clear()
        with pytest.raises(api.GlioError, match="error -4"):
            a.edge_localmap_build(leaf=0.0)
    finally:
        a.close(); b.close()
