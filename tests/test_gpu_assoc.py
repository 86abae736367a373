"""K0+K1 parity: CUDA scan-to-map association vs the CPU oracle, through the C ABI (bit-exact bar)."""
import numpy as np
import pytest

from glio_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from glio_b200 import api
    c = api.Context(0, keep_debug=1)
    yield c
    c.close()


def _check_slot(ctx, oracle, P, k, t2, q2, tree):
    o = oracle.assoc_scan_to_map(P["map_xyz"], P["scans"][k], t2, q2, tree=tree)
    Q = len(P["scans"][k])
    d = ctx.get_assoc_debug(k, Q)
    assert np.array_equal(d["pm"], o["pm"]), "transformed query points differ"
    assert np.array_equal(d["status"], o["status"]), f"status mismatch at {np.nonzero(d['status'] != o['status'])[0][:10]}"
    ok = o["status"] != oracle.GO_FAIL_RADIUS
    assert np.array_equal(d["idx5"][ok], o["idx5"][ok]), "kNN indices differ"
    assert np.array_equal(d["sqd5"][ok], o["sqd5"][ok]), "kNN distances differ"
    assert np.array_equal(d["plane"][ok], o["plane"][ok]), "plane parameters differ (bit-exact expected)"
    m = ctx.get_matches(k, Q)
    v = o["status"] == oracle.GO_VALID
    assert m["n"] == o["nvalid"] == int(v.sum())
    assert np.array_equal(m["src"], np.nonzero(v)[0].astype(np.int32))
    assert np.array_equal(m["cp"], P["scans"][k][v])
    assert np.array_equal(m["nsd"], o["nsd"][v])
    assert np.array_equal(m["weight"], o["weight"][v])
    return o


@pytest.mark.parametrize("W,Q,M,seed", [(3, 2000, 30000, 11), (5, 1000, 50000, synth.SEED0 + 1)])
def test_scan_to_map_single_slot_calls(ctx, oracle, W, Q, M, seed):
    P = synth.window_problem(W=W, Q=Q, M=M, seed=seed)
    ctx.set_map(P["map_xyz"])
    tree = oracle.KdTree(P["map_xyz"])
    for k in range(W):
        t2, q2 = ctx.lidar_pose(P["poses_init"][k])
        n = ctx.assoc_scan_to_map(k, P["scans"][k], t2, q2)
        o = _check_slot(ctx, oracle, P, k, t2, q2, tree)
        assert n == o["nvalid"]


def test_window_associate_equals_single_calls(ctx, oracle):
    P = synth.window_problem(W=4, Q=3000, M=40000, seed=5)
    ctx.set_map(P["map_xyz"])
    tree = oracle.KdTree(P["map_xyz"])
    ctx.window_set_scans(P["scans"])
    nm = ctx.window_associate(P["poses_init"])
    for k in range(4):
        t2, q2 = ctx.lidar_pose(P["poses_init"][k])
        o = _check_slot(ctx, oracle, P, k, t2, q2, tree)
        assert nm[k] == o["nvalid"]


def test_window_slide_equals_fresh_window(ctx, oracle):
    """slideWindow on the device: after glio_window_slide + one new scan in the last slot, the association of the shifted
    window equals the association of the same keyframes handed over from scratch (scans and matches moved with their slots)."""
    W = 4
    P = synth.window_problem(W=W + 1, Q=2500, M=40000, seed=23)
    ctx.set_map(P["map_xyz"])
    ctx.window_set_scans(P["scans"][:W])
    ctx.window_associate(P["poses_init"][:W])
    ctx.window_slide(W)
    ctx.window_set_scan(W - 1, P["scans"][W])
    nm = ctx.window_associate(P["poses_init"][1:W + 1])
    snap = [(ctx.get_assoc_debug(k, 2500), ctx.get_matches(k, 2500)) for k in range(W)]
    ctx.window_set_scans(P["scans"][1:W + 1])
    nm2 = ctx.window_associate(P["poses_init"][1:W + 1])
    assert np.array_equal(nm, nm2)
    for k in range(W):
        d, m = ctx.get_assoc_debug(k, 2500), ctx.get_matches(k, 2500)
        for key in ("status", "idx5", "sqd5", "plane"):
            assert np.array_equal(d[key], snap[k][0][key])
        for key in ("cp", "nsd", "weight", "src"):
            assert np.array_equal(m[key], snap[k][1][key])


def test_map_prefetch_equals_inline_upload(ctx, oracle):
    """glio_map_prefetch + glio_set_map (staged copy, copy stream) gives the association of the in-line upload; a prefetch that
    does not match the following set_map (other pointer) is ignored."""
    P = synth.window_problem(W=2, Q=2000, M=30000, seed=29)
    other = synth.window_problem(W=1, Q=10, M=30000, seed=30)["map_xyz"]
    ctx.window_set_scans(P["scans"])
    ctx.set_map(P["map_xyz"])
    nm0 = ctx.window_associate(P["poses_init"]); d0 = ctx.get_assoc_debug(1, 2000)
    m = np.ascontiguousarray(P["map_xyz"])
    ctx.map_prefetch(m); ctx.set_map(m)
    nm1 = ctx.window_associate(P["poses_init"]); d1 = ctx.get_assoc_debug(1, 2000)
    ctx.map_prefetch(other); ctx.set_map(m)                 # stale prefetch of another buffer: the in-line path is taken
    nm2 = ctx.window_associate(P["poses_init"]); d2 = ctx.get_assoc_debug(1, 2000)
    assert np.array_equal(nm0, nm1) and np.array_equal(nm0, nm2)
    for k in ("status", "idx5", "sqd5", "plane"):
        assert np.array_equal(d0[k], d1[k]) and np.array_equal(d0[k], d2[k])


def test_displaced_keyframe_search_is_bit_exact(oracle):
    """the K1a box search gives the oracle's association bit for bit when one keyframe is displaced: the pose error is large
    enough that many queries grow their box beyond the 3x3x3 start box"""
    from glio_b200 import api
    P = synth.window_problem(W=3, Q=6000, M=120000, seed=91)
    poses = P["poses_init"].copy()
    poses[1, :3] += [0.35, -0.2, 0.15]                      # displaced keyframe: many queries leave their start box
    c = api.Context(0, keep_debug=1)
    try:
        c.set_map(P["map_xyz"])
        tree = oracle.KdTree(P["map_xyz"])
        c.window_set_scans(P["scans"])
        nm = c.window_associate(poses)
        for k in range(3):
            t2, q2 = c.lidar_pose(poses[k])
            o = _check_slot(c, oracle, P, k, t2, q2, tree)
            assert nm[k] == o["nvalid"]
        assert nm.sum() > 3000
    finally:
        c.close()
