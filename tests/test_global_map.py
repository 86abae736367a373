"""The references of the sort-based VoxelGrid and of save_pcd's global map, checked on the CPU: the oracle's stable voxel filter
(pyoracle.voxel_filter) and its global map (tests/global_map_reference.global_map, built on the oracle primitives) against an
independent numpy formulation, bit for bit, on boxes below and above 2^28 voxels, at both sides of PCL's INT32_MAX leaf-size
check, on voxel keys that wrap past 2^32 or go negative in int32, and on a loop drive's keyframe store.
tests/test_gpu_global_map.py runs the device against the oracle on the same fixtures."""
import numpy as np
import pytest

from glio_b200 import synth
from tests.global_map_reference import (ABOVE_INT32_MAX, BELOW_INT32_MAX, F32, KEY_BIT_BOXES, NEGATIVE_KEY_BOX, box_cloud, concatenation,
                                        global_map, np_global_map, np_transform, np_voxel_filter, np_voxel_keys, wrap_cloud)


# a tilted extrinsic: with the shipped one (identity rotation) Tbl only shifts z, and the extra rounding rarely shows
EXTRINSIC = dict(q_lb=synth.quat_from_rpy(0.01, -0.015, 0.02), t_lb=(0.1, -0.05, 0.28))


@pytest.fixture(scope="module")
def pl():
    from oracle import pyoracle_loop
    return pyoracle_loop


def oracle_filter(po, x, leaf):
    r = po.voxel_filter(x, leaf, stable=True)
    return (x, False) if r is None else (r[0], True)


def assert_same_filter(po, x, leaf, filtered=True):
    got, f = oracle_filter(po, x, leaf)
    ref, g = np_voxel_filter(x, leaf)
    assert f == g == filtered
    assert got.shape == ref.shape and np.array_equal(got, ref)
    return ref


def test_transform_matches_the_oracle(oracle):
    rng = np.random.default_rng(1)
    x = rng.uniform(-50, 50, (20000, 3)).astype(F32)
    for off in (0.0, 3000.0, 20000.0):
        q = synth.quat_from_rpy(*rng.uniform(-np.pi, np.pi, 3)); t = rng.uniform(-1, 1, 3) * off + rng.uniform(-5, 5, 3)
        assert np.array_equal(np_transform(x, t, q), oracle.transform_points(x, t, q))


@pytest.mark.parametrize("leaf", [0.9, 0.4, 0.2])
def test_voxel_filter_below_2_28_voxels(oracle, leaf):
    rng = np.random.default_rng(int(leaf * 10))
    x = np.concatenate([rng.uniform(-40, 40, (30000, 3)), rng.normal(0, 3, (20000, 3))]).astype(F32)
    key, ok = np_voxel_keys(x, leaf)
    assert ok
    ref = assert_same_filter(oracle, x, leaf)
    assert len(ref) < len(x)


def test_voxel_filter_above_2_28_voxels(oracle):
    """the cloud the dense filter refuses: 3921 x 3921 x 41 voxels at leaf 1"""
    rng = np.random.default_rng(34)
    x = np.concatenate([[[3900.5, 3900.5, 0.5]], rng.uniform(-20, 20, (20000, 3))]).astype(F32)
    mn = np.floor(x.min(0)); mx = np.floor(x.max(0))
    assert np.prod(mx - mn + 1) > 2**28
    assert_same_filter(oracle, x, 1.0)


def test_leaf_size_check_at_int32_max(oracle):
    lo, hi = BELOW_INT32_MAX
    x = box_cloud(lo, hi, 3000, seed=2)
    assert_same_filter(oracle, x, 1.0, filtered=True)
    lo, hi = ABOVE_INT32_MAX
    x = box_cloud(lo, hi, 3000, seed=3)
    assert oracle.voxel_filter(x, 1.0) is None
    assert_same_filter(oracle, x, 1.0, filtered=False)


def test_wrapped_and_negative_keys(oracle):
    x = wrap_cloud()
    key, ok = np_voxel_keys(x, 1.0)
    assert ok
    z = x[:, 2]
    merged = np.intersect1d(key[z < 4], key[z > 1e9])
    assert len(merged) > 0                                   # voxels 2^30 apart share a key after the wrap
    assert_same_filter(oracle, x, 1.0)
    lo, hi = NEGATIVE_KEY_BOX
    x = box_cloud(lo, hi, 5000, seed=4)
    key, ok = np_voxel_keys(x, 1.0)
    assert ok and key.max() > 2**31                            # negative as int32, last in the unsigned order
    assert_same_filter(oracle, x, 1.0)


@pytest.mark.parametrize("bits", sorted(KEY_BIT_BOXES))
def test_key_width_boxes(oracle, bits):
    lo, hi = KEY_BIT_BOXES[bits]
    x = box_cloud(lo, hi, 4000, seed=bits)
    key, ok = np_voxel_keys(x, 1.0)
    assert ok and int(key.max()).bit_length() == bits
    assert_same_filter(oracle, x, 1.0)


def test_one_far_voxel_sums_in_input_order(oracle):
    rng = np.random.default_rng(6)
    c = np.array([1000.3, -1000.3, 40.3])
    x = (c + rng.uniform(-0.08, 0.08, (5000, 3))).astype(F32)
    ref = assert_same_filter(oracle, x, 0.2)
    assert len(ref) == 1
    lit = oracle.voxel_filter(x, 0.2, stable=False)[0]
    assert not np.array_equal(lit, ref)                        # std::sort's order gives other bits: the stable order is pinned


@pytest.mark.parametrize("interval,leaf", [(1, 0.2), (3, 0.2), (3, 0.4)])
def test_global_map_matches_numpy(oracle, pl, interval, leaf):
    D = synth.loop_drive(K=40, n_points=1500, dt=1.0, seed=synth.SEED0 + 41)
    L = pl.LoopOracle()
    for k in range(D["K"]):
        L.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
    for stage in range(2):
        got = global_map(oracle, L, interval, leaf)
        ref = np_global_map(L.clouds, L.poses, L.q_bl, L.t_bl, interval, leaf)
        assert got[1] == ref[1] and got[2] == ref[2] == sum(len(c) for c in L.clouds[::interval])
        assert np.array_equal(got[0], ref[0])
        new = np.array(L.poses); new[:, 0] += 0.05; new[:, 1] -= 0.02
        L.set_poses(0, new)


def test_two_transforms_differ_from_the_combined_pose(oracle, pl):
    D = synth.loop_drive(K=20, n_points=1500, dt=1.0, seed=synth.SEED0 + 42)
    L = pl.LoopOracle(**EXTRINSIC)
    for k in range(D["K"]):
        L.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
    two = concatenation(oracle, L, 1)
    one = np.concatenate([oracle.transform_points(L.clouds[i], *map(np.array, pl.world_of_cloud(L.poses[i], L.q_bl, L.t_bl)))
                          for i in range(len(L.clouds))])
    assert two.shape == one.shape and not np.array_equal(two, one)
