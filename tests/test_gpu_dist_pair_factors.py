"""Keyframe-sharded batch solves with the device pair-factor lists: two ranks (torchrun, gloo, rendezvous on 127.0.0.1) share the one
GPU, pass the same pose (and DD pseudorange) lists with their own active masks (the rank that owns a factor's lower keyframe
evaluates it) and the plane matches of their own pairs; the all-reduce hook sums the K x 28 and (P + P_pose [+ P_dd]) x 36
buffers.  The sharded glio_eval_pose_factors / glio_eval_dd_psr_factors and solve must reproduce the single-rank ones."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "workers", "batch_pair_factor_shard_worker.py")


def _run(tmp_path, world, tag, kind, port):
    out = str(tmp_path / tag)
    env = dict(os.environ); env["OMP_NUM_THREADS"] = "4"
    if world == 1:
        subprocess.check_call([sys.executable, WORKER, out, kind], env=env, timeout=600)
    else:
        subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                               "--master-port", str(port), WORKER, out, kind], env=env, timeout=600)
    return [json.load(open(out + f".rank{r}.json")) for r in range(world)]


def test_sharded_batch_solve_with_pose_factors_equals_single_rank(tmp_path):
    one = _run(tmp_path, 1, "one", "pose", 29631)[0]
    two = _run(tmp_path, 2, "two", "pose", 29631)
    # each factor and each pair's matches on exactly one rank
    assert 0 < two[0]["n_active"] < one["n_active"] == one["n_factors"] and two[0]["n_active"] + two[1]["n_active"] == one["n_active"]
    assert 0 < two[0]["n_match_own"] and two[0]["n_match_own"] + two[1]["n_match_own"] == one["n_match_own"]
    for r in two:
        assert r["n_pose_pairs"] == one["n_pose_pairs"]
        # glio_eval_pose_factors: one all-reduce per buffer; the solve's off-diagonal buffer holds the LiDAR and the pose pairs
        assert r["eval_hook_calls"] == 2 and r["hook_calls"] == two[0]["hook_calls"]
        assert (r["n_pairs"] + r["n_pose_pairs"]) * 36 in r["hook_counts"] and r["n_pose_pairs"] * 36 in r["hook_counts"]
        for k in ("Hdiag", "Hoff", "g"):
            a, b = np.array(r["eval"][k]), np.array(one["eval"][k])
            assert np.max(np.abs(a - b)) <= 1e-12 * np.max(np.abs(b))
        assert abs(r["eval"]["cost"] - one["eval"]["cost"]) <= 1e-12 * abs(one["eval"]["cost"])
        assert r["iterations"] == one["iterations"] >= 3
        assert abs(r["final_cost"] - one["final_cost"]) <= 1e-9 * abs(one["final_cost"])
        assert np.max(np.abs(np.array(r["poses"])[:, :3] - np.array(one["poses"])[:, :3])) <= 1e-7
        assert np.max(np.abs(np.array(r["poses"])[:, 3:] - np.array(one["poses"])[:, 3:])) <= 1e-8
    assert np.array_equal(np.array(two[0]["poses"]), np.array(two[1]["poses"]))


def test_sharded_batch_solve_with_dd_factors_equals_single_rank(tmp_path):
    one = _run(tmp_path, 1, "one", "dd", 29641)[0]
    two = _run(tmp_path, 2, "two", "dd", 29641)
    # each DD factor and each pair's matches on exactly one rank
    assert 0 < two[0]["n_active"] < one["n_active"] == one["n_factors"] and two[0]["n_active"] + two[1]["n_active"] == one["n_active"]
    assert 0 < two[0]["n_match_own"] and two[0]["n_match_own"] + two[1]["n_match_own"] == one["n_match_own"]
    for r in two:
        assert r["n_dd_pairs"] == one["n_dd_pairs"] > 0 and r["n_pose_pairs"] == one["n_pose_pairs"]
        # glio_eval_dd_psr_factors: one all-reduce per buffer; the solve's off-diagonal buffer holds LiDAR, pose and DD pairs
        assert r["eval_hook_calls"] == 2 and r["hook_calls"] == two[0]["hook_calls"]
        assert (r["n_pairs"] + r["n_pose_pairs"] + r["n_dd_pairs"]) * 36 in r["hook_counts"] and r["n_dd_pairs"] * 36 in r["hook_counts"]
        for k in ("Hdiag", "Hoff", "g"):
            a, b = np.array(r["eval"][k]), np.array(one["eval"][k])
            assert np.max(np.abs(a - b)) <= 1e-12 * np.max(np.abs(b))
        assert abs(r["eval"]["cost"] - one["eval"]["cost"]) <= 1e-12 * abs(one["eval"]["cost"])
        assert r["iterations"] == one["iterations"] >= 3
        assert abs(r["final_cost"] - one["final_cost"]) <= 1e-9 * abs(one["final_cost"])
        assert np.max(np.abs(np.array(r["poses"])[:, :3] - np.array(one["poses"])[:, :3])) <= 1e-7
        assert np.max(np.abs(np.array(r["poses"])[:, 3:] - np.array(one["poses"])[:, 3:])) <= 1e-8
    assert np.array_equal(np.array(two[0]["poses"]), np.array(two[1]["poses"]))
