"""Keyframe-sharded level-1 batch solve with the IMU factors on the device: two ranks (torchrun, gloo, rendezvous on 127.0.0.1)
share the one GPU, pass the same attitude and IMU lists with their own active masks (the rank that owns a factor's lower keyframe
evaluates it) and the plane matches of their own pairs; the all-reduce hook sums the 6-column buffers and then the IMU buffers
(K x 241 and P_imu x 225), one call per buffer.  The sharded glio_eval_imu_factors and solve must reproduce the single-rank ones."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "workers", "batch_imu_shard_worker.py")


def _run(tmp_path, world, tag, port):
    out = str(tmp_path / tag)
    env = dict(os.environ); env["OMP_NUM_THREADS"] = "4"
    if world == 1:
        subprocess.check_call([sys.executable, WORKER, out], env=env, timeout=600)
    else:
        subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                               "--master-port", str(port), WORKER, out], env=env, timeout=600)
    return [json.load(open(out + f".rank{r}.json")) for r in range(world)]


def test_sharded_batch_solve_with_imu_factors_equals_single_rank(tmp_path):
    one = _run(tmp_path, 1, "one", 29651)[0]
    two = _run(tmp_path, 2, "two", 29651)
    assert 0 < two[0]["n_active"] < one["n_active"] == one["n_factors"] and two[0]["n_active"] + two[1]["n_active"] == one["n_active"]
    assert 0 < two[0]["n_match_own"] and two[0]["n_match_own"] + two[1]["n_match_own"] == one["n_match_own"]
    K = len(one["poses"])
    for r in two:
        assert r["n_imu_pairs"] == one["n_imu_pairs"] == K - 1
        # glio_eval_imu_factors: one all-reduce per IMU buffer; the solve reduces the IMU buffers as well
        assert r["eval_hook_calls"] == 2 and r["hook_calls"] == two[0]["hook_calls"]
        assert K * 241 in r["hook_counts"] and r["n_imu_pairs"] * 225 in r["hook_counts"]
        for k in ("Hdiag", "Hoff", "g"):
            a, b = np.array(r["eval"][k]), np.array(one["eval"][k])
            assert np.max(np.abs(a - b)) <= 1e-12 * np.max(np.abs(b))
        assert abs(r["eval"]["cost"] - one["eval"]["cost"]) <= 1e-12 * abs(one["eval"]["cost"])
        assert r["iterations"] == one["iterations"] >= 3 and r["termination"] == one["termination"]
        assert abs(r["final_cost"] - one["final_cost"]) <= 1e-9 * abs(one["final_cost"])
        assert np.max(np.abs(np.array(r["poses"])[:, :3] - np.array(one["poses"])[:, :3])) <= 1e-7
        assert np.max(np.abs(np.array(r["poses"])[:, 3:] - np.array(one["poses"])[:, 3:])) <= 1e-8
    assert np.array_equal(np.array(two[0]["poses"]), np.array(two[1]["poses"]))
