"""Keyframe-sharded batch solve with the device minimizer: two ranks (torchrun, gloo, rendezvous on 127.0.0.1) share the one GPU
and every rank assembles its band on the device from the block buffers the all-reduce hook has summed in place.  At level 1
(LiDAR pairs, attitude and IMU factors) and at level 0 (LiDAR pairs, pose and DD pseudorange factors), each rank's device solve
must reproduce the single-rank device solve and the sharded host solve, with as many hook calls as the host solve, and both ranks
must end with bit-identical poses."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "workers", "batch_device_solve_shard_worker.py")


def _run(tmp_path, world, tag, port):
    out = str(tmp_path / tag)
    env = dict(os.environ); env["OMP_NUM_THREADS"] = "4"
    if world == 1:
        subprocess.check_call([sys.executable, WORKER, out], env=env, timeout=600)
    else:
        subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                               "--master-port", str(port), WORKER, out], env=env, timeout=600)
    return [json.load(open(out + f".rank{r}.json")) for r in range(world)]


def _same_solve(a, b):
    assert a["iterations"] == b["iterations"] >= 3 and a["termination"] == b["termination"] and a["steps_ok"] == b["steps_ok"]
    assert abs(a["final_cost"] - b["final_cost"]) <= 1e-9 * abs(b["final_cost"]) and a["final_cost"] < a["initial_cost"]
    pa, pb = np.array(a["poses"]), np.array(b["poses"])
    assert np.max(np.abs(pa[:, :3] - pb[:, :3])) <= 1e-7
    assert np.max(np.abs(pa[:, 3:] - pb[:, 3:])) <= 1e-8


def test_sharded_device_solve_equals_single_rank_and_sharded_host(tmp_path):
    one = _run(tmp_path, 1, "one", 29653)[0]
    two = _run(tmp_path, 2, "two", 29653)
    assert one["world"] == 1 and [r["world"] for r in two] == [2, 2] and [r["rank"] for r in two] == [0, 1]
    for level in ("level1", "level0"):
        assert one[level]["host"]["hook_calls"] == one[level]["device"]["hook_calls"] == 0
        for r in two:
            o = r[level]
            assert o["hb"] == one[level]["hb"]
            assert o["device"]["hook_calls"] == o["host"]["hook_calls"] > 0
            _same_solve(o["device"], one[level]["device"])
            _same_solve(o["device"], o["host"])
        assert two[0][level]["device"]["poses_hex"] == two[1][level]["device"]["poses_hex"], level
