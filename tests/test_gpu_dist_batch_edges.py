"""A keyframe-sharded batch solve with binary edge factors: two ranks (torchrun, gloo, rendezvous on 127.0.0.1) share the one GPU,
each associates the planes and edges of its own pairs, and the all-reduce hook sums the K x 28 / P x 36 buffers, which carry the
plane and edge blocks together.  The sharded solve must reproduce the single-rank solve."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "workers", "batch_edge_shard_worker.py")


def _run(tmp_path, world, tag):
    out = str(tmp_path / tag)
    env = dict(os.environ); env["OMP_NUM_THREADS"] = "4"
    if world == 1:
        subprocess.check_call([sys.executable, WORKER, out], env=env, timeout=600)
    else:
        subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                               "--master-port", "29617", WORKER, out], env=env, timeout=600)
    return [json.load(open(out + f".rank{r}.json")) for r in range(world)]


def test_sharded_batch_solve_with_edges_equals_single_rank(tmp_path):
    one = _run(tmp_path, 1, "one")[0]
    two = _run(tmp_path, 2, "two")
    assert two[0]["hook_calls"] > 0 and two[0]["hook_calls"] == two[1]["hook_calls"]
    assert 0 < two[0]["n_edge_own"] < one["n_edge_own"] and two[0]["n_edge_own"] + two[1]["n_edge_own"] == one["n_edge_own"]
    for r in two:
        assert r["iterations"] == one["iterations"] >= 3
        assert abs(r["final_cost"] - one["final_cost"]) <= 1e-9 * abs(one["final_cost"])
        assert np.max(np.abs(np.array(r["poses"])[:, :3] - np.array(one["poses"])[:, :3])) <= 1e-7
        assert np.max(np.abs(np.array(r["poses"])[:, 3:] - np.array(one["poses"])[:, 3:])) <= 1e-8
    assert np.array_equal(np.array(two[0]["poses"]), np.array(two[1]["poses"]))
