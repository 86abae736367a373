"""Keyframe-sharded batch solve with the device minimizer's block cyclic reduction: two ranks (torchrun, gloo, rendezvous on
127.0.0.1) share the one GPU, and every rank runs the same deterministic reduction on the same summed band.  Both ranks must end
with bit-identical poses, each equal to the single-rank solve by tests/test_gpu_dist_device_solve.py's criteria."""
import json
import os
import subprocess
import sys

import pytest

from tests.test_gpu_dist_device_solve import _same_solve

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "workers", "batch_bcr_shard_worker.py")


def _run(tmp_path, world, tag, port):
    out = str(tmp_path / tag)
    env = dict(os.environ); env["OMP_NUM_THREADS"] = "4"
    if world == 1:
        subprocess.check_call([sys.executable, WORKER, out], env=env, timeout=600)
    else:
        subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                               "--master-port", str(port), WORKER, out], env=env, timeout=600)
    return [json.load(open(out + f".rank{r}.json")) for r in range(world)]


def test_sharded_bcr_solve_equals_single_rank(tmp_path):
    one = _run(tmp_path, 1, "one", 29657)[0]
    two = _run(tmp_path, 2, "two", 29657)
    assert [r["rank"] for r in two] == [0, 1]
    for level in ("level1", "level0"):
        assert one[level]["hook_calls"] == 0
        for r in two:
            assert r[level]["hook_calls"] > 0
            _same_solve(r[level], one[level])
        assert two[0][level]["poses_hex"] == two[1][level]["poses_hex"], level
