"""Worker of tests/test_gpu_dist_band_bcr.py: one rank of a keyframe-sharded batch solve with the device minimizer and the block
cyclic reduction (glio_batch_use_device_solver, GLIO_FACTOR_BCR), on tests/workers/batch_device_solve_shard_worker.py's two problems
(level 1 and level 0, K = 30, search range 3).  Every rank solves the whole band from the block buffers the all-reduce hook has
summed.  Writes each problem's solve and the hook calls it made."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    out_path = sys.argv[1]
    import torch
    import torch.distributed as dist
    from glio_b200 import api, dist as gdist, synth
    from tests import eval_reference as er
    from tests import gloo_hook
    from tests.workers import batch_device_solve_shard_worker as w
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        dist.init_process_group("gloo")
    torch.cuda.set_device(0)
    K, sr = 30, 3
    res = dict(rank=rank, world=world)
    for name, setup in (("level1", w._level1), ("level0", w._level0)):
        ctx = api.Context(0)
        cb, calls, counts = gloo_hook.staging_allreduce()
        if world > 1:
            ctx.set_allreduce(cb, None)
        poses, sb, hf = setup(api, gdist, synth, er, ctx, K, sr, rank, world)
        ctx.batch_use_device_solver(True); ctx.batch_device_factorization(api.FACTOR_BCR)
        before = calls[0]
        r = ctx.batch_solve(poses, sb, hf, api.batch_solver_options(max_num_iterations=12))
        s = r["summary"]
        res[name] = dict(hook_calls=calls[0] - before, initial_cost=float(s.initial_cost), final_cost=float(s.final_cost),
                         iterations=int(s.num_iterations), termination=int(s.termination),
                         steps_ok=[int(it["step_is_successful"]) for it in r["iterations"]], poses=r["poses"].tolist(),
                         poses_hex=[float(v).hex() for v in r["poses"].reshape(-1)])
        ctx.close()
    if world > 1:
        dist.destroy_process_group()
    with open(out_path + f".rank{rank}.json", "w") as fo:
        json.dump(res, fo)


if __name__ == "__main__":
    main()
