"""Worker of tests/test_gpu_dist_product.py: one rank of a keyframe-sharded batch solve of the PRODUCT (glio_set_allreduce,
glio_batch_declare_pairs, glio_batch_associate_pairs on owned pairs, glio_batch_solve).  Both ranks may share one GPU: the
all-reduce hook is tests/gloo_hook.py's, which stages the device buffer through the host and sums it with torch.distributed (gloo)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    out_path = sys.argv[1]
    import torch
    import torch.distributed as dist
    from glio_b200 import api, dist as gdist, synth
    from tests import gloo_hook
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        dist.init_process_group("gloo")
    torch.cuda.set_device(0)
    K, Q, sr = 10, 3000, 2
    cur, oth = gdist.batch_pairs(K, sr)
    own = gdist.owner_of(cur, K, world) == rank
    need = gdist.frames_needed(cur, oth, own)
    B = synth.batch_problem(K=K, Q=Q, seed=77, search_range=sr, rng_range=6.0, frames=need)
    ctx = api.Context(0)
    cb, calls, _ = gloo_hook.staging_allreduce()
    if world > 1:
        ctx.set_allreduce(cb, None)
    for k in need:
        ctx.batch_set_frame(int(k), B["scans"][k], B["poses_init"][k])
    ctx.batch_declare_pairs(cur, oth)
    nm = ctx.batch_associate_pairs(cur[own], oth[own])
    hf = api.HostFactorSet(); T = B["poses_true"]; rng = np.random.default_rng(7)
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.zeros(9)])
    hf.add_prior(0, T[0, :3], T[0, 3:], None, sw * 3)
    for i in range(K - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        hf.add_between(i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw)
    ev = ctx.eval_binary(B["poses_init"])
    r = ctx.batch_solve(B["poses_init"], None, hf, api.batch_solver_options(max_num_iterations=12))
    s = r["summary"]
    res = dict(rank=rank, world=world, n_match_own=int(nm.sum()), hook_calls=calls[0], initial_cost=float(s.initial_cost), final_cost=float(s.final_cost),
               iterations=int(s.num_iterations), poses=r["poses"].tolist(), steps=[st.tolist() for st in r["steps"]],
               eval_cost=ev["cost"], eval_g=ev["g"].tolist(), eval_Hdiag=ev["Hdiag"].tolist())
    ctx.close()
    if world > 1:
        tot = torch.tensor([float(nm.sum())]); dist.all_reduce(tot); res["n_match_total"] = float(tot.item())
        dist.destroy_process_group()
    else:
        res["n_match_total"] = float(nm.sum())
    with open(out_path + f".rank{rank}.json", "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    main()
