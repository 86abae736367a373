"""Worker of tests/test_gpu_edge_select.py: one rank of a keyframe-sharded batch solve with binary edge factors and seeded edge
selection (glio_batch_associate_edges_pairs and glio_batch_select_random_edges on owned pairs only, glio_batch_use_edges,
glio_batch_solve).  Both ranks may share one GPU through tests/gloo_hook.py's all-reduce hook."""
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
    K, sr = 10, 2
    cur, oth = gdist.batch_pairs(K, sr)
    own = gdist.owner_of(cur, K, world) == rank
    need = gdist.frames_needed(cur, oth, own)
    B = synth.batch_problem(K=K, Q=3000, seed=78, search_range=sr, rng_range=6.0, frames=need)
    E = synth.batch_edge_problem(K=K, Q=2000, seed=78, search_range=sr, frames=need, rng_range=6.0)
    ctx = api.Context(0)
    cb, calls, _ = gloo_hook.staging_allreduce()
    if world > 1:
        ctx.set_allreduce(cb, None)
    for k in need:
        ctx.batch_set_frame(int(k), B["scans"][k], B["poses_init"][k])
        ctx.batch_set_edge_frame(int(k), E["corner_scans"][k])
    ctx.batch_declare_pairs(cur, oth)
    nm = ctx.batch_associate_pairs(cur[own], oth[own])
    ne = ctx.batch_associate_edges_pairs(cur[own], oth[own])
    # each rank selects its own pairs only: the streams (cur << 32 | oth) make the lists those of a single context
    opt = api.select_default_options(batch_feature_res_num=40, batch_rand_set_num=400, seed=5, nonce=3)
    ctx.batch_select_random(cur[own], oth[own], 0, opt)
    na = ctx.batch_select_random_edges(cur[own], oth[own], 0, opt)
    sel = []
    for c, o in zip(cur[own], oth[own]):
        keep = ctx.batch_get_edge_selection(int(c), int(o))
        sel.append([[int(c), int(o)], None if keep is None else keep.tolist()])
    ctx.batch_use_edges(True)
    hf = api.HostFactorSet(); T = B["poses_true"]; rng = np.random.default_rng(7)
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.zeros(9)])
    hf.add_prior(0, T[0, :3], T[0, 3:], None, sw * 3)
    for i in range(K - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        hf.add_between(i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw)
    r = ctx.batch_solve(B["poses_init"], None, hf, api.batch_solver_options(max_num_iterations=12))
    s = r["summary"]
    res = dict(rank=rank, world=world, n_match_own=int(nm.sum()), n_edge_own=int(ne.sum()), n_edge_active=int(na.sum()),
               edge_selection=sel, hook_calls=calls[0], initial_cost=float(s.initial_cost), final_cost=float(s.final_cost),
               iterations=int(s.num_iterations), poses=r["poses"].tolist())
    ctx.close()
    if world > 1:
        dist.destroy_process_group()
    with open(out_path + f".rank{rank}.json", "w") as f:
        json.dump(res, f)


if __name__ == "__main__":
    main()
