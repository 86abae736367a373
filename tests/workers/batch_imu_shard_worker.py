"""Worker of tests/test_gpu_dist_imu_factors.py: one rank of a keyframe-sharded level-1 batch solve with LiDAR plane pairs, the
attitude factors and the IMU factors on the device.  Every rank declares the same pairs and passes the same lists; a rank uploads
the plane matches of the pairs whose cur it owns (dist.owner_of) and marks active the factors whose lower keyframe it owns
(dist.pose_factor_active).  Both ranks may share one GPU through tests/gloo_hook.py's all-reduce hook.  Writes the solve and one
glio_eval_imu_factors result."""
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
    from tests import eval_reference as er
    from tests import gloo_hook
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        dist.init_process_group("gloo")
    torch.cuda.set_device(0)
    K, sr = 30, 3
    P = synth.imu_problem(K=K, search_range=sr, seed=93)
    cur, oth = P["pairs"]
    own = gdist.owner_of(cur, K, world) == rank
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"], active=gdist.pose_factor_active(P["i"], P["j"], K, world, rank))
    active = gdist.pose_factor_active(P["imu"]["i"], P["imu"]["j"], K, world, rank)
    f = api.imu_factor_records(**P["imu"], active=active)
    ctx = api.Context(0)
    cb, calls, counts = gloo_hook.staging_allreduce()
    if world > 1:
        ctx.set_allreduce(cb, None)
    ctx.batch_declare_pairs(cur, oth)
    n_match = 0
    for k, (a, b) in enumerate(zip(cur, oth)):
        if own[k]:
            m = er.make_pair(np.random.default_rng([93, int(a), int(b)]), P["poses_true"][a], P["poses_true"][b], 30, noise=0.02)
            ctx.batch_set_pair_matches(int(a), int(b), m["cp"], m["nc"], m["weight"]); n_match += 30
    ctx.batch_set_pose_factors(pf); ctx.batch_use_pose_factors(True)
    ctx.batch_set_imu_factors(f); ctx.batch_use_imu_factors(True)
    e = ctx.eval_imu_factors(P["poses_init"], P["sb_init"])
    n_eval_calls = calls[0]
    hf = api.HostFactorSet(); T = P["poses_true"]
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)])
    hf.add_prior(0, T[0, :3], T[0, 3:], P["sb_true"][0], sw * 3)
    r = ctx.batch_solve(P["poses_init"], P["sb_init"], hf, api.batch_solver_options(max_num_iterations=12))
    s = r["summary"]
    res = dict(rank=rank, world=world, n_match_own=n_match, n_active=int(active.sum()), n_factors=len(f), n_pairs=len(cur),
               n_pose_pairs=len(ctx.batch_pose_pair_list()[0]), n_imu_pairs=len(ctx.batch_imu_pair_list()[0]), hook_calls=calls[0],
               eval_hook_calls=n_eval_calls, hook_counts=sorted(set(counts)),
               eval=dict(Hdiag=e["Hdiag"].tolist(), Hoff=e["Hoff"].tolist(), g=e["g"].tolist(), cost=e["cost"]),
               initial_cost=float(s.initial_cost), final_cost=float(s.final_cost), iterations=int(s.num_iterations),
               termination=int(s.termination), poses=r["poses"].tolist(), speed_bias=r["speed_bias"].tolist())
    ctx.close()
    if world > 1:
        dist.destroy_process_group()
    with open(out_path + f".rank{rank}.json", "w") as fo:
        json.dump(res, fo)


if __name__ == "__main__":
    main()
