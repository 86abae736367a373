"""Worker of tests/test_gpu_dist_device_solve.py: one rank of a keyframe-sharded batch solve with the device minimizer
(glio_batch_use_device_solver), next to the same rank's sharded host solve.  Two problems, K = 30 and search range 3:
- level 1: LiDAR plane pairs, attitude factors and IMU factors (tests/workers/batch_imu_shard_worker.py's problem);
- level 0: LiDAR plane pairs, pose factors and DD pseudorange factors (tests/workers/batch_pair_factor_shard_worker.py's "dd").
Every rank declares the same pairs and passes the same lists; a rank uploads the plane matches of the pairs whose cur it owns
(dist.owner_of) and marks active the factors whose lower keyframe it owns (dist.pose_factor_active).  Both ranks may share one GPU
through tests/gloo_hook.py's all-reduce hook.  The device minimizer assembles its band from the buffers the hook has summed, so
every rank must solve the whole problem.  Writes both solves of both problems and the hook calls each made."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def _level1(api, gdist, synth, er, ctx, K, sr, rank, world):
    P = synth.imu_problem(K=K, search_range=sr, seed=93)
    cur, oth = P["pairs"]
    own = gdist.owner_of(cur, K, world) == rank
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"], active=gdist.pose_factor_active(P["i"], P["j"], K, world, rank))
    f = api.imu_factor_records(**P["imu"], active=gdist.pose_factor_active(P["imu"]["i"], P["imu"]["j"], K, world, rank))
    ctx.batch_declare_pairs(cur, oth)
    for k, (a, b) in enumerate(zip(cur, oth)):
        if own[k]:
            m = er.make_pair(np.random.default_rng([93, int(a), int(b)]), P["poses_true"][a], P["poses_true"][b], 30, noise=0.02)
            ctx.batch_set_pair_matches(int(a), int(b), m["cp"], m["nc"], m["weight"])
    ctx.batch_set_pose_factors(pf); ctx.batch_use_pose_factors(True)
    ctx.batch_set_imu_factors(f); ctx.batch_use_imu_factors(True)
    hf = api.HostFactorSet(); T = P["poses_true"]
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)])
    hf.add_prior(0, T[0, :3], T[0, 3:], P["sb_true"][0], sw * 3)
    return P["poses_init"], P["sb_init"], hf


def _level0(api, gdist, synth, er, ctx, K, sr, rank, world):
    P = synth.dd_psr_problem(K=K, search_range=sr, seed=91)
    cur, oth = gdist.batch_pairs(K, sr)
    own = gdist.owner_of(cur, K, world) == rank
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"], active=gdist.pose_factor_active(P["i"], P["j"], K, world, rank))
    f = api.dd_psr_factor_records(**P["dd"], active=gdist.pose_factor_active(P["dd"]["i"], P["dd"]["j"], K, world, rank))
    ctx.batch_declare_pairs(cur, oth)
    for k, (a, b) in enumerate(zip(cur, oth)):
        if own[k]:
            m = er.make_pair(np.random.default_rng([91, int(a), int(b)]), P["poses_true"][a], P["poses_true"][b], 30, noise=0.02)
            ctx.batch_set_pair_matches(int(a), int(b), m["cp"], m["nc"], m["weight"])
    ctx.batch_set_pose_factors(pf); ctx.batch_use_pose_factors(True)
    ctx.batch_set_dd_psr_factors(f, api.dd_psr_sat_records(**P["dd_sats"]), P["R"], P["anchor"]); ctx.batch_use_dd_psr_factors(True)
    hf = api.HostFactorSet(); T = P["poses_true"]
    hf.add_prior(0, T[0, :3], T[0, 3:], None, np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.zeros(9)]))
    return P["poses_init"], None, hf


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
    res = dict(rank=rank, world=world)
    for name, setup in (("level1", _level1), ("level0", _level0)):
        ctx = api.Context(0)
        cb, calls, counts = gloo_hook.staging_allreduce()
        if world > 1:
            ctx.set_allreduce(cb, None)
        poses, sb, hf = setup(api, gdist, synth, er, ctx, K, sr, rank, world)
        hb = ctx.batch_normal_equations(poses, sb, hf)[0].shape[1] - 1         # collective as well: every rank evaluates
        assert hb <= api.BAND_MAX_HB, hb
        out = dict(hb=hb)
        for path, on in (("host", False), ("device", True)):
            ctx.batch_use_device_solver(on)
            before = calls[0]
            r = ctx.batch_solve(poses, sb, hf, api.batch_solver_options(max_num_iterations=12))
            s = r["summary"]
            out[path] = dict(hook_calls=calls[0] - before, initial_cost=float(s.initial_cost), final_cost=float(s.final_cost),
                             iterations=int(s.num_iterations), termination=int(s.termination),
                             steps_ok=[int(it["step_is_successful"]) for it in r["iterations"]], poses=r["poses"].tolist(),
                             poses_hex=[float(v).hex() for v in r["poses"].reshape(-1)])
        res[name] = out
        ctx.close()
    if world > 1:
        dist.destroy_process_group()
    with open(out_path + f".rank{rank}.json", "w") as fo:
        json.dump(res, fo)


if __name__ == "__main__":
    main()
