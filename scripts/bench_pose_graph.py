#!/usr/bin/env python
"""The batch refinement's pose factors (K2p) at the reference's sms_fusion_level 0, on level-0 problems of K = 200, 2 000 and
3 457 keyframes (synth.pose_graph_problem: search range 6, about 22 factors per keyframe; 3 457 is the reference's sample run).
Reports, after warm-up: glio_eval_pose_factors, the median of --reps calls (host clock around the call, which ends in a stream
synchronisation); its two kernels, the mean over the same --reps launches (CUDA events on the context's stream, glio_profile_*,
which accumulates a total per kernel); glio_batch_solve of the level-0 problem with the pose factors on the device, the median
of --solve-reps solves (the reference's batch options: SUBSPACE_DOGLEG, nonmonotonic steps, at most --iters iterations; a prior
on keyframe 0 as the one host factor); the GPU's name and power limit, read in the same run.  Prints one JSON line."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--K", type=int, nargs="+", default=[200, 2000, 3457])
ap.add_argument("--iters", type=int, default=100)
ap.add_argument("--solve-reps", type=int, default=5)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_pose_graph.py needs a CUDA device")


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def kernel_ms(ctx, fn, names, reps):
    fn()
    ctx.lib_profile(True)
    for _ in range(reps):
        fn()
    prof = ctx.lib_profile_read(); ctx.lib_profile(False)
    return {n: round(prof[n][0] / prof[n][1], 4) for n in names if n in prof}


out = dict(workload="level-0 batch refinement: relative-pose and attitude factors (K2p)", gpu=torch.cuda.get_device_name(0),
           reps=a.reps, solve_reps=a.solve_reps, runs=[])
for K in a.K:
    P = synth.pose_graph_problem(K=K)
    f = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    ctx = api.Context(0)
    ctx.batch_set_pose_factors(f)
    n_pairs = len(ctx.batch_pose_pair_list()[0])
    x = P["poses_init"]
    run = dict(K=K, factors=len(f), pose_pairs=n_pairs,
               eval_call_ms=round(median_ms(lambda: ctx.eval_pose_factors(x), a.reps), 4),
               kernels_mean_ms=kernel_ms(ctx, lambda: ctx.eval_pose_factors(x), ["k_pose_pair_sums", "k_pose_assemble"], a.reps))
    hf = api.HostFactorSet()
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], None, np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.zeros(9)]))
    ctx.batch_use_pose_factors(True)
    opts = api.batch_solver_options(max_num_iterations=a.iters)
    res = {}
    def solve():
        res["r"] = ctx.batch_solve(x, None, hf, opts)
    run["solve_median_ms"] = round(median_ms(solve, a.solve_reps), 2)
    s = res["r"]["summary"]
    run.update(solve_iterations=int(s.num_iterations), initial_cost=float(s.initial_cost), final_cost=float(s.final_cost))
    out["runs"].append(run)
    ctx.close()
out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                   capture_output=True, text=True).stdout.strip()
print(json.dumps(out))
