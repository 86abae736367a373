#!/usr/bin/env python
"""glio_batch_solve on the host path against the device minimizer (glio_batch_use_device_solver) on K = 200, 2 000 and 3 457
keyframes (3 457 is the reference's sample run):
  level 0: synth.dd_psr_problem, pose and DD factors on the device, a prior on keyframe 0 as the host factor;
  level 1: synth.imu_problem with its LiDAR pairs within the search range of 6 (the device factorisation takes a half bandwidth up
           to 160), attitude and IMU factors on the device, a prior on keyframe 0.
For each: --iters iterations, the per-iteration split from glio_solver_summary (eval_seconds, linear_solver_seconds,
total_seconds), the half bandwidth glio_batch_solve used (from glio_batch_normal_equations), and on the device path the mean time
of k_band_chol_solve and k_band_assemble per launch (CUDA events, glio_profile_*).  Also the GPU's name, power limit and clocks,
read in the same run.  Prints one JSON line."""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, synth
from tests import eval_reference as er

ap = argparse.ArgumentParser()
ap.add_argument("--K", type=int, nargs="+", default=[200, 2000, 3457])
ap.add_argument("--iters", type=int, default=10)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_batch_device_solve.py needs a CUDA device")


def level0(K):
    P = synth.dd_psr_problem(K=K)
    c = api.Context(0)
    c.batch_set_dd_psr_factors(api.dd_psr_factor_records(**P["dd"]), api.dd_psr_sat_records(**P["dd_sats"]), P["R"], P["anchor"])
    c.batch_use_dd_psr_factors(True)
    c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
    hf = api.HostFactorSet()
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], None, np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.zeros(9)]))
    return c, P, None, hf


def level1(K):
    P = synth.imu_problem(K=K)
    c = api.Context(0)
    cur, oth = (np.asarray(v) for v in P["pairs"])
    keep = np.abs(cur - oth) <= 6
    cur, oth = cur[keep], oth[keep]
    rng = np.random.default_rng(3)
    c.batch_declare_pairs(cur, oth)
    for i, j in zip(cur, oth):
        m = er.make_pair(rng, P["poses_true"][i], P["poses_true"][j], 40, noise=0.02)
        c.batch_set_pair_matches(int(i), int(j), m["cp"], m["nc"], m["weight"])
    c.batch_set_pose_factors(api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])); c.batch_use_pose_factors(True)
    c.batch_set_imu_factors(api.imu_factor_records(**P["imu"])); c.batch_use_imu_factors(True)
    hf = api.HostFactorSet()
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], P["sb_true"][0],
                 3 * np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)]))
    return c, P, P["sb_init"], hf


def run(c, P, sb, hf, on, iters):
    c.batch_use_device_solver(on)
    c.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=1))       # warm-up
    if on:
        c.lib_profile(True)
    r = c.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=iters))
    s = r["summary"]; it = max(int(s.num_iterations), 1)
    out = dict(iterations=int(s.num_iterations), linear_solves=int(s.num_linear_solves), final_cost=float(s.final_cost),
               eval_ms_per_iter=round(1e3 * s.eval_seconds / it, 2), linear_solver_ms_per_iter=round(1e3 * s.linear_solver_seconds / it, 2),
               total_ms_per_iter=round(1e3 * s.total_seconds / it, 2))
    if on:
        prof = c.lib_profile_read(); c.lib_profile(False)
        out["kernels_mean_ms"] = {k: round(prof[k][0] / prof[k][1], 3) for k in ("k_band_chol_solve", "k_band_assemble") if k in prof}
    return out, r


res = dict(workload="batch refinement: host band algebra against the device minimizer", gpu=torch.cuda.get_device_name(0), iters=a.iters, runs=[])
for K in a.K:
    for level, make in ((0, level0), (1, level1)):
        c, P, sb, hf = make(K)
        hb = c.batch_normal_equations(P["poses_init"], sb, hf)[0].shape[1] - 1
        host, rh = run(c, P, sb, hf, False, a.iters)
        dev, rd = run(c, P, sb, hf, True, a.iters)
        c.close()
        res["runs"].append(dict(K=K, level=level, n=len(rh["poses"]) * (15 if sb is not None else 6), hb=hb, host=host, device=dev,
                                max_position_diff_m=float(np.max(np.abs(rh["poses"][:, :3] - rd["poses"][:, :3])))))
        print(json.dumps(res["runs"][-1]), file=sys.stderr, flush=True)
res["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.draw,clocks.sm,clocks.max.sm,clocks.mem",
                                    "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps(res))
