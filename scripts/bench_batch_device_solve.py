#!/usr/bin/env python
"""glio_batch_solve on the host path against the device minimizer (glio_batch_use_device_solver) with each of its factorisations,
K4 (GLIO_FACTOR_SEQUENTIAL) and the block cyclic reduction (GLIO_FACTOR_BCR), on K = 200, 2 000 and 3 457 keyframes (3 457 is the
reference's sample run):
  level 0: synth.dd_psr_problem, pose and DD factors on the device, a prior on keyframe 0 as the host factor;
  level 1: synth.imu_problem with its LiDAR pairs within --pair-reach keyframes (default 6: hb = 104, which K4 takes; 12 keeps all of
           the generator's pairs: hb = 194, which only BCR takes, and K4 is reported as refused), attitude and IMU factors on the
           device, a prior on keyframe 0.
For each: --iters iterations, the per-iteration split from glio_solver_summary (eval_seconds, linear_solver_seconds, total_seconds)
over --repeat timed solves (median, min and max of the linear-solver time), the half bandwidth glio_batch_solve used, and on the
device paths the mean time per launch of the factorisation's kernels (CUDA events, glio_profile_*, in a profiled solve of its own).
For BCR also the FP64 operations of one factor-and-solve (tests/band_bcr_reference.py's flops, from n and the block size) over
the summed kernel time of one solve.  Also the GPU's name, power limit and clocks, read in the same run.  Prints one JSON line.
--plan prints the problems' sizes and operation counts without a device."""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from glio_b200 import api, synth
from tests import band_bcr_reference as bcr
from tests import eval_reference as er

ap = argparse.ArgumentParser()
ap.add_argument("--K", type=int, nargs="+", default=[200, 2000, 3457])
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--repeat", type=int, default=3)
ap.add_argument("--pair-reach", type=int, default=6)
ap.add_argument("--levels", type=int, nargs="+", default=[0, 1])
ap.add_argument("--plan", action="store_true")
a = ap.parse_args()
BCR_KERNELS = ("k_bcr_gather", "k_bcr_potrf", "k_bcr_trsm", "k_bcr_update", "k_bcr_back", "k_bcr_finish")


def level1_pairs(P):
    cur, oth = (np.asarray(v) for v in P["pairs"])
    keep = np.abs(cur - oth) <= a.pair_reach
    return cur[keep], oth[keep]


def planned_hb(level, K, P):
    """the half bandwidth glio_batch_solve will use: (largest keyframe span + 1) * nt - 1"""
    nt = 15 if level == 1 else 6
    span = max(1, int(np.max(np.abs(np.asarray(P["i"]) - np.asarray(P["j"])))))
    if level == 1:
        cur, oth = level1_pairs(P)
        span = max(span, int(np.max(np.abs(cur - oth))))
    return min((span + 1) * nt - 1, K * nt - 1)


if a.plan:
    for K in a.K:
        for level in a.levels:
            P = synth.imu_problem(K=K) if level == 1 else synth.dd_psr_problem(K=K)
            n, hb = K * (15 if level == 1 else 6), planned_hb(level, K, P)
            print(json.dumps(dict(K=K, level=level, n=n, hb=hb, bcr_block=bcr.block_size(hb), bcr_gflop=round(bcr.flops(n, hb) / 1e9, 3),
                                  k4_takes=hb <= api.BAND_MAX_HB)))
    sys.exit(0)

import torch
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
    cur, oth = level1_pairs(P)
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


def run(c, P, sb, hf, on, kind, iters, kernels):
    c.batch_use_device_solver(on)
    c.batch_device_factorization(kind)
    c.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=1))       # warm-up
    lin, tot, ev = [], [], []
    for _ in range(a.repeat):
        r = c.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=iters))
        s = r["summary"]; it = max(int(s.num_iterations), 1)
        lin.append(1e3 * s.linear_solver_seconds / it); tot.append(1e3 * s.total_seconds / it); ev.append(1e3 * s.eval_seconds / it)
    out = dict(iterations=int(s.num_iterations), linear_solves=int(s.num_linear_solves), final_cost=float(s.final_cost),
               eval_ms_per_iter=round(float(np.median(ev)), 2), linear_solver_ms_per_iter=round(float(np.median(lin)), 2),
               linear_solver_ms_per_iter_min_max=[round(min(lin), 2), round(max(lin), 2)],
               total_ms_per_iter=round(float(np.median(tot)), 2))
    if on:
        c.lib_profile(True)
        c.batch_solve(P["poses_init"], sb, hf, api.batch_solver_options(max_num_iterations=iters))
        prof = c.lib_profile_read(); c.lib_profile(False)
        out["kernels_mean_ms"] = {k: round(prof[k][0] / prof[k][1], 4) for k in kernels if k in prof}
        if kind == api.FACTOR_BCR and "k_bcr_finish" in prof:
            solves = prof["k_bcr_finish"][1]
            out["bcr_ms_per_solve"] = round(sum(prof[k][0] for k in BCR_KERNELS if k in prof) / solves, 4)
            out["bcr_potrf_launches_per_solve"] = prof["k_bcr_potrf"][1] // solves
    return out, r


res = dict(workload="batch refinement: host band algebra against the device minimizer, K4 and BCR", gpu=torch.cuda.get_device_name(0),
           iters=a.iters, repeat=a.repeat, pair_reach=a.pair_reach, runs=[])
for K in a.K:
    for level in a.levels:
        c, P, sb, hf = (level0 if level == 0 else level1)(K)
        hb = c.batch_normal_equations(P["poses_init"], sb, hf)[0].shape[1] - 1
        n = len(P["poses_init"]) * (15 if sb is not None else 6)
        host, rh = run(c, P, sb, hf, False, api.FACTOR_SEQUENTIAL, a.iters, ())
        row = dict(K=K, level=level, n=n, hb=hb, host=host)
        if hb <= api.BAND_MAX_HB:
            row["k4"], rk = run(c, P, sb, hf, True, api.FACTOR_SEQUENTIAL, a.iters, ("k_band_chol_solve", "k_band_shift", "k_band_assemble"))
            row["k4"]["max_position_diff_m"] = float(np.max(np.abs(rh["poses"][:, :3] - rk["poses"][:, :3])))
        else:
            row["k4"] = "refused: hb > GLIO_BAND_MAX_HB"
        row["bcr"], rb = run(c, P, sb, hf, True, api.FACTOR_BCR, a.iters, BCR_KERNELS + ("k_band_assemble",))
        row["bcr"]["max_position_diff_m"] = float(np.max(np.abs(rh["poses"][:, :3] - rb["poses"][:, :3])))
        f = bcr.flops(n, hb)
        row["bcr"]["block"] = bcr.block_size(hb); row["bcr"]["gflop_per_solve"] = round(f / 1e9, 3)
        if "bcr_ms_per_solve" in row["bcr"]:
            row["bcr"]["fp64_gflops_achieved"] = round(f / (row["bcr"]["bcr_ms_per_solve"] * 1e-3) / 1e9, 1)
        c.close()
        res["runs"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
res["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.draw,clocks.sm,clocks.max.sm,clocks.mem",
                                    "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps(res))
