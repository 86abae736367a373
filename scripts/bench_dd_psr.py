#!/usr/bin/env python
"""The batch refinement's double-differenced pseudorange factors (K2g) in the reference's level-0 problem, on problems of K = 200,
2 000 and 3 457 keyframes (synth.dd_psr_problem: the pose factors of synth.pose_graph_problem, GNSS epochs at 10 Hz, one kept epoch
per metre, up to four constellation blocks per epoch; 3 457 is the reference's sample run).
Reports, after warm-up: glio_eval_dd_psr_factors, the median of --reps calls (host clock around the call, which ends in a stream
synchronisation); its two kernels, the mean over the same --reps launches (CUDA events on the context's stream, glio_profile_*);
glio_batch_solve of the level-0 problem (pose factors on the device; DD factors on the device, and off) through the reference's
4 outer passes, each with its own DD list (threshold 1e9, 10, 8, 6, the 1 m rule against the pass's starting states), at most
--iters iterations per pass, a prior on keyframe 0 as the one host factor; the GPU's name and power limit, read in the same run.
Prints one JSON line."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--K", type=int, nargs="+", default=[200, 2000, 3457])
ap.add_argument("--iters", type=int, default=100)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_dd_psr.py needs a CUDA device")


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


def outer_passes(ctx, P, dd_on, iters):
    """the 4 outer passes: each rebuilds its DD list from the current states and solves; returns per-pass (factors, ms, iterations)
    and the final translation error against the truth"""
    x = P["poses_init"].copy()
    hf = api.HostFactorSet()
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], None, np.concatenate([np.full(3, 30.0), np.full(3, 90.0), np.zeros(9)]))
    opts = api.batch_solver_options(max_num_iterations=iters)
    out = []
    for p, thr in enumerate(synth.DD_PSR_THRESHOLDS):
        cols, sats = synth.dd_psr_factors(P["epochs"], P["kf_times"], x[:, :3], P["station"], thr)
        if dd_on:
            ctx.batch_set_dd_psr_factors(api.dd_psr_factor_records(**cols), api.dd_psr_sat_records(**sats), P["R"], P["anchor"])
        ctx.batch_use_dd_psr_factors(dd_on)
        t0 = time.perf_counter(); r = ctx.batch_solve(x, None, hf, opts); ms = 1e3 * (time.perf_counter() - t0)
        x = r["poses"]
        out.append(dict(dd_factors=len(cols["i"]) if dd_on else 0, ms=round(ms, 2), iterations=int(r["summary"].num_iterations)))
    err = float(np.mean(np.linalg.norm(x[:, :3] - P["poses_true"][:, :3], axis=1)))
    return out, err


out = dict(workload="level-0 batch refinement: DD pseudorange factors (K2g) beside the pose factors (K2p)",
           gpu=torch.cuda.get_device_name(0), reps=a.reps, runs=[])
for K in a.K:
    P = synth.dd_psr_problem(K=K)
    f = api.dd_psr_factor_records(**P["dd"]); sats = api.dd_psr_sat_records(**P["dd_sats"])
    ctx = api.Context(0)
    ctx.batch_set_dd_psr_factors(f, sats, P["R"], P["anchor"])
    n_pairs = len(ctx.batch_dd_psr_pair_list()[0])
    x = P["poses_init"]
    run = dict(K=K, epochs=len(P["epochs"]), dd_factors=len(f), dd_rows=int(np.sum(f["n_sat"] - 1)), dd_pairs=n_pairs,
               eval_call_ms=round(median_ms(lambda: ctx.eval_dd_psr_factors(x), a.reps), 4),
               kernels_mean_ms=kernel_ms(ctx, lambda: ctx.eval_dd_psr_factors(x), ["k_psr_pair_sums", "k_psr_assemble"], a.reps))
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    ctx.batch_set_pose_factors(pf); ctx.batch_use_pose_factors(True)
    for name, on in (("dd_on", True), ("dd_off", False)):
        passes, err = outer_passes(ctx, P, on, a.iters)
        run[name] = dict(passes=passes, total_ms=round(sum(p["ms"] for p in passes), 2), mean_translation_error_m=round(err, 4))
    out["runs"].append(run)
    ctx.close()
out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                   capture_output=True, text=True).stdout.strip()
print(json.dumps(out))
