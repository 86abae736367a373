#!/usr/bin/env python
"""The batch refinement's IMU factors (K2i) in a level-1-shaped problem (synth.imu_problem: the attitude factors and LiDAR pairs of
synth.pose_graph_problem(level=1), one IMU factor per consecutive keyframe pair), on K = 200, 2 000 and 3 457 keyframes (3 457 is
the reference's sample run).
Reports, after warm-up: glio_eval_imu_factors, the median of --reps calls (host clock around the call, which ends in a stream
synchronisation); its two kernels, the mean over the same --reps launches (CUDA events on the context's stream, glio_profile_*);
glio_batch_solve of the level-1 problem with speed-bias (attitude factors on the device, no LiDAR matches, a prior on keyframe 0
as the host factor) for --iters iterations, with the IMU blocks on the device, and with the same blocks from a host band callback.
The host arm's callback is the Python longdouble restatement tests/imu_factor_reference.py (no C++ host ImuFactor exists here), so
it bounds nothing about a compiled host evaluation; it runs for K <= --host-max-K only, larger K are "not measured".  Also the
GPU's name, power limit and clocks, read in the same run.  Prints one JSON line."""
import argparse, ctypes as C, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--K", type=int, nargs="+", default=[200, 2000, 3457])
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--host-max-K", type=int, default=3457)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_imu_factors.py needs a CUDA device")


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


def host_factors(P):
    hf = api.HostFactorSet()
    hf.add_prior(0, P["poses_true"][0, :3], P["poses_true"][0, 3:], P["sb_true"][0],
                 3 * np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)]))
    return hf


def solve_device(P, f, pf, iters):
    ctx = api.Context(0)
    ctx.batch_set_pose_factors(pf); ctx.batch_use_pose_factors(True)
    ctx.batch_set_imu_factors(f); ctx.batch_use_imu_factors(True)
    hf = host_factors(P)
    t0 = time.perf_counter()
    r = ctx.batch_solve(P["poses_init"], P["sb_init"], hf, api.batch_solver_options(max_num_iterations=iters))
    ms = 1e3 * (time.perf_counter() - t0)
    ctx.close()
    return dict(ms=round(ms, 2), iterations=int(r["summary"].num_iterations), final_cost=float(r["summary"].final_cost))


def solve_host(P, f, pf, iters):
    from tests import imu_factor_reference as ir
    ctx = api.Context(0)
    ctx.batch_set_pose_factors(pf); ctx.batch_use_pose_factors(True)
    pairs = np.array(ir.pair_table(f)[0], np.int32).reshape(-1, 2)
    ctx.batch_declare_pairs(pairs[:, 0], pairs[:, 1])
    hf = host_factors(P); L = ctx._lib
    cb_ms = []

    def cb(user, K, p, s, want_jac, H, hb, g, cost):
        t0 = time.perf_counter()
        L.glio_hf_evaluate_band(hf._h, K, p, s, want_jac, H, hb, g, cost)
        e = ir.imu_blocks(np.ctypeslib.as_array(p, (K * 7,)).reshape(K, 7), np.ctypeslib.as_array(s, (K * 9,)).reshape(K, 9), f)
        cost[0] = cost[0] + e["cost"]
        if want_jac:
            w = hb + 1
            band = np.ctypeslib.as_array(H, (K * 15 * w,)).reshape(K * 15, w); gv = np.ctypeslib.as_array(g, (K * 15,))
            for k in range(K):
                for i in range(15):
                    band[15 * k + i, hb - i:hb + 1] += e["Hdiag"][k, i, :i + 1]
                gv[15 * k:15 * k + 15] += e["g"][k]
            for q, (ka, kb) in enumerate(e["pairs"]):
                for y in range(15):
                    i = 15 * kb + y
                    band[i, 15 * ka - i + hb:15 * ka + 15 - i + hb] += e["Hoff"][q][:, y]
        cb_ms.append(1e3 * (time.perf_counter() - t0))
        return 0
    fn = api.HOST_FACTORS_BAND_FN(cb)
    pb = np.array(P["poses_init"]).copy(); sb = np.array(P["sb_init"]).copy(); K = len(pb)
    opt = api.batch_solver_options(max_num_iterations=iters); summ = api.SolverSummary(); log = (api.Iteration * 64)()
    t0 = time.perf_counter()
    ctx._chk(L.glio_batch_solve(ctx._h, C.c_int(K), api._ptr(pb), api._ptr(sb), fn, None, C.byref(opt), C.byref(summ), log, C.c_int(64),
                                None, C.c_int64(0)))
    ms = 1e3 * (time.perf_counter() - t0)
    ctx.close()
    return dict(ms=round(ms, 2), iterations=int(summ.num_iterations), final_cost=float(summ.final_cost),
                callback_median_ms=round(float(np.median(cb_ms)), 2))


out = dict(workload="level-1 batch refinement: IMU factors (K2i) from caller-supplied pre-integration",
           gpu=torch.cuda.get_device_name(0), reps=a.reps, iters=a.iters, runs=[])
for K in a.K:
    P = synth.imu_problem(K=K)
    f = api.imu_factor_records(**P["imu"])
    pf = api.pose_factor_records(P["i"], P["j"], P["kind"], P["dq"], P["dp"])
    ctx = api.Context(0)
    ctx.batch_set_imu_factors(f)
    x, sb = P["poses_init"], P["sb_init"]
    run = dict(K=K, imu_factors=len(f), imu_pairs=len(ctx.batch_imu_pair_list()[0]),
               eval_call_ms=round(median_ms(lambda: ctx.eval_imu_factors(x, sb), a.reps), 4),
               eval_cost_only_call_ms=round(median_ms(lambda: ctx.eval_imu_factors(x, sb, want_jac=False), a.reps), 4),
               kernels_mean_ms=kernel_ms(ctx, lambda: ctx.eval_imu_factors(x, sb), ["k_imu_pair_sums", "k_imu_assemble"], a.reps))
    ctx.close()
    run["solve_imu_on_device"] = solve_device(P, f, pf, a.iters)
    run["solve_imu_in_host_callback"] = solve_host(P, f, pf, a.iters) if K <= a.host_max_K else "not measured"
    out["runs"].append(run)
out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.draw,clocks.sm,clocks.max.sm,clocks.mem",
                                    "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps(out))
