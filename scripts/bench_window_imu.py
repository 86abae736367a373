#!/usr/bin/env python
"""The sliding window's IMU chain: host stand-in versus device ImuFactor (glio_window_use_imu_factors), on bench.py's cfg-2 window
shape (Q = 100k surf points per scan, M = 1M map points) at W = 5 (the shipped slide_window_width) and W = 20 (bench.py's).
Both arms solve the same associated window with a speed-bias prior on KF0 as a host factor, through glio_window_solve_band:
  host    the IMU chain is the stand-in `between` of host_factors.cpp (same block structure: 15 x [t, q, sb | t, q, sb] per pair);
  device  the IMU chain is synth.window_imu_problem's ImuFactor records, evaluated by K2i ahead of K2.
Reports per W and arm, after warm-up: the median of --reps solves and of --reps synchronous marginalisations (host clock around
calls that end in a synchronisation), the solve's iterations and evaluations, kernel launches per evaluation, and the K2i kernel
times (mean per launch, CUDA events through glio_profile_*); also the GPU's name and power limit, read in the same run.  Prints one
JSON line."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--W", type=int, nargs="+", default=[5, 20])
ap.add_argument("--Q", type=int, default=100_000)
ap.add_argument("--M", type=int, default=1_000_000)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_window_imu.py needs a CUDA device")
KERNELS = ["k_imu_pair_sums", "k_imu_pair_sums_cost", "k_imu_assemble", "k_imu_pair_sums_ambient", "k_eval_unary", "k_eval_unary_cost"]


def host_set(P, W, stand_in):
    hf = api.HostFactorSet()
    T = P["poses_true"]
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.full(9, 1.0)])
    hf.add_prior(0, T[0, :3], T[0, 3:], P["sb_true"][0], 3 * sw)
    if stand_in:
        for i in range(W - 1):
            dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:])
            dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
            hf.add_between(i, i + 1, dp, dq, P["sb_true"][i + 1, :3] - P["sb_true"][i, :3], float(np.diff(P["kf_times"])[i]), 0.5 * sw)
    return hf


def measure(P, W, device):
    ctx = api.Context(0)
    ctx.set_map(P["map_xyz"]); ctx.window_set_scans(P["scans"]); ctx.window_associate(P["poses_init"])
    if device:
        ctx.window_set_imu_factors(api.imu_factor_records(**P["imu"])); ctx.window_use_imu_factors(True)
    hf = host_set(P, W, not device)
    solve = lambda: ctx.window_solve(P["poses_init"], P["sb_init"], hf, band=29)
    r = solve()
    marg = lambda: ctx.window_marginalize(r["poses"], r["speed_bias"], hf)
    marg()
    ts, tm = [], []
    ctx.lib_profile(True)
    n0 = ctx.launch_count
    for _ in range(a.reps):
        t0 = time.perf_counter(); r = solve(); ts.append(time.perf_counter() - t0)
    n_solve = ctx.launch_count - n0
    prof_solve = ctx.lib_profile_read(); ctx.lib_profile(False); ctx.lib_profile(True)
    n0 = ctx.launch_count
    for _ in range(a.reps):
        t0 = time.perf_counter(); marg(); tm.append(time.perf_counter() - t0)
    n_marg = ctx.launch_count - n0
    prof_marg = ctx.lib_profile_read(); ctx.lib_profile(False)
    s = r["summary"]
    ctx.close()
    per = lambda prof: {k: dict(mean_ms=round(prof[k][0] / prof[k][1], 4), launches=prof[k][1]) for k in KERNELS if k in prof}
    return dict(solve_ms=round(1e3 * float(np.median(ts)), 3), marg_ms=round(1e3 * float(np.median(tm)), 3),
                iterations=int(s.num_iterations), evaluations=int(s.num_evaluations),
                launches_per_evaluation=round(n_solve / (a.reps * max(s.num_evaluations, 1)), 2), launches_per_marg=n_marg / a.reps,
                final_cost=float(s.final_cost), kernels_solve=per(prof_solve), kernels_marg=per(prof_marg))


out = dict(workload="window IMU chain: host stand-in vs device ImuFactor, cfg-2 window shape", Q=a.Q, M=a.M, reps=a.reps)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                    os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]], capture_output=True, text=True)
out["gpu"] = q.stdout.strip() or torch.cuda.get_device_name(0)
for W in a.W:
    P = synth.window_imu_problem(W=W, Q=a.Q, M=a.M)
    out[f"W{W}"] = dict(host=measure(P, W, False), device=measure(P, W, True))
print(json.dumps(out))
