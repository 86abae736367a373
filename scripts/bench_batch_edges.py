#!/usr/bin/env python
"""Scan-to-multiscan edges at cfg 3's shape: K = 200 keyframes, search_range 6 (2 400 pairs), 100 000 surf points and 10 000 corner
points per frame (synth.batch_problem / synth.batch_edge_problem, the same scene and poses).  Reports:
  - one glio_batch_associate_edges_pairs call over all pairs (host clock around the call, which ends in a stream synchronisation;
    the corner grids are rebuilt each time, as after a pose update) and the edge count;
  - the k_eval_binary_edge kernel time (CUDA events on the context's stream, glio_profile_*) of one glio_eval_binary_edge;
  - glio_batch_solve time and iterations with glio_batch_use_edges off and on (stand-in prior + between host factors, at most
    --iters iterations; the solve is a host loop that waits for every device evaluation);
  - the GPU's name and power limit, read in the same run.
Medians.  Prints one JSON line."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, dist as gdist, synth

ap = argparse.ArgumentParser()
ap.add_argument("--K", type=int, default=200)
ap.add_argument("--search-range", type=int, default=6)
ap.add_argument("--Q", type=int, default=100_000)
ap.add_argument("--Qe", type=int, default=10_000)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=10)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_batch_edges.py needs a CUDA device")

K, sr = a.K, a.search_range
B = synth.batch_problem(K=K, Q=a.Q, search_range=sr)
E = synth.batch_edge_problem(K=K, Q=a.Qe, search_range=sr)
cur, oth = gdist.batch_pairs(K, sr)
ctx = api.Context(0)
for k in range(K):
    ctx.batch_set_frame(k, B["scans"][k], B["poses_init"][k])
    ctx.batch_set_edge_frame(k, E["corner_scans"][k])
ctx.batch_declare_pairs(cur, oth)
nm = ctx.batch_associate_pairs(cur, oth)


def assoc():
    for k in range(K):                      # a pose update drops the grids: every call builds all K corner grids
        ctx.batch_set_pose(k, B["poses_init"][k])
    return ctx.batch_associate_edges_pairs(cur, oth)


ne = assoc()                                 # warm-up: module load, work-space growth
ts = []
for _ in range(a.reps):
    t0 = time.perf_counter(); assoc(); ts.append(time.perf_counter() - t0)
ctx.eval_binary_edge(B["poses_init"])
ctx.lib_profile(True)
for _ in range(a.reps):
    ctx.eval_binary_edge(B["poses_init"])
prof = ctx.lib_profile_read(); ctx.lib_profile(False)
eval_ms = prof["k_eval_binary_edge"][0] / prof["k_eval_binary_edge"][1]

hf = api.HostFactorSet(); T = B["poses_true"]; rng = np.random.default_rng(7)
sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.zeros(9)])
hf.add_prior(0, T[0, :3], T[0, 3:], None, sw * 3)
for i in range(K - 1):
    dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
    hf.add_between(i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw)
opts = api.batch_solver_options(max_num_iterations=a.iters)
solve = {}
for on in (False, True):
    ctx.batch_use_edges(on)
    ctx.batch_solve(B["poses_init"], None, hf, opts)
    st, it = [], 0
    for _ in range(max(3, a.reps)):
        t0 = time.perf_counter(); r = ctx.batch_solve(B["poses_init"], None, hf, opts); st.append(time.perf_counter() - t0)
        it = int(r["summary"].num_iterations)
    solve["edges_on" if on else "edges_off"] = dict(solve_ms=1e3 * float(np.median(st)), iterations=it,
                                                    final_cost=float(r["summary"].final_cost))
ctx.close()

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps(dict(workload="batch edges: K frames, 2*search_range pairs each", gpu=torch.cuda.get_device_name(0), nvidia_smi=smi,
                      K=K, search_range=sr, pairs=int(len(cur)), Q=a.Q, Qe=a.Qe, reps=a.reps, plane_matches=int(nm.sum()),
                      edges=int(ne.sum()), assoc_edges_ms_median=1e3 * float(np.median(ts)), assoc_edges_ms_min=1e3 * float(np.min(ts)),
                      k_eval_binary_edge_ms=round(eval_ms, 4), kernel_ms={k: round(v[0] / v[1], 4) for k, v in sorted(prof.items())},
                      batch_solve=solve)))
