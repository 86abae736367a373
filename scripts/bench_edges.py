#!/usr/bin/env python
"""Scan-to-map edge association on the device (glio_window_associate_edges): W = 20 corner scans of 10 000 points against a
corner map of 200 000 points (synth.window_edge_problem), shipped options, and the window solve (dogleg, poses only) and the
marginalisation of the same window with its surf matches (synth.window_problem, 10 000 points per scan, 200 000-point map) with
glio_window_use_edges off and on.  Reports the association call time, the per-kernel device time of one call (CUDA events on the
context's stream, glio_profile_*), the launches per call and the edge count; solve and marginalisation times.  Every timed call
ends in a stream synchronisation of its own (the solve and the marginalisation are host loops that wait for each device
evaluation), so the host clock around a call spans the device work; medians.  Prints one JSON line with the GPU's name and power
limit, read in the same run."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--W", type=int, default=20)
ap.add_argument("--Q", type=int, default=10_000)
ap.add_argument("--M", type=int, default=200_000)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_edges.py needs a CUDA device")

E = synth.window_edge_problem(W=a.W, Q=a.Q, M=a.M)
ctx = api.Context(0)
ctx.set_edge_map(E["map_xyz"])
for k in range(a.W):
    ctx.window_set_edge_scan(k, E["scans"][k])
ne = ctx.window_associate_edges(E["poses_init"])            # warm-up: module load, work-space growth
ts = []
for _ in range(a.reps):
    t0 = time.perf_counter(); ctx.window_associate_edges(E["poses_init"]); ts.append(time.perf_counter() - t0)
n0 = ctx.launch_count
ctx.lib_profile(True); ctx.window_associate_edges(E["poses_init"]); prof = ctx.lib_profile_read(); ctx.lib_profile(False)
launches = ctx.launch_count - n0


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


P = synth.window_problem(W=a.W, Q=a.Q, M=a.M)
ctx.set_map(P["map_xyz"]); ctx.window_set_scans(P["scans"]); ctx.window_associate(P["poses_init"])
ctx.window_associate_edges(P["poses_init"])
sb = np.zeros((a.W, 9))
solve = {}
for on in (False, True):
    ctx.window_use_edges(on)
    key = "edges_on" if on else "edges_off"
    r = ctx.window_solve(P["poses_init"])
    solve[key] = dict(solve_ms=median_ms(lambda: ctx.window_solve(P["poses_init"]), max(3, a.reps // 5)),
                      iterations=int(r["summary"].num_iterations),
                      marginalize_ms=median_ms(lambda: ctx.window_marginalize(r["poses"], sb), max(3, a.reps // 5)))
ctx.close()

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps(dict(workload="edge association: W corner scans against one corner map", gpu=torch.cuda.get_device_name(0), nvidia_smi=smi,
                      W=a.W, Q=a.Q, M=a.M, reps=a.reps, edges=int(ne.sum()), call_ms_median=1e3 * float(np.median(ts)),
                      call_ms_min=1e3 * float(np.min(ts)), launches_per_call=int(launches),
                      kernel_ms={k: round(v[0], 4) for k, v in sorted(prof.items())}, window=solve)))
