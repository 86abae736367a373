#!/usr/bin/env python
"""Seeded edge selection (glio_select_random_edges, glio_batch_select_random_edges) and what it does to the solves, at two shapes:
  - window: W = 20 corner scans of 10 000 points against a corner map of 200 000 points (the shape of bench_edges.py), with the
    surf matches of synth.window_problem (10 000 points per scan, 200 000-point map) selected at F = 100 (shipped options);
  - batch: cfg 3's shape (bench_batch_edges.py): K = 200 keyframes, search range 6 (2 400 pairs), 100 000 surf and 10 000 corner
    points per frame, plane matches selected at B = 25 (--mode, default 0: start/end).
Reports, as medians: the edge selection call (host clock around the call and a stream synchronisation) and its k_sel_sample time
(CUDA events on the context's stream, glio_profile_*); glio_window_solve / glio_batch_solve time and iterations with edges on,
unselected and selected (edge sizes F = 100 / B = 25, the plane sizes); the K2e / K2be kernel time of one evaluation, unselected
and selected; the GPU's name and power limit, read in the same run.  Prints one JSON line."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, dist as gdist, synth

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--W", type=int, default=20)
ap.add_argument("--Q", type=int, default=10_000)
ap.add_argument("--M", type=int, default=200_000)
ap.add_argument("--K", type=int, default=200)
ap.add_argument("--search-range", type=int, default=6)
ap.add_argument("--Qb", type=int, default=100_000)
ap.add_argument("--Qe", type=int, default=10_000)
ap.add_argument("--mode", type=int, default=0)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--no-batch", action="store_true")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_edge_select.py needs a CUDA device")


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def kernel_ms(ctx, fn, name, reps):
    fn()
    ctx.lib_profile(True)
    for _ in range(reps):
        fn()
    prof = ctx.lib_profile_read(); ctx.lib_profile(False)
    return round(prof[name][0] / prof[name][1], 4) if name in prof else 0.0


out = dict(workload="edge selection: window (W corner scans, one corner map) and batch (cfg 3) solves with edges",
           gpu=torch.cuda.get_device_name(0), reps=a.reps)

# ---- window
E = synth.window_edge_problem(W=a.W, Q=a.Q, M=a.M)
P = synth.window_problem(W=a.W, Q=a.Q, M=a.M)
ctx = api.Context(0)
ctx.set_map(P["map_xyz"]); ctx.window_set_scans(P["scans"]); ctx.window_associate(P["poses_init"])
ctx.set_edge_map(E["map_xyz"])
for k in range(a.W):
    ctx.window_set_edge_scan(k, E["scans"][k])
ne = ctx.window_associate_edges(P["poses_init"])
ids = np.arange(a.W, dtype=np.int64)
opt = api.select_default_options(seed=1, nonce=0)
na_planes = ctx.select_random(ids, opt)
ctx.window_use_edges(True)
win = dict(W=a.W, Q=a.Q, M=a.M, edges=int(ne.sum()), planes_active=int(na_planes.sum()))
eval_edge = lambda: ctx.eval_edge(P["poses_init"])                                                       # noqa: E731
for key in ("edges_unselected", "edges_selected"):
    if key == "edges_selected":
        def sel():
            ctx.select_random_edges(ids, opt); ctx.synchronize()
        win["select_edges_call_ms"] = median_ms(sel, a.reps)
        win["k_sel_sample_ms"] = kernel_ms(ctx, sel, "k_sel_sample", a.reps)
        win["edges_active"] = int(ctx.select_random_edges(ids, opt).sum())
    r = ctx.window_solve(P["poses_init"])
    win[key] = dict(solve_ms=median_ms(lambda: ctx.window_solve(P["poses_init"]), a.reps), iterations=int(r["summary"].num_iterations),
                    final_cost=float(r["summary"].final_cost), k_eval_edge_ms=kernel_ms(ctx, eval_edge, "k_eval_edge", a.reps))
ctx.close()
out["window"] = win

# ---- batch
if not a.no_batch:
    K, sr = a.K, a.search_range
    B = synth.batch_problem(K=K, Q=a.Qb, search_range=sr)
    Eb = synth.batch_edge_problem(K=K, Q=a.Qe, search_range=sr)
    cur, oth = gdist.batch_pairs(K, sr)
    ctx = api.Context(0)
    for k in range(K):
        ctx.batch_set_frame(k, B["scans"][k], B["poses_init"][k])
        ctx.batch_set_edge_frame(k, Eb["corner_scans"][k])
    ctx.batch_declare_pairs(cur, oth)
    nm = ctx.batch_associate_pairs(cur, oth)
    neb = ctx.batch_associate_edges_pairs(cur, oth)
    na_planes = ctx.batch_select_random(cur, oth, a.mode, opt)
    hf = api.HostFactorSet(); T = B["poses_true"]; rng = np.random.default_rng(7)
    sw = np.concatenate([np.full(3, 10.0), np.full(3, 30.0), np.zeros(9)])
    hf.add_prior(0, T[0, :3], T[0, 3:], None, sw * 3)
    for i in range(K - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]); dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        hf.add_between(i, i + 1, dp + rng.normal(0, 0.005, 3), dq, np.zeros(3), 0.1, sw)
    opts = api.batch_solver_options(max_num_iterations=a.iters)
    ctx.batch_use_edges(True)
    bat = dict(K=K, search_range=sr, pairs=int(len(cur)), Q=a.Qb, Qe=a.Qe, mode=a.mode, plane_matches=int(nm.sum()),
               planes_active=int(na_planes.sum()), edges=int(neb.sum()))
    eval_bedge = lambda: ctx.eval_binary_edge(B["poses_init"])                                           # noqa: E731
    sreps = max(3, a.reps // 3)
    for key in ("edges_unselected", "edges_selected"):
        if key == "edges_selected":
            def bsel():
                ctx.batch_select_random_edges(cur, oth, a.mode, opt); ctx.synchronize()
            bat["select_edges_call_ms"] = median_ms(bsel, a.reps)
            bat["k_sel_sample_ms"] = kernel_ms(ctx, bsel, "k_sel_sample", a.reps)
            bat["edges_active"] = int(ctx.batch_select_random_edges(cur, oth, a.mode, opt).sum())
        r = ctx.batch_solve(B["poses_init"], None, hf, opts)
        bat[key] = dict(solve_ms=median_ms(lambda: ctx.batch_solve(B["poses_init"], None, hf, opts), sreps),
                        iterations=int(r["summary"].num_iterations), final_cost=float(r["summary"].final_cost),
                        k_eval_binary_edge_ms=kernel_ms(ctx, eval_bedge, "k_eval_binary_edge", a.reps))
    ctx.close()
    out["batch"] = bat

out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                   capture_output=True, text=True).stdout.strip()
print(json.dumps(out))
