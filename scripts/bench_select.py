#!/usr/bin/env python
"""The Estimator's feature selection on the device (glio_select_random / glio_batch_select_random) against the host round trip
a caller needs without it: draw the indices on the host, then one glio_select / glio_batch_select per slot or pair, each an
upload, a launch, a read-back and a stream synchronisation.  Shipped options (F 100, B 25).  Two workloads:
  window  W = 20 keyframes of Q = 100 000 points associated against a 1 M-point map (cfg 2's shape);
  batch   cfg 3's pair list (K = 200, search_range 6: 2 400 pairs), start/end mode, with the same lists on both paths, and the
          binary evaluation after each checked for identical H, g and cost.
Times are host wall clock per call including a final synchronise, medians.  Prints one JSON line with the GPU's name and power
limit, read in the same run."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from glio_b200 import api, dist, synth

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--batch-Q", type=int, default=20000, help="points per batch keyframe (the selection's cost does not follow Q)")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_select.py needs a CUDA device")


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


# ---- window
W = 20
P = synth.window_problem(W=W, Q=100_000, M=1_000_000)
ctx = api.Context(0)
ctx.set_map(P["map_xyz"]); ctx.window_set_scans(P["scans"]); nm = ctx.window_associate(P["poses_init"])
ids = np.arange(W, dtype=np.int64)
opt = api.select_default_options(seed=1)
F = opt.feature_res_num
state = dict(nonce=0)


def device_window():
    opt.nonce = state["nonce"]; state["nonce"] += 1
    ctx.select_random(ids, opt); ctx.synchronize()


rng = np.random.default_rng(0)


def host_window():
    counts = ctx.get_match_counts(W, active=False)
    for k in range(W):
        n = int(counts[k])
        if n >= F + 1:
            ctx.select(k, rng.choice(n - 1, F, replace=False).astype(np.int32))
    ctx.synchronize()


device_window(); host_window()
win = dict(W=W, Q=100_000, matches_per_slot=int(np.median(nm)), device_ms=median_ms(device_window, a.reps),
           host_round_trip_ms=median_ms(host_window, a.reps))
ctx.lib_profile(True); device_window(); win["k_sel_sample_ms"] = ctx.lib_profile_read()["k_sel_sample"][0]; ctx.lib_profile(False)
ctx.close()

# ---- batch, cfg 3
K = 200
cur, oth = dist.batch_pairs(K, 6)
Bp = synth.batch_problem(K=K, Q=a.batch_Q)
ctx = api.Context(0)
for k in range(K):
    ctx.batch_set_frame(k, Bp["scans"][k], Bp["poses_init"][k])
nmb = ctx.batch_associate_pairs(cur, oth)
bopt = api.select_default_options(seed=1)


def device_batch():
    ctx.batch_select_random(cur, oth, 0, bopt); ctx.synchronize()


device_batch()
lists = [ctx.batch_get_selection(int(c), int(o)) for c, o in zip(cur, oth)]
ev_dev = ctx.eval_binary(Bp["poses_init"])


def host_batch():
    for c, o, keep in zip(cur, oth, lists):
        ctx.batch_select(int(c), int(o), keep)


host_batch()
ev_host = ctx.eval_binary(Bp["poses_init"])
same = all(np.array_equal(ev_dev[k], ev_host[k]) for k in ("Hdiag", "Hoff", "g")) and ev_dev["cost"] == ev_host["cost"]
assert same, "eval_binary differs between the device selection and the list-input loop"
bat = dict(K=K, pairs=int(len(cur)), Q=a.batch_Q, sampled_pairs=int(sum(x is not None for x in lists)),
           device_ms=median_ms(device_batch, a.reps), host_loop_ms=median_ms(host_batch, max(3, a.reps // 10)),
           eval_binary_identical=bool(same))
ctx.lib_profile(True); device_batch(); bat["k_sel_sample_ms"] = ctx.lib_profile_read()["k_sel_sample"][0]; ctx.lib_profile(False)
ctx.close()

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps(dict(workload="feature selection: seeded device sampler vs host draws + per-slot / per-pair list input",
                      gpu=torch.cuda.get_device_name(0), nvidia_smi=smi, reps=a.reps, window=win, batch=bat)))
