#!/usr/bin/env python
"""Loop-closure registration on the device (SURVEY 8 f-7): a seeded closed drive (synth.loop_drive, --keyframes keyframe surf clouds of
--points points each, pcl::PointXYZI layout in pinned host memory) goes through glio_loop_add_keyframe one keyframe at a time, and
after each one glio_loop_step runs with the keyframe that just left the window, as the Estimator's loop thread does.  Timed: the
steps that accepted a loop, with CUDA events on the context's stream around the whole step (detection, both clouds, ICP, fitness)
and, in a second pass, around glio_icp_align on the same two filtered clouds (the registration alone); medians.  Also: cloud sizes,
ICP iterations, launches and host synchronisations per step, and the CPU oracle's step (oracle/pyoracle_loop.py, one thread) on
--cpu-steps of the same steps.  Prints one JSON line with the card and its power limit.  Standalone; not bench.py's metric."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--keyframes", type=int, default=240); ap.add_argument("--points", type=int, default=2500)
ap.add_argument("--cpu-steps", type=int, default=10); ap.add_argument("--seed", type=int, default=synth.SEED0 + 14)
a = ap.parse_args()


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


D = synth.loop_drive(K=a.keyframes, n_points=a.points, seed=a.seed)
SWW = 5
bufs = []
for c in D["clouds"]:
    b = np.zeros((len(c), 8), np.float32); b[:, :3] = c; b[:, 3] = 1.0           # pcl::PointXYZI: x y z 1 | intensity pad pad pad
    bufs.append(torch.from_numpy(b).pin_memory())

ctx = api.Context(0); st = torch.cuda.ExternalStream(ctx.stream)
loop = api.LoopClosure(ctx)                                        # the shipped configuration (config_urban_hk.yaml)
t_step, wall_step, launches, iters, syncs, sizes, acc_steps, n_detected = [], [], [], [], [], [], [], 0
for k in range(a.keyframes):
    loop.add_keyframe(bufs[k].numpy(), D["poses"][k], D["times"][k])
    if len(loop) < SWW:
        continue
    j = len(loop) - SWW
    sel = D["poses"][j][:3].astype(np.float32)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n0 = ctx.launch_count
    w0 = time.perf_counter()
    e0.record(st)
    r = loop.step(sel, D["times"][j])
    e1.record(st)
    torch.cuda.synchronize()
    w1 = time.perf_counter()
    n_detected += int(r["detected"])
    if r["accepted"]:
        t_step.append(e0.elapsed_time(e1)); wall_step.append((w1 - w0) * 1e3); launches.append(ctx.launch_count - n0)
        iters.append(r["icp"]["iterations"]); syncs.append(r["icp"]["host_syncs"])
        sizes.append((r["n_latest"], r["n_latest_ds"], r["n_his"], r["n_his_ds"]))
        acc_steps.append((k, sel, D["times"][j]))
# the registration alone, on the filtered clouds of a few accepted steps (re-run through a second loop object to recover them)
t_reg = []
probe = api.LoopClosure(ctx)
pick = set(s[0] for s in acc_steps[:: max(1, len(acc_steps) // 20)])
for k in range(a.keyframes):
    probe.add_keyframe(bufs[k].numpy(), D["poses"][k], D["times"][k])
    if k not in pick:
        continue
    j = len(probe) - SWW
    probe.step(D["poses"][j][:3].astype(np.float32), D["times"][j])
    lat, his = probe.clouds()
    dl, dh = torch.from_numpy(lat).cuda(), torch.from_numpy(his).cuda()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    ctx.icp_align(dl, dh, iter_log=False, aligned=False)
    e1.record(st)
    torch.cuda.synchronize()
    t_reg.append(e0.elapsed_time(e1))
card = torch.cuda.get_device_name(0); plim = power_limit()
probe.close(); loop.close(); ctx.close()

# the CPU oracle's step on one thread, on the same steps (its keyframe store replays the drive; only the steps are timed)
cpu_ms = None
try:
    from oracle import pyoracle_loop as olp
    o = olp.LoopOracle()
    want = set(s[0] for s in acc_steps[: a.cpu_steps])
    ts = []
    for k in range(a.keyframes):
        o.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
        if len(o.clouds) < SWW:
            continue
        j = len(o.clouds) - SWW
        if k in want:
            o.time_last_loop = 0.0
            t0 = time.perf_counter(); o.step(D["poses"][j][:3].astype(np.float32), D["times"][j]); ts.append((time.perf_counter() - t0) * 1e3)
    cpu_ms = round(float(np.median(ts[1:] if len(ts) > 1 else ts)), 2)
except Exception as e:      # the oracle needs its CPU library (built by build())
    print(f"cpu oracle not run: {e}", file=sys.stderr)

sz = np.median(np.array(sizes), axis=0).astype(int).tolist() if sizes else [0, 0, 0, 0]
print(json.dumps(dict(gpu=card, power_limit=plim, keyframes=a.keyframes, points_per_keyframe=a.points, steps_detected=n_detected,
                      steps_accepted=len(t_step), latest_points=sz[0], latest_ds_points=sz[1], his_points=sz[2], his_ds_points=sz[3],
                      icp_iterations_median=float(np.median(iters)) if iters else None,
                      device_step_ms=round(float(np.median(t_step)), 3) if t_step else None,
                      wall_step_ms=round(float(np.median(wall_step)), 3) if wall_step else None,
                      device_registration_ms=round(float(np.median(t_reg)), 3) if t_reg else None,
                      launches_per_step=int(np.median(launches)) if launches else None,
                      host_syncs_per_registration=int(np.median(syncs)) if syncs else None, cpu_oracle_step_ms=cpu_ms)))
