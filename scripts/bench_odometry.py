#!/usr/bin/env python
"""The front end on the device, sensor to odometry (SURVEY 8 f-5 + f-4 + f-6): a seeded 32-line drive of about 60 k raw points per
sweep in pinned host memory -> glio_prepare_scan (output stays on the device) -> glio_extract_features -> glio_odom_step with the
full cloud device-resident, one sweep after the other as the node sees them.  Per sweep: CUDA events on the context's stream around
upload + prepare + extract + odometry and around the odometry alone; medians over --sweeps timed sweeps after --warmup.  Also:
LM iterations per sweep, the keyframe ratio, per-kernel device times from lib_profile (a separate pass), and the CPU oracle's
odometry step on one thread for the same sweeps.  Prints one JSON line with the card and its power limit.  Standalone; not
bench.py's metric."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--sweeps", type=int, default=300); ap.add_argument("--warmup", type=int, default=20)
ap.add_argument("--profile-sweeps", type=int, default=50); ap.add_argument("--cpu-sweeps", type=int, default=20)
a = ap.parse_args()


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


K = a.warmup + a.sweeps + a.profile_sweeps
D = synth.raw_drive(K)
sweeps, qs = [], []
st_imu = api.ImuState()
for k in range(K):
    raw = D["sweeps"][k]
    buf = np.full((len(raw), 8), np.nan, np.float32)                 # pcl::PointXYZI: x y z 1 | intensity pad pad pad
    buf[:, :3] = raw[:, :3]; buf[:, 3] = 1.0; buf[:, 4] = raw[:, 3]
    sweeps.append(torch.from_numpy(buf).pin_memory())
    qs.append(api.imu_sweep_rotation(st_imu, D["stamps"], D["gyro"], D["t_scan_next"][k]))

ctx = api.Context(0); st = torch.cuda.ExternalStream(ctx.stream)
odo = api.Odometry(ctx)                                              # the shipped configuration (config_urban_hk.yaml)
feat = dict(ds_rate=1, edge_thres=1.0, surf_thres=0.1, ds_v=0.4)
t_all, t_odo, iters, kfs, n_raw, n_surf, n_map = [], [], [], [], [], [], []
surfs, fulls = [], []
for i in range(a.warmup + a.sweeps):
    torch.cuda.synchronize()
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record(st)
    cloud, ss, se = ctx.prepare_scan(sweeps[i].numpy(), 32, q_imu=qs[i], out="device")
    f = ctx.extract_features(cloud, ss, se, **feat)
    e1.record(st)
    r = odo.step(f["less_flat_ds"], cloud, out="device")
    e2.record(st)
    torch.cuda.synchronize()
    if i >= a.warmup:
        t_all.append(e0.elapsed_time(e2)); t_odo.append(e1.elapsed_time(e2))
        iters.append(sum(x["iterations"] for x in r["rounds"])); kfs.append(r["keyframe"])
        n_raw.append(len(sweeps[i])); n_surf.append(r["n_scan"]); n_map.append(r["n_map"])
        if len(surfs) < a.cpu_sweeps + 2:
            surfs.append(f["less_flat_ds"].copy()); fulls.append(cloud.cpu().numpy())
# per-kernel device times over a separate pass (events around every launch slow the host down)
ctx.lib_profile(True)
for i in range(a.warmup + a.sweeps, K):
    cloud, ss, se = ctx.prepare_scan(sweeps[i].numpy(), 32, q_imu=qs[i], out="device")
    f = ctx.extract_features(cloud, ss, se, **feat)
    odo.step(f["less_flat_ds"], cloud, out="device")
prof = {k: round(v[0] / max(a.profile_sweeps, 1), 4) for k, v in ctx.lib_profile_read().items()}
ctx.lib_profile(False)
card = torch.cuda.get_device_name(0); pl = power_limit()
odo.close(); ctx.close()

# the CPU oracle's odometry on one thread, on sweeps of the same drive (its state starts fresh at the first of them)
cpu_ms = None
try:
    from oracle import pyoracle_odom as od
    o = od.OdometryOracle(nthreads=1)
    ts = []
    for k in range(len(surfs)):
        t0 = time.perf_counter(); o.step(surfs[k], fulls[k]); t1 = time.perf_counter()
        if k >= 2:
            ts.append((t1 - t0) * 1e3)
    cpu_ms = round(float(np.median(ts)), 3)
except Exception as e:      # the oracle needs its CPU library (built by build())
    print(f"cpu oracle not run: {e}", file=sys.stderr)

print(json.dumps(dict(gpu=card, power_limit=pl, raw_points=int(np.median(n_raw)), surf_points=int(np.median(n_surf)),
                      map_points=int(np.median(n_map)), sweeps_timed=len(t_all), device_sweep_ms=round(float(np.median(t_all)), 3),
                      device_odometry_ms=round(float(np.median(t_odo)), 3), lm_iterations_per_sweep=round(float(np.mean(iters)), 2),
                      keyframe_ratio=round(float(np.mean(kfs)), 3), cpu_oracle_odometry_ms=cpu_ms, kernel_ms_per_sweep=prof)))
