#!/usr/bin/env python
"""The front end on the device, sensor to features (SURVEY 8 f-5 + f-4): a raw 32-line sweep of about 60 k pcl::PointXYZI points
(stride 8) in pinned host memory -> glio_prepare_scan (upload, NaN / 3 m filters, rings, relTime, IMU de-skew, ring
concatenation; output stays on the device) -> glio_extract_features on that device-resident cloud.  Per sweep: CUDA events on
the context's stream around both calls, median over --sweeps timed sweeps after --warmup; per-kernel device times from
lib_profile.  Beside it: the CPU oracle's prepare + extract on one thread for the same sweeps.  Prints one JSON line with the
card and its power limit.  Standalone; not bench.py's metric."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from glio_b200 import api, synth

ap = argparse.ArgumentParser()
ap.add_argument("--sweeps", type=int, default=300); ap.add_argument("--warmup", type=int, default=20)
ap.add_argument("--distinct", type=int, default=6); ap.add_argument("--n-az", type=int, default=1875)
ap.add_argument("--yaw-rate", type=float, default=0.5); ap.add_argument("--cpu-sweeps", type=int, default=6)
a = ap.parse_args()


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


sweeps, qs = [], []
for k in range(a.distinct):
    s = synth.raw_sweep(32, n_az=a.n_az, yaw_rate=a.yaw_rate, seed=synth.SEED0 + 100 + k)
    buf = np.full((len(s["raw"]), 8), np.nan, np.float32)            # pcl::PointXYZI: x y z 1 | intensity pad pad pad
    buf[:, :3] = s["raw"][:, :3]; buf[:, 3] = 1.0; buf[:, 4] = s["raw"][:, 3]
    sweeps.append(torch.from_numpy(buf).pin_memory())
    qs.append(api.imu_sweep_rotation(api.ImuState(), s["stamps"], s["gyro"], s["t_scan_next"]))

ctx = api.Context(0); st = torch.cuda.ExternalStream(ctx.stream)
feat = dict(ds_rate=1, edge_thres=1.0, surf_thres=0.1, ds_v=0.4)


def one(k):
    cloud, ss, se = ctx.prepare_scan(sweeps[k].numpy(), 32, q_imu=qs[k], out="device")
    return cloud, ctx.extract_features(cloud, ss, se, **feat)


for i in range(a.warmup):
    one(i % a.distinct)
ts, tp = [], []
for i in range(a.sweeps):
    k = i % a.distinct
    torch.cuda.synchronize()
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record(st)
    cloud, ss, se = ctx.prepare_scan(sweeps[k].numpy(), 32, q_imu=qs[k], out="device")
    e1.record(st)
    d = ctx.extract_features(cloud, ss, se, **feat)
    e2.record(st)
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e2)); tp.append(e0.elapsed_time(e1))
ctx.lib_profile(True)
for i in range(a.distinct):
    one(i)
ctx.synchronize()
prof = {k: round(v[0] / v[1], 4) for k, v in ctx.lib_profile_read().items()}
ctx.lib_profile(False)
n_raw = int(sweeps[0].shape[0]); n_kept = int(cloud.shape[0])

from oracle import pyoracle as po, pyoracle_scanprep as ps
po.build(); ps.build()
tc = []
for i in range(a.cpu_sweeps):
    k = i % a.distinct
    raw = sweeps[k].numpy()
    t0 = time.perf_counter()
    o = ps.prepare_scan(raw, 32, qs[k], synth.Q_LB)
    po.extract_features(o["cloud"], o["scan_start"], o["scan_end"], stable=False, **feat)
    tc.append(1e3 * (time.perf_counter() - t0))
print(json.dumps(dict(workload="front end: raw 32-line sweep (pcl::PointXYZI, pinned host) -> prepare_scan -> extract_features on device",
                      gpu=torch.cuda.get_device_name(), power_limit=power_limit(), raw_points=n_raw, kept_points=n_kept,
                      sweeps_timed=a.sweeps, device_sweep_ms=float(np.median(ts)), device_prepare_ms=float(np.median(tp)),
                      device_what="upload + prepare_scan + extract_features, CUDA events on the context stream, median",
                      cpu_sweep_ms=float(np.median(tc)), cpu_what="oracle prepare_scan + extract_features (literal std::sort), 1 thread, median of %d" % len(tc),
                      guard_hits=ctx.scanprep_guard_hits(), kernels_ms=prof)))
ctx.close()
