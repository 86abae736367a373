#!/usr/bin/env python
"""ceres::Solve through the Ceres-API shim, host-routed against device-routed, for the batch refinement's pose factors (K2p):
  - level 0 (the shipped sms_fusion_level 0 problem of synth.pose_graph_problem: attitude then relative factors, unused
    speed-bias and receiver-clock blocks, constant yaw and anchor, pseudorange-like host stand-ins) at K = 200, 2 000 and 3 457
    keyframes (the sample run's size);
  - level 1 at K = 200: attitude factors, 20 BinaryLidarPlaneNormFactor blocks per batch pair and an IMU-like host chain.
The Estimator's options (SUBSPACE_DOGLEG, nonmonotonic steps).  Every solve is capped at --iters iterations, both routings, and
timed with a host clock around ceres::Solve (which ends with the device results on the host) inside the driver
tests/cpp/shim_pose_routes_test.cpp, compiled here into a temporary directory; the table reports the median wall time per solve and
per iteration.  Before timing, one untimed device-routed solve of each case checks that every pose block was routed.  Prints the
GPU's name, power limit and SM clock limit, then one JSON line."""
import argparse, json, os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from tests import shim_common as sc
from tests import test_shim_pose_routes as tp


def timed(exe, mode, path, reps, iters):
    rows = sc.run_driver(exe, mode, [path], "--repeat", str(reps + 1), "--max-iter", str(iters))[0]["times"][1:]   # the first solve warms up
    ms = [r[0] for r in rows]; its = [r[1] for r in rows]
    return dict(median_ms=float(np.median(ms)), iterations=sorted(set(its)), median_ms_per_iteration=float(np.median([m / max(i, 1) for m, i in zip(ms, its)])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps-large", type=int, default=2, help="host-routed solves of the K >= 2000 cases")
    ap.add_argument("--iters", type=int, default=3, help="iteration cap of every timed solve")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shim_pose_routes.py needs a CUDA device")
    gpu = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
    print("gpu:", gpu, flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        exe = sc.build_driver(tmp, "shim_pose_routes_test")
        out = dict(gpu=gpu, iteration_cap=a.iters, cases={})
        for name, level, K in (("level0_k200", 0, 200), ("level0_k2000", 0, 2000), ("level0_k3457", 0, 3457), ("level1_k200", 1, 200)):
            c = tp.level0(K) if level == 0 else tp.level1(K)
            path = os.path.join(tmp, name + ".bin")
            tp.write_case(path, c)
            n_pose = len(c["pose"])
            r = sc.run_driver(exe, "device", [path], "--max-iter", "1")[0]
            if r["device_pose"] != n_pose:
                sys.exit(f"{name}: {r['device_pose']} of {n_pose} pose blocks were routed to the device")
            info = dict(pose_blocks=n_pose, binary_blocks=len(c["kw"].get("binary", ())))
            info["host"] = timed(exe, "host", path, a.host_reps_large if K >= 2000 else a.reps, a.iters)
            info["device"] = timed(exe, "device", path, a.reps, a.iters)
            info["speedup_per_iteration"] = info["host"]["median_ms_per_iteration"] / info["device"]["median_ms_per_iteration"]
            out["cases"][name] = info
            print(name, json.dumps(info), flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
