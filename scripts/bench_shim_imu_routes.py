#!/usr/bin/env python
"""ceres::Solve through the Ceres-API shim, host-routed against device-routed, for the batch refinement's IMU factors (K2i,
ImuFactor): the shipped sms_fusion_level 1 problem of tests/test_shim_imu_routes.py (attitude factors, BinaryLidarPlaneNormFactor
blocks of the batch pairs, then the IMU chain of synth.imu_problem) at K = 200, 2 000 and 3 457 keyframes (the sample run's size).
Host-routed, every block is evaluated on the host (no context attached); device-routed, every block is on the GPU (attitude blocks
by K2p, binary-plane blocks by K2b, IMU blocks by K2i).  A third timing, "imu_on_host", is the routing without this route: the
same problem with the IMU factors added through a ceres::CostFunction*, so they run on the host and the rest on the GPU.  The
Estimator's options (SUBSPACE_DOGLEG, nonmonotonic steps), every solve capped at --iters iterations, timed with a host clock around
ceres::Solve (which ends with the device results on the host) inside the driver tests/cpp/shim_imu_routes_test.cpp, compiled here
into a temporary directory.  Before timing, one untimed solve of each routing checks that the device-routed one routes every
residual block and that both take the same iterations to the same termination.  The table reports the median wall time per solve
and per iteration.  Prints the GPU's name, power limit and SM clock limit, then one JSON line."""
import argparse, json, os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from tests import shim_common as sc
from tests import test_shim_imu_routes as ti


def timed(exe, mode, path, reps, iters, *flags):
    rows = sc.run_driver(exe, mode, [path], *flags, "--repeat", str(reps + 1), "--max-iter", str(iters))[0]["times"][1:]   # the first solve warms up
    ms = [r[0] for r in rows]; its = [r[1] for r in rows]
    return dict(median_ms=float(np.median(ms)), iterations=sorted(set(its)), median_ms_per_iteration=float(np.median([m / max(i, 1) for m, i in zip(ms, its)])),
                device_imu_blocks=sorted(set(r[3] for r in rows)), device_blocks=sorted(set(r[4] for r in rows)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps-large", type=int, default=2, help="host-routed solves of the K >= 2000 cases")
    ap.add_argument("--iters", type=int, default=3, help="iteration cap of every timed solve")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shim_imu_routes.py needs a CUDA device")
    gpu = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
    print("gpu:", gpu, flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        exe = sc.build_driver(tmp, "shim_imu_routes_test")
        out = dict(gpu=gpu, iteration_cap=a.iters, cases={})
        for K in (200, 2000, 3457):
            name = f"level1_k{K}"
            c = ti.level1(K)
            path = os.path.join(tmp, name + ".bin")
            ti.write_case(path, c, max_iter=a.iters)
            dev = sc.run_driver(exe, "device", [path])[0]
            host = sc.run_driver(exe, "host", [path])[0]
            if dev["device_imu"] != K - 1 or dev["device_blocks"] != dev["blocks"]:
                sys.exit(f"{name}: {dev['device_blocks']} of {dev['blocks']} blocks ({dev['device_imu']} of {K - 1} IMU) were routed to the device")
            if (dev["n_iters"], dev["termination"]) != (host["n_iters"], host["termination"]):
                sys.exit(f"{name}: device-routed {dev['n_iters']} iterations / termination {dev['termination']}, host-routed "
                         f"{host['n_iters']} / {host['termination']}")
            info = dict(blocks=dev["blocks"], imu_blocks=K - 1, attitude_blocks=len(c["att"][0]), binary_blocks=len(c["binary"]),
                        iterations=dev["n_iters"], termination=dev["termination"])
            info["host"] = timed(exe, "host", path, a.host_reps_large if K >= 2000 else a.reps, a.iters)
            info["imu_on_host"] = timed(exe, "device", path, a.reps, a.iters, "--imu-as-cost-function")
            info["device"] = timed(exe, "device", path, a.reps, a.iters)
            info["speedup_per_iteration"] = info["host"]["median_ms_per_iteration"] / info["device"]["median_ms_per_iteration"]
            info["speedup_per_iteration_vs_imu_on_host"] = info["imu_on_host"]["median_ms_per_iteration"] / info["device"]["median_ms_per_iteration"]
            out["cases"][name] = info
            print(name, json.dumps(info), flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
