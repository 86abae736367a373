#!/usr/bin/env python
"""ceres::Solve through the Ceres-API shim, host-routed against device-routed, for the batch refinement's DD pseudorange factors
(K2g, dd_psr_factor_20): the shipped sms_fusion_level 0 problem of synth.dd_psr_problem (attitude then relative factors, constant
yaw and anchor, the DD factors of outer pass 1 per epoch and constellation) at K = 200, 2 000 and 3 457 keyframes (the sample
run's size).  Host-routed, every block is evaluated on the host (no context attached); device-routed, every block is on the GPU
(pose blocks by K2p, DD blocks by K2g).  A third timing, "pose_only", is the routing without this route: the same problem with the DD
factors added through a ceres::CostFunction*, so the pose blocks run on K2p and the DD blocks on the host.  The Estimator's options (SUBSPACE_DOGLEG, nonmonotonic steps), every solve capped at --iters iterations, timed with a host clock
around ceres::Solve (which ends with the device results on the host) inside the driver tests/cpp/shim_dd_psr_routes_test.cpp,
compiled here into a temporary directory.  Before timing, one untimed solve of each routing checks that the device-routed one
routes every residual block and that both take the same iterations to the same termination.  The table reports the median wall
time per solve and per iteration.  Prints the GPU's name, power limit and SM clock limit, then one JSON line."""
import argparse, json, os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from glio_b200 import api, synth
from tests import shim_common as sc
from tests import test_shim_dd_psr_routes as td


def timed(exe, mode, path, reps, iters, *flags):
    rows = sc.run_driver(exe, mode, [path], *flags, "--repeat", str(reps + 1), "--max-iter", str(iters))[0]["times"][1:]   # the first solve warms up
    ms = [r[0] for r in rows]; its = [r[1] for r in rows]
    return dict(median_ms=float(np.median(ms)), iterations=sorted(set(its)), median_ms_per_iteration=float(np.median([m / max(i, 1) for m, i in zip(ms, its)])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps-large", type=int, default=2, help="host-routed solves of the K >= 2000 cases")
    ap.add_argument("--iters", type=int, default=3, help="iteration cap of every timed solve")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shim_dd_psr_routes.py needs a CUDA device")
    gpu = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
    print("gpu:", gpu, flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        exe = sc.build_driver(tmp, "shim_dd_psr_routes_test")
        out = dict(gpu=gpu, iteration_cap=a.iters, cases={})
        for K in (200, 2000, 3457):
            name = f"level0_k{K}"
            P = synth.dd_psr_problem(K=K)
            dd, s = P["dd"], P["dd_sats"]
            f = api.dd_psr_factor_records(dd["i"], dd["j"], dd["n_sat"], dd["master"], dd["ratio"], dd["threshold"], dd["station"])
            dds = td.dd_from_records(f, api.dd_psr_sat_records(s["sat_user"], s["sat_ref"], s["psr_user"], s["psr_ref"]))
            path = os.path.join(tmp, name + ".bin")
            td.write_problem(path, P["poses_init"], pose=P, dds=dds, frames=[(0.3, P["anchor"], 1, 1)], max_iter=a.iters)
            dev = sc.run_driver(exe, "device", [path])[0]
            host = sc.run_driver(exe, "host", [path])[0]
            if dev["device_dd"] != len(dds) or dev["device_blocks"] != dev["blocks"]:
                sys.exit(f"{name}: {dev['device_blocks']} of {dev['blocks']} blocks ({dev['device_dd']} of {len(dds)} DD) were routed to the device")
            if (dev["n_iters"], dev["termination"]) != (host["n_iters"], host["termination"]):
                sys.exit(f"{name}: device-routed {dev['n_iters']} iterations / termination {dev['termination']}, host-routed "
                         f"{host['n_iters']} / {host['termination']}")
            info = dict(dd_blocks=len(dds), dd_rows=int(sum(len(d["user"]) - 1 for d in dds)), pose_blocks=len(P["i"]),
                        iterations=dev["n_iters"], termination=dev["termination"])
            info["host"] = timed(exe, "host", path, a.host_reps_large if K >= 2000 else a.reps, a.iters)
            info["pose_only"] = timed(exe, "device", path, a.reps, a.iters, "--dd-as-cost-function")
            info["device"] = timed(exe, "device", path, a.reps, a.iters)
            info["speedup_per_iteration"] = info["host"]["median_ms_per_iteration"] / info["device"]["median_ms_per_iteration"]
            info["speedup_per_iteration_vs_pose_only"] = info["pose_only"]["median_ms_per_iteration"] / info["device"]["median_ms_per_iteration"]
            out["cases"][name] = info
            print(name, json.dumps(info), flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
