#!/usr/bin/env python
"""ceres::Solve through the Ceres-API shim, host-routed against device-routed, for the routes of LidarPlaneNormIncreFactor (K2 in
a front-end context) and LidarEdgeFactor (K2e):
  - front end: one scan-matching round, one pose, about 10 000 LidarPlaneNormIncreFactor blocks (the oracle's association of an
    11 500-point scan against a 54 000-point map with the front end's gates), HuberLoss(0.1), LEVENBERG_MARQUARDT, DENSE_QR, at
    most 4 iterations and the reference's 0.015 s time limit (LidarOdometry.cpp:499-530); and the same round with the time
    limit lifted, so that both routings run the same 4 iterations;
  - window: W = 20 keyframes with speed-bias, a prior and the IMU-like chain, plane and edge blocks per keyframe at 100 + 100 (the
    shipped selection sizes) and 10 000 + 8 000 (no selection); Estimator.cpp's options (DOGLEG, 15 iterations).
Each solve is timed with a host clock around ceres::Solve (which ends with the device results on the host) inside the driver
tests/cpp/shim_routes_test.cpp, compiled here into a temporary directory.  Before timing, one untimed device-routed solve of each
case checks that every LiDAR block was routed.  Prints the GPU's name and power limit, then one JSON
line with the median wall time and the iteration counts per case and routing."""
import argparse, json, os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from glio_b200 import synth
from oracle import pyoracle as oracle
from tests import eval_reference as er
from tests import shim_common as sc
from tests import test_shim_routes as tr


def front_end_problem(path, time_limit=0.015):
    P = synth.window_problem(W=1, Q=11_500, M=54_000, seed=synth.SEED0 + 9)
    t2, q2 = synth.lidar_pose_in_world(P["poses_init"][0, :3], P["poses_init"][0, 3:])
    prm = oracle.default_params(); prm.kd_max_radius = 1.0; prm.surf_dist_thres = 0.06; prm.weight_min = 0.4; prm.lidar_const = 1.0
    o = oracle.assoc_scan_to_map(P["map_xyz"], P["scans"][0], t2, q2, prm=prm)
    v = o["status"] == oracle.GO_VALID
    tr.write_problem(path, np.concatenate([t2, q2])[None, :], tr.incre_records(P["scans"][0][v], o["nsd"][v]), tr.FRONT_CTX, strategy=1,
                     max_iter=4, time_limit=time_limit)
    return int(v.sum())


def window_problem(path, n_plane, n_edge, W=20, seed=11):
    """correspondences generated at the true poses (eval_reference's plane and edge fixtures), solved from perturbed poses"""
    rng = np.random.default_rng(seed)
    T = np.concatenate([np.stack([np.arange(W) * 1.0, np.zeros(W), np.zeros(W)], 1), np.tile([1.0, 0, 0, 0], (W, 1))], 1)
    init = synth.perturb(T, rng)
    ql, tl = synth.Q_LB, synth.T_LB
    lid = []
    for k in range(W):
        u = er.make_unary(rng, T[k], n_plane, ql, tl, noise=0.03)
        e = er.make_edges(rng, T[k], n_edge, ql, tl, noise=0.03)
        lid.append(tr.lidar_records(tr.PLANE, k, u["cp"], a=u["nsd"][:, :3], d=u["nsd"][:, 3], s=tr.LIDAR_CONST * u["weight"].astype(np.float64),
                                    q_lb=ql, t_lb=tl, loss=tr.HUBER))
        lid.append(tr.lidar_records(tr.EDGE, k, e["cp"], a=e["pa"], b=e["pb"], s=e["s"], q_lb=ql, t_lb=tl, loss=tr.HUBER))
    sw = np.concatenate([np.full(3, 20.0), np.full(3, 50.0), np.full(9, 5.0)])
    sb0 = np.zeros((W, 9))
    priors = [(0, T[0, :3], T[0, 3:], sb0[0], sw)]
    betweens = [(i, i + 1, synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3]), synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:]),
                 np.zeros(3), 0.1, sw * 0.5) for i in range(W - 1)]
    ctx = dict(q_lb=ql, t_lb=tl, lidar_const=tr.LIDAR_CONST, huber=tr.HUBER, unit_score=0)
    tr.write_problem(path, init, lid, ctx, sb=sb0, priors=priors, betweens=betweens)


def timed(exe, mode, path, reps):
    rows = sc.run_driver(exe, mode, [path], "--repeat", str(reps + 1))[0]["times"][1:]          # the first solve warms up
    return dict(median_ms=float(np.median([r[0] for r in rows])), iterations=sorted({r[1] for r in rows}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--host-reps-large", type=int, default=3, help="host-routed solves of the unselected window case")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shim_routes.py needs a CUDA device")
    gpu = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    print("gpu:", gpu, flush=True)
    oracle.build()
    with tempfile.TemporaryDirectory() as tmp:
        exe = sc.build_driver(tmp, "shim_routes_test")
        out = dict(gpu=gpu, cases={})
        cases = [("front_end_incre", None, 0.015), ("front_end_incre_no_time_limit", None, 1e9), ("window_w20_100p_100e", (100, 100), None),
                 ("window_w20_10000p_8000e", (10_000, 8_000), None)]
        for name, shape, time_limit in cases:
            path = os.path.join(tmp, name + ".bin")
            info = {}
            if shape is None:
                info["blocks"] = n_lidar = front_end_problem(path, time_limit)
                info["time_limit_s"] = time_limit
            else:
                window_problem(path, *shape)
                info["blocks_per_keyframe"] = dict(plane=shape[0], edge=shape[1])
                n_lidar = 20 * (shape[0] + shape[1])
            routed = sc.run_driver(exe, "device", [path])[0]["device_blocks"]
            if routed != n_lidar:
                sys.exit(f"{name}: {routed} of {n_lidar} LiDAR blocks were routed to the device")
            host_reps = a.host_reps_large if shape is not None and shape[0] >= 1000 else a.reps
            info["host"] = timed(exe, "host", path, host_reps)
            info["device"] = timed(exe, "device", path, a.reps)
            info["speedup"] = info["host"]["median_ms"] / info["device"]["median_ms"]
            out["cases"][name] = info
            print(name, json.dumps(info), flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
