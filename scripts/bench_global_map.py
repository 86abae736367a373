#!/usr/bin/env python
"""The sort-based VoxelGrid (glio_voxel_filter) beside the dense one of glio_localmap_build, and save_pcd's global map
(glio_loop_global_map), on the device; the oracle's stable VoxelGrid on one CPU thread beside each.  Device numbers are medians of
CUDA-event timings of whole calls (each call returns when its work is complete); localmap_build's also include its K0 grid build,
so the per-kernel device times of one profiled call of each are printed too.  Prints one JSON line with the GPU's name and power
limit, read in the same run.  Not bench.py's metric."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from glio_b200 import api, synth
from oracle import pyoracle as po, pyoracle_loop as pl
from tests.global_map_reference import global_map

ap = argparse.ArgumentParser()
ap.add_argument("--scan", type=int, default=30000, help="points of the keyframe scan")
ap.add_argument("--frames", type=int, default=50); ap.add_argument("--frame_points", type=int, default=20000)
ap.add_argument("--reps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
a = ap.parse_args()
po.build(); pl.build()

ctx = api.Context(0); st = torch.cuda.ExternalStream(ctx.stream)
IDENT = (np.zeros(3), np.array([1.0, 0, 0, 0]))


def device_ms(fn):
    for _ in range(a.warmup):
        fn()
    ts = []
    for _ in range(a.reps):
        torch.cuda.synchronize(); e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(st); fn(); e1.record(st); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    return round(float(np.median(ts)), 4)


def kernels(fn):
    ctx.lib_profile(True)
    fn(); ctx.synchronize()
    p = {k: round(v[0], 4) for k, v in ctx.lib_profile_read().items()}
    ctx.lib_profile(False)
    return p


def cpu_ms(fn, reps=3):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(1e3 * (time.perf_counter() - t0))
    return round(float(np.median(ts)), 3)


def both_paths(cloud, leaf):
    """the sort path on a device-resident cloud vs localmap_build of one frame at the identity pose"""
    d = torch.from_numpy(np.ascontiguousarray(cloud)).cuda()
    ctx.localmap_clear(); ctx.localmap_push(d, *IDENT)
    sort = lambda: ctx.voxel_filter(d, leaf, out="device")
    dense = lambda: ctx.localmap_build(leaf)
    m, f = sort()
    assert f and np.array_equal(m.cpu().numpy(), (dense(), ctx.get_map())[1])
    r = dict(points=len(cloud), leaf=leaf, out_points=len(m), sort_ms=device_ms(sort), dense_build_ms=device_ms(dense),
             sort_kernels_ms=kernels(sort), dense_build_kernels_ms=kernels(dense),
             oracle_1thread_ms=cpu_ms(lambda: po.voxel_filter(cloud, leaf, stable=True)))
    ctx.localmap_clear()
    return r


rng = np.random.default_rng(7)
scene = synth.Scene(-60.0, a.frames + 60.0, rng)
poses = synth.trajectory(a.frames + 1, rng)
out = {}
scan = synth.scan_in_lidar_frame(scene, poses[0], a.scan, rng)
out["keyframe_scan_0.9"] = both_paths(scan, 0.9)
world = np.concatenate([po.transform_points(synth.scan_in_lidar_frame(scene, poses[k], a.frame_points, rng),
                                            *synth.lidar_pose_in_world(poses[k, :3], poses[k, 3:7])) for k in range(a.frames)])
out["local_map_%d_frames_0.4" % a.frames] = both_paths(world, 0.4)

D = synth.loop_drive()
loop = api.LoopClosure(ctx); L = pl.LoopOracle()
for k in range(D["K"]):
    loop.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k]); L.add_keyframe(D["clouds"][k], D["poses"][k], D["times"][k])
for interval in (1, 3):
    g = lambda: loop.global_map(interval, 0.2, out="device")
    m, f, n_raw = g()
    assert np.array_equal(m.cpu().numpy(), global_map(po, L, interval, 0.2)[0])
    out["global_map_interval_%d_0.2" % interval] = dict(keyframes=D["K"], raw_points=n_raw, out_points=len(m), device_ms=device_ms(g),
                                                        kernels_ms=kernels(g), oracle_1thread_ms=cpu_ms(lambda: global_map(po, L, interval, 0.2)))

big = np.concatenate([[[3900.5, 3900.5, 0.5]], rng.uniform(-20, 20, (1_000_000, 3))]).astype(np.float32)   # > 2^28 voxels at leaf 1
d = torch.from_numpy(big).cuda()
s = lambda: ctx.voxel_filter(d, 1.0, out="device")
m, f = s()
assert f and np.array_equal(m.cpu().numpy(), po.voxel_filter(big, 1.0, stable=True)[0])
out["box_above_2_28_voxels_1.0"] = dict(points=len(big), out_points=len(m), sort_ms=device_ms(s), sort_kernels_ms=kernels(s),
                                        dense="refused (more than 2^28 voxels)", oracle_1thread_ms=cpu_ms(lambda: po.voxel_filter(big, 1.0, stable=True)))

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps(dict(workload="sort-based VoxelGrid and global map export", gpu=torch.cuda.get_device_name(0), nvidia_smi=smi,
                      reps=a.reps, warmup=a.warmup, **out)))
ctx.close()
