"""Helpers for the Ceres-shim tests: build and run the shim drivers under tests/cpp, serialise tests/cpp/shim_test's window
problem, compare two solves."""
import os
import struct
import subprocess

import numpy as np
import pytest

from glio_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_driver(tmpdir, name):
    """compile tests/cpp/<name>.cpp against the shim headers and the in-tree libglio_b200.so"""
    exe = os.path.join(str(tmpdir), name)
    cmd = ["/usr/bin/g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "glio_b200", "shim"), os.path.join(ROOT, "tests", "cpp", name + ".cpp"),
           "-o", exe, "-L", os.path.join(ROOT, "glio_b200"), "-lglio_b200", "-Wl,-rpath," + os.path.join(ROOT, "glio_b200"),
           "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"]
    subprocess.check_call(cmd)
    return exe


def run_driver(exe, mode, paths, *flags, desc_ints=0):
    """run a shim driver on problem files; one record per `solve` line it prints, each with the lines that follow as `text`.
    desc_ints: how many leading integers the driver's `desc` lines have before their hex-float values"""
    out = subprocess.check_output([exe, mode, *flags, *[str(p) for p in paths]], text=True)
    res, head = [], {}
    for line in out.splitlines():
        key, *v = line.split()
        if key == "preload_cost":
            head["preload_cost"] = float(v[0])
        if key.startswith("preload"):
            continue
        if key == "solve":
            res.append(dict(iters=[], poses={}, sb={}, text=[], desc=[], frames=[], times=[])); continue
        r = res[-1]
        r["text"].append(line)
        if key == "iters": r["n_iters"] = int(v[0])
        elif key in ("termination", "blocks") or key.startswith("device_") or key.endswith("_launches"):
            r[key] = int(v[0]) if len(v) == 1 else tuple(int(x) for x in v)
        elif key in ("cost", "const"): r[key] = (float(v[0]), float(v[1]))
        elif key in ("eval_cost", "gate_margin"): r[key] = float(v[0])
        elif key == "it": r["iters"].append((int(v[0]), int(v[1]), float(v[2]), float(v[3])))
        elif key in ("pose", "sb"): r["poses" if key == "pose" else "sb"][int(v[0])] = np.array([float(x) for x in v[1:]])
        elif key == "gradient": r["gradient"] = np.array([float(x) for x in v])
        elif key == "frame": r["frames"].append(np.array([float.fromhex(x) for x in v]).reshape(3, 3))
        elif key == "time": r["times"].append((float(v[0]), *(int(x) for x in v[1:])))
        elif key == "desc": r["desc"].append((*(int(x) for x in v[:desc_ints]), [float.fromhex(x) for x in v[desc_ints:]]))
    for r in res:
        if r["poses"]:
            r["poses"] = np.array([r["poses"][k] for k in sorted(r["poses"])]); r["sb"] = np.array([r["sb"][k] for k in sorted(r["sb"])])
    if res:
        res[0].update(head)
    return res


def rot_err(qa, qb):
    """rotation angle between two sets of unit quaternions (N, 4)"""
    qa = np.atleast_2d(qa); qb = np.atleast_2d(qb)
    d = np.array([synth.quat_mul(synth.quat_conj(a), b) for a, b in zip(qa, qb)])
    return float(np.max(2.0 * np.linalg.norm(d[:, 1:], axis=1)))


def assert_same_solve(a, b, sb=True, iterate_abs=0.0):
    """same termination, iterations and accept/reject decisions, initial and final cost rel 1e-9, poses 1e-6 m / 1e-8 rad,
    speed-bias 1e-6 (sb).  Iterates compare within 1e-9 relative plus iterate_abs of the initial cost: an iterate's cost carries
    the rounding of the steps, taken at the scale of the initial cost, and the batch problems' attitude factors (weight 10^4) make
    the first step drop the cost by three to five orders of magnitude."""
    assert a["termination"] == b["termination"]
    assert a["n_iters"] == b["n_iters"] >= 2
    assert [i[1] for i in a["iters"]] == [i[1] for i in b["iters"]]
    assert a["cost"][0] == pytest.approx(b["cost"][0], rel=1e-9)
    for x, y in zip(a["iters"], b["iters"]):
        assert x[2] == pytest.approx(y[2], rel=1e-9, abs=iterate_abs * b["cost"][0])
    assert a["cost"][1] == pytest.approx(b["cost"][1], rel=1e-9)
    assert np.max(np.abs(a["poses"][:, :3] - b["poses"][:, :3])) <= 1e-6
    assert rot_err(a["poses"][:, 3:], b["poses"][:, 3:]) <= 1e-8
    if sb:
        assert np.max(np.abs(a["sb"] - b["sb"])) <= 1e-6


def write_problem(path, poses, sb, q_lb, t_lb, lidar_const, huber, kf, cp, nsd, w, priors, betweens, ranges, binary=None):
    W = len(poses)
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", W, 1 if sb is not None else 0))
        f.write(np.ascontiguousarray(poses, np.float64).tobytes())
        f.write(np.ascontiguousarray(sb if sb is not None else np.zeros((W, 9)), np.float64).tobytes())
        f.write(np.ascontiguousarray(q_lb, np.float64).tobytes()); f.write(np.ascontiguousarray(t_lb, np.float64).tobytes())
        f.write(struct.pack("<dd", lidar_const, huber))
        f.write(struct.pack("<i", len(kf)))
        f.write(np.ascontiguousarray(kf, np.int32).tobytes()); f.write(np.ascontiguousarray(cp, np.float32).tobytes())
        f.write(np.ascontiguousarray(nsd, np.float32).tobytes()); f.write(np.ascontiguousarray(w, np.float32).tobytes())
        f.write(struct.pack("<i", len(priors)))
        for (k, t0, q0, sb0, sw) in priors:
            f.write(struct.pack("<i", k)); f.write(np.asarray(t0, np.float64).tobytes()); f.write(np.asarray(q0, np.float64).tobytes())
            f.write(np.asarray(sb0 if sb0 is not None else np.zeros(9), np.float64).tobytes()); f.write(np.asarray(sw, np.float64).tobytes())
        f.write(struct.pack("<i", len(betweens)))
        for (i, j, dp, dq, dv, dt, sw) in betweens:
            f.write(struct.pack("<ii", i, j)); f.write(np.asarray(dp, np.float64).tobytes()); f.write(np.asarray(dq, np.float64).tobytes())
            f.write(np.asarray(dv, np.float64).tobytes()); f.write(struct.pack("<d", dt)); f.write(np.asarray(sw, np.float64).tobytes())
        f.write(struct.pack("<i", len(ranges)))
        for (k, lever, sat, rho, w_) in ranges:
            f.write(struct.pack("<i", k)); f.write(np.asarray(lever, np.float64).tobytes()); f.write(np.asarray(sat, np.float64).tobytes())
            f.write(struct.pack("<dd", rho, w_))
        if binary is not None:
            kc, ko, bcp, bnc, bsc = binary
            f.write(struct.pack("<i", len(kc)))
            f.write(np.ascontiguousarray(kc, np.int32).tobytes()); f.write(np.ascontiguousarray(ko, np.int32).tobytes())
            f.write(np.ascontiguousarray(bcp, np.float32).tobytes()); f.write(np.ascontiguousarray(bnc, np.float64).tobytes())
            f.write(np.ascontiguousarray(bsc, np.float64).tobytes())


def make_problem(oracle, synth, W=4, Q=800, M=20000, seed=17, n_sel=150):
    """Matches from the ORACLE association (CPU), a fixed selection, host factor specs; returns everything both sides need."""
    P = synth.window_problem(W=W, Q=Q, M=M, seed=seed)
    rng = np.random.default_rng(seed)
    tree = oracle.KdTree(P["map_xyz"])
    kf, cp, nsd, w = [], [], [], []
    for k in range(W):
        t2, q2 = synth.lidar_pose_in_world(P["poses_init"][k, :3], P["poses_init"][k, 3:])
        o = oracle.assoc_scan_to_map(P["map_xyz"], P["scans"][k], t2, q2, tree=tree)
        v = np.nonzero(o["status"] == 0)[0][:n_sel]
        kf.append(np.full(len(v), k, np.int32)); cp.append(P["scans"][k][v]); nsd.append(o["nsd"][v]); w.append(o["weight"][v])
    kf, cp, nsd, w = map(np.concatenate, (kf, cp, nsd, w))
    sb0 = rng.normal(0, 0.1, (W, 9))
    T = P["poses_true"]
    sw = np.concatenate([np.full(3, 20.0), np.full(3, 50.0), np.full(9, 5.0)])
    priors = [(0, T[0, :3] + 0.01, T[0, 3:], sb0[0], sw)]
    betweens = []
    for i in range(W - 1):
        dq = synth.quat_mul(synth.quat_conj(T[i, 3:]), T[i + 1, 3:])
        dp = synth.quat_to_R(T[i, 3:]).T @ (T[i + 1, :3] - T[i, :3])
        betweens.append((i, i + 1, dp + rng.normal(0, 0.01, 3), dq, np.zeros(3), 0.1, sw * 0.5))
    ranges = [(k, [0.0, 0.1, 0.2], np.array([2.0e4 * np.cos(k), 2.0e4 * np.sin(k), 2.0e4]), 0.0, 0.7) for k in range(W)]
    ranges = [(k, lv, sat, float(np.linalg.norm(T[k, :3] - sat) + 0.3), wt) for (k, lv, sat, _, wt) in ranges]
    return P, kf, cp, nsd, w, sb0, priors, betweens, ranges


def make_binary(oracle, synth, P, pairs=((0, 1), (1, 0), (2, 1), (3, 2), (1, 3)), n_sel=120, batch_score=2.5, Qb=5000):
    """Scan-to-multiscan matches between keyframes of the window problem, from the ORACLE pair association.  The batch
    path applies the keyframe poses directly to the stored scan points (quirk Q7), so denser body-frame scans of the
    same scene / trajectory are drawn here (same RNG order as synth.window_problem rebuilds scene and truth)."""
    rng = np.random.default_rng(P["seed"])
    scene = synth.Scene(-60.0, P["W"] + 60.0, rng, n_boxes=30)
    truth = synth.trajectory(P["W"], rng)
    assert np.array_equal(truth, P["poses_true"])
    r2 = np.random.default_rng(P["seed"] + 1000)
    scans = [synth.scan_in_body_frame(scene, truth[k], Qb, r2, rng_range=12.0) for k in range(P["W"])]
    kc, ko, cp, nc, sc = [], [], [], [], []
    for (c, o) in pairs:
        a = oracle.assoc_pair(scans[c], P["poses_init"][c, :3], P["poses_init"][c, 3:], scans[o], P["poses_init"][o, :3], P["poses_init"][o, 3:])
        v = np.nonzero(a["status"] == 0)[0][:n_sel]
        assert len(v) > 20, len(v)
        kc.append(np.full(len(v), c, np.int32)); ko.append(np.full(len(v), o, np.int32)); cp.append(scans[c][v])
        nc.append(a["normal_cent"][v]); sc.append(batch_score * a["weight"][v].astype(np.float64))
    return tuple(map(np.concatenate, (kc, ko, cp, nc, sc)))


def oracle_solve(oracle, P, kf, cp, nsd, w, sb0, priors, betweens, ranges, lidar_const=7.5, binary=None):
    prob = oracle.WindowProblem(P["poses_init"], sb0, P["q_lb"], P["t_lb"], huber_delta=1.0)
    prob.add_unary(kf, cp, nsd, lidar_const * w.astype(np.float64))
    if binary is not None:
        prob.add_binary(*binary)
    for a in priors: prob.add_prior(*a)
    for a in betweens: prob.add_between(*a)
    for a in ranges: prob.add_range(*a)
    return prob.solve(oracle.solver_options(), mode=0)
