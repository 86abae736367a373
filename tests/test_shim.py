"""Ceres-API shim (glio_b200/shim/ceres): a problem built with the reference's own call sequence
(AddParameterBlock / AddResidualBlock(AutoDiffCostFunction, HuberLoss, ...) / ceres::Solve) gives the oracle's iterates —
host-only (CPU) and with the LiDAR residual blocks routed to the CUDA kernels (GPU)."""
import numpy as np
import pytest

from glio_b200 import synth
from tests import shim_common as sc


def _check(res, ro, W):
    so = ro["summary"]
    assert res["termination"] == so.termination
    assert res["n_iters"] == so.num_iterations >= 3
    for (i, ok, cost, radius), io in zip(res["iters"], ro["iterations"]):
        assert ok == io["step_is_successful"]
        assert cost == pytest.approx(io["cost"], rel=1e-9)
        assert radius == pytest.approx(io["trust_region_radius"], rel=1e-9)
    assert np.max(np.abs(res["poses"] - ro["poses"])) <= 1e-6
    assert np.max(np.abs(res["sb"] - ro["speed_bias"])) <= 1e-6
    assert res["const"] == (0.3, 3.0)                      # constant blocks untouched
    assert res["blocks"] == (3 * W, 15 * W)                # unused / constant blocks removed from the program


def test_shim_host_only_matches_oracle(tmp_path, oracle):
    exe = sc.build_driver(tmp_path, "shim_test")
    P, kf, cp, nsd, w, sb0, priors, betweens, ranges = sc.make_problem(oracle, synth)
    path = str(tmp_path / "p.bin")
    sc.write_problem(path, P["poses_init"], sb0, P["q_lb"], P["t_lb"], 7.5, 1.0, kf, cp, nsd, w, priors, betweens, ranges)
    ro = sc.oracle_solve(oracle, P, kf, cp, nsd, w, sb0, priors, betweens, ranges)
    res = sc.run_driver(exe, "host", [path])[0]
    assert res["device_blocks"] == 0
    _check(res, ro, 4)


@pytest.mark.gpu
def test_shim_device_routing_matches_oracle(tmp_path, oracle):
    exe = sc.build_driver(tmp_path, "shim_test")
    P, kf, cp, nsd, w, sb0, priors, betweens, ranges = sc.make_problem(oracle, synth)
    path = str(tmp_path / "p.bin")
    sc.write_problem(path, P["poses_init"], sb0, P["q_lb"], P["t_lb"], 7.5, 1.0, kf, cp, nsd, w, priors, betweens, ranges)
    ro = sc.oracle_solve(oracle, P, kf, cp, nsd, w, sb0, priors, betweens, ranges)
    res = sc.run_driver(exe, "device", [path])[0]
    assert res["device_blocks"] == len(kf)                 # every LidarPlaneNormFactor block ran on the GPU
    _check(res, ro, 4)


def _binary_case(tmp_path, oracle, mode):
    exe = sc.build_driver(tmp_path, "shim_test")
    P, kf, cp, nsd, w, sb0, priors, betweens, ranges = sc.make_problem(oracle, synth)
    binary = sc.make_binary(oracle, synth, P)
    path = str(tmp_path / "pb.bin")
    sc.write_problem(path, P["poses_init"], sb0, P["q_lb"], P["t_lb"], 7.5, 1.0, kf, cp, nsd, w, priors, betweens, ranges, binary=binary)
    ro = sc.oracle_solve(oracle, P, kf, cp, nsd, w, sb0, priors, betweens, ranges, binary=binary)
    res = sc.run_driver(exe, mode, [path])[0]
    return res, ro, len(kf), len(binary[0])


def test_shim_host_only_with_binary_factors(tmp_path, oracle):
    res, ro, nu, nb = _binary_case(tmp_path, oracle, "host")
    assert res["device_blocks"] == 0
    _check(res, ro, 4)


@pytest.mark.gpu
def test_shim_device_routing_with_binary_factors(tmp_path, oracle):
    """LidarPlaneNormFactor AND BinaryLidarPlaneNormFactor blocks of one problem both run on the GPU (K2 + K2b)."""
    res, ro, nu, nb = _binary_case(tmp_path, oracle, "device")
    assert res["device_blocks"] == nu + nb
    _check(res, ro, 4)
