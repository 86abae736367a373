"""Ceres' own unit-test expectations (loss_function_test.cc, corrector_test.cc, local_parameterization_test.cc, rotation /
jet checks; the reference vendors Ceres 2.0.0) against the PRODUCT's Ceres-API shim (glio_b200/shim/ceres)."""
import subprocess

from tests import shim_common as sc


def test_shim_against_ceres_known_answers(tmp_path):
    exe = sc.build_driver(tmp_path, "shim_known_answers")
    p = subprocess.run([exe], text=True, capture_output=True)
    lines = p.stdout.splitlines()
    assert len(lines) == 38, p.stdout + p.stderr
    bad = [l for l in lines if l.split()[1] != "ok"]
    assert not bad and p.returncode == 0, bad
