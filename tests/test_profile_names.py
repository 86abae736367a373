"""Every kernel name the CUDA library hands its launch counter is one Context.lib_profile_read() reports: a name missing from
Context.KERNELS would have its times dropped without an error.  Reads the sources only (no library, no GPU)."""
import glob
import os
import re

from glio_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _launch_names():
    names = set()
    for path in glob.glob(os.path.join(ROOT, "glio_b200", "csrc", "*.cu")):
        src = open(path).read()
        for arg in re.findall(r"\blc\.begin\(([^,;]*),", src):          # first argument: "k_x" or cond ? "k_a" : "k_b"
            found = re.findall(r'"(k_\w+)"', arg)
            assert found, f"{os.path.basename(path)}: lc.begin({arg}, ...) names no kernel literally"
            names.update(found)
    return names


def test_every_launch_counter_name_is_profiled():
    names = _launch_names()
    assert {"k_eval_unary", "k_eval_unary_cost", "k_eval_binary_edge_cost", "k_plane_fit_pair"} <= names   # both arms of the conditionals
    missing = sorted(names - set(api.Context.KERNELS))
    assert not missing, missing
