"""The edge selection's specification on the CPU (tests/edge_select_reference.py): the plane rules of tests/select_reference.py
applied to edge counts in Philox domains 3 (window), 4 (batch start/end) and 5 (batch incremental), and the Python mirror of the
four C calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import select_reference as sr
from tests.edge_select_reference import batch_select, window_select

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["glio_select_random_edges", "glio_get_edge_selection", "glio_batch_select_random_edges", "glio_batch_get_edge_selection"]


# ---- the edge rules differ from the plane rules only through the domain ---------------------------------------------------------

@pytest.mark.parametrize("n", [0, 1, 2, 99, 100, 101, 102, 103, 299, 300, 301, 302, 1000, 8300])
def test_window_rule_at_the_plane_domain_is_the_plane_rule(n):
    for F, R, rs in ((100, 300, True), (7, 2, True), (100, 300, False)):
        assert window_select(n, 17, 3, 1, F=F, R=R, random_select=rs, domain=sr.DOMAIN_WINDOW) == \
            sr.window_select(n, 17, 3, 1, F=F, R=R, random_select=rs)


@pytest.mark.parametrize("mode", [0, 1])
def test_batch_rules_at_the_plane_domains_are_the_plane_rules(mode):
    pairs = [(5, 2), (5, 3), (5, 4), (5, 6), (6, 3), (6, 4), (7, 1), (7, 2)]
    n = [500, 40, 500, 500, 50, 9300, 26, 24]
    plane_domain = sr.DOMAIN_BATCH_STARTEND if mode == 0 else sr.DOMAIN_BATCH_ADD
    assert batch_select(pairs, n, mode, 2, 0, domain=plane_domain) == sr.batch_select(pairs, n, mode, 2, 0)


@pytest.mark.parametrize("n", [101, 102, 1000, 8300])
def test_window_edge_draws_are_their_own(n):
    keep, undefined = window_select(n, 4, 9, 0)
    plane, plane_undefined = sr.window_select(n, 4, 9, 0)
    assert len(keep) == 100 and len(set(keep)) == 100 and max(keep) <= n - 2
    assert undefined == plane_undefined and keep != plane
    assert keep == sr.sample_from_draws(n, sr.draws(9, 3, 4, 0, n, 100))


def test_batch_edge_draws_are_their_own():
    pairs = [(1, 2), (1, 3), (2, 1)]
    n = [9300, 60, 1000]
    for mode, dom in ((0, 4), (1, 5)):
        edge, plane = batch_select(pairs, n, mode, 1, 7), sr.batch_select(pairs, n, mode, 1, 7)
        assert [k is None for k, _ in edge] == [k is None for k, _ in plane]
        assert [u for _, u in edge] == [u for _, u in plane]
        for (cur, oth), cnt, (k, _), (p, _) in zip(pairs, n, edge, plane):
            assert k != p and k == sr.sample_from_draws(cnt, sr.draws(1, dom, sr.stream_of_pair(cur, oth), 7, cnt, 25))
    (a, _), = batch_select([(1, 2)], [1000], 0, 1, 7)
    (b, _), = batch_select([(1, 2)], [1000], 1, 1, 7)
    assert a != b                                                  # start/end and incremental edge draws differ


@pytest.mark.parametrize("n,expect", [(0, None), (49, None), (50, "undefined"), (51, 25), (425, 25), (426, 25)])
def test_startend_edge_sizes(n, expect):
    (keep, undef), = batch_select([(3, 4)], [n], 0, seed=1, nonce=0)
    if expect is None:
        assert keep is None and not undef
    else:
        assert len(keep) == 25 and max(keep) <= n - 2 and undef == (expect == "undefined")


def test_last_edge_is_never_drawn():
    for s in range(40):
        keep, _ = window_select(102, s, 0, 0)
        assert 101 not in keep
        (k, _), = batch_select([(0, 1)], [26], 1, s, 0)
        assert 25 not in k and len(k) == 25


# ---- the Python mirror passes the declared arguments --------------------------------------------------------------------------

def _header_params():
    src = open(os.path.join(ROOT, "include", "glio_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for name in NEW:
        m = re.search(r"\b" + name + r"\s*\(([^)]*)\)\s*;", src)
        assert m, name
        out[name] = [p.strip() for p in m.group(1).split(",")]
    return out


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return 0
        return f


def _ctype_ok(decl, arg):
    if decl.startswith("glio_ctx*"):
        return arg is None
    if "*" in decl:
        return arg is None or isinstance(arg, C.c_void_p) or type(arg).__name__ == "CArgObject"
    if decl.startswith("int64_t"):
        return isinstance(arg, C.c_int64)
    if decl.startswith("int "):
        return isinstance(arg, C.c_int)
    return False


def test_new_symbols_are_exported_and_the_mirror_passes_their_arguments():
    from glio_b200 import api
    lib = C.CDLL(os.path.join(ROOT, "glio_b200", "libglio_b200.so"))
    for n in NEW:
        assert hasattr(lib, n), n
    params = _header_params()
    ctx = object.__new__(api.Context)
    rec = _Recorder()
    ctx._lib = rec; ctx._h = None; ctx._chk = lambda rc: None
    opt = api.SelectOptions()
    ctx.select_random_edges([3, 4], opt)
    ctx.get_edge_selection(1)
    ctx.batch_select_random_edges([0, 0], [1, 2], 1, opt)
    ctx.batch_get_edge_selection(0, 1)
    called = [c for c in rec.calls if c[0] in NEW]
    assert {c[0] for c in called} == set(NEW)
    for name, args in called:
        decl = params[name]
        assert len(args) == len(decl), (name, len(args), decl)
        for d, a in zip(decl, args):
            assert _ctype_ok(d, a), (name, d, a)
    with pytest.raises(ValueError):
        ctx.batch_select_random_edges([0, 0], [1], 1, opt)
    assert np.array_equal(ctx.select_random_edges([3, 4], opt), [0, 0])
