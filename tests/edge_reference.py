"""Sequential restatement of the edge association (glio_window_associate_edges, include/glio_b200.h steps 1-8).

Steps 1-2 use the CPU oracle's transform and exact 5-NN (brute force or kd-tree, oracle/pyoracle.py); steps 3-8 are written
here in Python floats: IEEE doubles, every operation rounded on its own (no fused multiply-add), math.sqrt correctly rounded.
That is the arithmetic the device's k_line_fit performs with -fmad=false and explicit *_rn intrinsics, so both agree bit for bit.
"""
import math

import numpy as np

VALID, FAIL_RADIUS, FAIL_LINE = 0, 1, 2
DEFAULTS = dict(max_sqdist=1.0, min_ratio=3.0, half_length=0.1, score=1.0)
MAX_SWEEPS = 32


def _rotate(a, v, p, q):
    apq = a[p][q]
    if apq == 0.0:
        return
    g = 100.0 * abs(apq)
    if abs(a[p][p]) + g == abs(a[p][p]) and abs(a[q][q]) + g == abs(a[q][q]):
        a[p][q] = 0.0; a[q][p] = 0.0
        return
    theta = (a[q][q] - a[p][p]) / (2.0 * apq)
    t = 1.0 / (abs(theta) + math.sqrt(theta * theta + 1.0))      # theta^2 overflowing to inf gives t = 0, as on the device
    if theta < 0.0:
        t = -t
    c = 1.0 / math.sqrt(t * t + 1.0)
    s = t * c
    tapq = t * apq
    a[p][p] = a[p][p] - tapq
    a[q][q] = a[q][q] + tapq
    a[p][q] = 0.0; a[q][p] = 0.0
    r = 3 - p - q
    arp, arq = a[r][p], a[r][q]
    a[r][p] = a[p][r] = c * arp - s * arq
    a[r][q] = a[q][r] = s * arp + c * arq
    for i in range(3):
        vip, viq = v[i][p], v[i][q]
        v[i][p] = c * vip - s * viq
        v[i][q] = s * vip + c * viq


def jacobi_eig3(C):
    """Cyclic Jacobi of the symmetric 3x3 C (nested lists or array of doubles).  Returns (lam ascending, stable by index;
    the eigenvector of lam[2] with its largest-magnitude component, lowest index on ties, positive; sweeps used)."""
    a = [[float(C[i][j]) for j in range(3)] for i in range(3)]
    v = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]
    sweeps = 0
    for _ in range(MAX_SWEEPS):
        if a[0][1] == 0.0 and a[0][2] == 0.0 and a[1][2] == 0.0:
            break
        _rotate(a, v, 0, 1); _rotate(a, v, 0, 2); _rotate(a, v, 1, 2)
        sweeps += 1
    order = sorted(range(3), key=lambda i: (a[i][i], i))
    lam = [a[i][i] for i in order]
    d = [v[0][order[2]], v[1][order[2]], v[2][order[2]]]
    big = d[0]
    if abs(d[1]) > abs(big):
        big = d[1]
    if abs(d[2]) > abs(big):
        big = d[2]
    if big < 0.0:
        d = [-d[0], -d[1], -d[2]]
    return lam, d, sweeps


def centroid_scatter(nb):
    """Step 4-5: centroid (sum nearest first, / 5.0) and the undivided scatter matrix of five float32 points, in double."""
    x = [[float(nb[j][i]) for i in range(3)] for j in range(5)]
    c = [((((x[0][i] + x[1][i]) + x[2][i]) + x[3][i]) + x[4][i]) / 5.0 for i in range(3)]
    A = [[0.0] * 3 for _ in range(3)]
    for j in range(5):
        dx, dy, dz = x[j][0] - c[0], x[j][1] - c[1], x[j][2] - c[2]
        A[0][0] += dx * dx; A[0][1] += dx * dy; A[0][2] += dx * dz
        A[1][1] += dy * dy; A[1][2] += dy * dz; A[2][2] += dz * dz
    A[1][0] = A[0][1]; A[2][0] = A[0][2]; A[2][1] = A[1][2]
    return c, A


def line_fit(nb, sqd4, opts=None):
    """Steps 3-8 for one query: nb (5, 3) float32 neighbours nearest first, sqd4 the squared 5th distance (float32).
    Returns (status, eig (3,), pa (3,) float32, pb (3,) float32)."""
    o = dict(DEFAULTS, **(opts or {}))
    zero = np.zeros(3, np.float32)
    if not (float(sqd4) < o["max_sqdist"]):
        return FAIL_RADIUS, np.zeros(3), zero, zero
    c, A = centroid_scatter(nb)
    lam, v, _ = jacobi_eig3(A)
    if not (lam[2] > o["min_ratio"] * lam[1]):
        return FAIL_LINE, np.array(lam), zero, zero
    h = o["half_length"]
    pa = np.array([c[i] + h * v[i] for i in range(3)]).astype(np.float32)
    pb = np.array([c[i] - h * v[i] for i in range(3)]).astype(np.float32)
    return VALID, np.array(lam), pa, pb


def associate_edges(po, map_xyz, scan_xyz, t2, q2, opts=None, tree=None):
    """The whole association of one corner scan against a corner map (po: oracle.pyoracle; tree: its KdTree, or None for the
    brute-force search).  Returns per-query pm, idx5, sqd5, status, eig and the emitted lists cp, pa, pb, s, src in scan order."""
    o = dict(DEFAULTS, **(opts or {}))
    m = np.ascontiguousarray(map_xyz, np.float32).reshape(-1, 3)
    s = np.ascontiguousarray(scan_xyz, np.float32)
    xyz = np.ascontiguousarray(s[:, :3])
    pm = po.transform_points(xyz, t2, q2)
    idx5, sqd5 = tree.knn5(pm) if tree is not None else po.knn5_brute(m, pm)[:2]
    Q = len(xyz)
    status = np.empty(Q, np.uint8); eig = np.zeros((Q, 3)); pa = np.zeros((Q, 3), np.float32); pb = np.zeros((Q, 3), np.float32)
    for i in range(Q):
        status[i], eig[i], pa[i], pb[i] = line_fit(m[idx5[i]], sqd5[i, 4], o)
    v = status == VALID
    return dict(pm=pm, idx5=idx5, sqd5=sqd5, status=status, eig=eig, cp=xyz[v], pa=pa[v], pb=pb[v],
                s=np.full(int(v.sum()), float(np.float32(o["score"]))), src=np.nonzero(v)[0].astype(np.int32), n=int(v.sum()))
