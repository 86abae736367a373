"""Sequential restatement of the scan-to-multiscan edge association (glio_batch_associate_edges_pairs, include/glio_b200.h
K1be steps 1-8).  Helper module for the tests (not collected).

Steps 1-2 use the CPU oracle's transform and exact 5-NN, with the searched frame's world cloud formed by the same transform; steps
3-7 are tests/edge_reference.py's line fit on the five world points, and step 8 repeats its centroid, scatter matrix and Jacobi on
the same five indices in the searched frame's stored coordinates.  All of it in Python floats (IEEE doubles, no fused
multiply-add), the arithmetic the device performs with -fmad=false, so both agree bit for bit.
"""
import numpy as np

from tests import edge_reference as er

VALID, FAIL_RADIUS, FAIL_LINE = er.VALID, er.FAIL_RADIUS, er.FAIL_LINE


def local_line(nb_local, half_length):
    """Step 8: the line of five local-frame points (float32, neighbour order): (pa, pb) float32, plus c and v."""
    c, A = er.centroid_scatter(nb_local)
    _, v, _ = er.jacobi_eig3(A)
    h = half_length
    pa = np.array([c[i] + h * v[i] for i in range(3)]).astype(np.float32)
    pb = np.array([c[i] - h * v[i] for i in range(3)]).astype(np.float32)
    return pa, pb, c, v


def associate_pair(po, cur_xyz, cur_pose, oth_xyz, oth_pose, opts=None, brute=False):
    """One pair (cur, oth): cur_xyz / oth_xyz the corner scans as stored ((n, stride) arrays), poses (t, q) as registered.
    Returns per-query status, idx5, sqd5, and the emitted lists cp, pa, pb, s, src, n in scan order."""
    o = dict(er.DEFAULTS, **(opts or {}))
    cs = np.ascontiguousarray(np.asarray(cur_xyz, np.float32)[:, :3])          # (n, stride) arrays: x, y, z first
    os_ = np.ascontiguousarray(np.asarray(oth_xyz, np.float32)[:, :3])
    Q = len(cs)
    status = np.full(Q, FAIL_RADIUS, np.uint8)
    idx5 = np.full((Q, 5), -1, np.int32); sqd5 = np.full((Q, 5), np.inf, np.float32)
    pa = np.zeros((Q, 3), np.float32); pb = np.zeros((Q, 3), np.float32)
    if Q and len(os_) >= 5:
        pw = po.transform_points(cs, cur_pose[:3], cur_pose[3:])
        ow = po.transform_points(os_, oth_pose[:3], oth_pose[3:])
        if brute:
            idx5, sqd5 = po.knn5_brute(ow, pw)[:2]
        else:
            idx5, sqd5 = po.KdTree(ow).knn5(pw)
        for i in range(Q):
            st, _, _, _ = er.line_fit(ow[idx5[i]], sqd5[i, 4], o)
            status[i] = st
            if st == VALID:
                pa[i], pb[i], _, _ = local_line(os_[idx5[i]], o["half_length"])
    v = status == VALID
    n = int(v.sum())
    return dict(status=status, idx5=idx5, sqd5=sqd5, cp=cs[v], pa=pa[v], pb=pb[v], s=np.full(n, float(np.float32(o["score"]))),
                src=np.nonzero(v)[0].astype(np.int32), n=n)
