"""Keyframe sharding of the batch (scan-to-multiscan) path across the GPUs of one box (SURVEY.md §8 e).

Units = (cur, oth) frame pairs.  A pair needs only the two scans and the two poses, so pairs are independent;
residual ownership follows the `cur` keyframe.  Every rank declares the same global pair list (same block
layout), associates and evaluates only the pairs it owns, and the pose-block buffers are summed over ranks once
per evaluation (one all-reduce of K*28 + P*36 doubles).  The band Cholesky / dogleg step is replicated.
"""
import ctypes as C
import os

import numpy as np


def batch_pairs(B, search_range, start_idx=0):
    """The (idx, search_idx) pairs optimizeBatchWithLandMark adds (GLIO/src/Estimator.cpp:3004-3019, 3034, 3056):
    a sliding neighbourhood of 2*search_range frames, shifted inwards at both ends of the batch."""
    cur, oth = [], []
    sr = search_range
    if B - start_idx < 2 * sr + 1:
        return np.zeros(0, np.int32), np.zeros(0, np.int32)
    for idx in range(start_idx, B):
        if idx >= sr + start_idx and idx < B - 1 - sr:
            s = idx - sr
        elif idx < sr + start_idx:
            s = start_idx
        else:
            s = B - 2 * sr - 1
        for j in range(s, s + 2 * sr + 1):
            if j != idx:
                cur.append(idx); oth.append(j)
    return np.asarray(cur, np.int32), np.asarray(oth, np.int32)


def owner_of(cur, K, world):
    """Contiguous keyframe ranges per rank."""
    cur = np.asarray(cur)
    bounds = [(K * r) // world for r in range(world + 1)]
    return np.searchsorted(bounds, cur, side="right") - 1


def pose_factor_active(i, j, K, world, rank):
    """The active mask of one rank's pose-factor or DD-pseudorange list: a factor belongs to the rank that owns its lower keyframe
    (owner_of's contiguous ranges).  Every rank passes the same list, so every rank gets the same pair layout."""
    lo = np.minimum(np.asarray(i), np.asarray(j))
    return (owner_of(lo, K, world) == rank).astype(np.int32)


def frames_needed(cur, oth, owned_mask):
    """Frames a rank must hold: its own cur frames plus the searched frames of its pairs (the +-2*search_range halo)."""
    return np.unique(np.concatenate([cur[owned_mask], oth[owned_mask]]))


class NcclHook:
    """ncclComm_t created through libglio_nccl.so; id exchange over an existing torch.distributed group (any backend)."""

    def __init__(self, rank, world):
        import torch
        import torch.distributed as dist
        here = os.path.dirname(os.path.abspath(__file__))
        self.lib = C.CDLL(os.path.join(here, "libglio_nccl.so"))
        nb = self.lib.glio_nccl_unique_id_bytes()
        buf = (C.c_ubyte * nb)()
        if rank == 0:
            assert self.lib.glio_nccl_get_unique_id(buf) == 0
        t = torch.tensor(list(buf), dtype=torch.uint8)
        if dist.get_backend() == "nccl":
            t = t.cuda()
        dist.broadcast(t, 0)
        ids = (C.c_ubyte * nb)(*t.cpu().tolist())
        self.comm = C.c_void_p()
        rc = self.lib.glio_nccl_comm_create(C.c_int(world), C.c_int(rank), ids, C.byref(self.comm))
        if rc != 0:
            raise RuntimeError("ncclCommInitRank failed")
        self.fn = C.cast(self.lib.glio_nccl_allreduce, C.c_void_p)

    def install(self, ctx):
        from . import api
        ctx.set_allreduce(C.cast(self.lib.glio_nccl_allreduce, api.ALLREDUCE_FN), self.comm)

    def close(self):
        if self.comm:
            self.lib.glio_nccl_comm_destroy(self.comm); self.comm = None
