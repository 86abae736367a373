"""The all-reduce hook of the sharded batch workers (tests/workers/*_shard_worker.py): a ctypes callback that stages the device
buffer through the host and sums it with torch.distributed (gloo), so that ranks may share one GPU - the C-ABI contract of
glio_allreduce_fn, with any transport underneath (libglio_nccl.so is the NCCL one; two NCCL ranks cannot share a device, so the
single-GPU test box uses this one)."""
import ctypes as C

import numpy as np


def staging_allreduce():
    """(callback, calls, counts): the api.ALLREDUCE_FN to hand to Context.set_allreduce, a one-element list with the number of
    calls that succeeded, and the element count of each of them"""
    import torch
    import torch.distributed as dist
    from glio_b200 import api
    cudart = C.CDLL("libcudart.so")
    calls, counts = [0], []

    def hook(user, d_buf, count, stream):
        try:
            n = int(count)
            h = np.empty(n, np.float64)
            # everything on the library's own (non-blocking) stream: a copy on the NULL stream would not be ordered with it
            s = C.c_void_p(stream)
            assert cudart.cudaMemcpyAsync(h.ctypes.data_as(C.c_void_p), C.c_void_p(d_buf), C.c_size_t(8 * n), C.c_int(2), s) == 0
            assert cudart.cudaStreamSynchronize(s) == 0
            t = torch.from_numpy(h)
            dist.all_reduce(t)
            assert cudart.cudaMemcpyAsync(C.c_void_p(d_buf), h.ctypes.data_as(C.c_void_p), C.c_size_t(8 * n), C.c_int(1), s) == 0
            assert cudart.cudaStreamSynchronize(s) == 0
            calls[0] += 1; counts.append(n)
            return 0
        except Exception:
            return -1
    return api.ALLREDUCE_FN(hook), calls, counts
