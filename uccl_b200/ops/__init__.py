"""Functional collective ops on a process-wide default communicator (the `ncclXxx(comm, ...)`
style without carrying the handle around):

    import uccl_b200.ops as ops
    ops.init(heap_bytes=4 << 30)            # once per process, after torch.distributed init
    ops.all_reduce(t, "avg"); ops.all_gather(out, t); ops.reduce_scatter(out, t) ...
"""
from __future__ import annotations

from typing import Optional

import torch

from ..parallel.comm import Communicator

_default: Optional[Communicator] = None


def init(comm: Optional[Communicator] = None, **kw) -> Communicator:
    global _default
    _default = comm if comm is not None else Communicator.from_torch_dist(**kw)
    return _default


def default() -> Communicator:
    if _default is None:
        raise RuntimeError("uccl_b200.ops: call ops.init() first")
    return _default


def empty(*shape, dtype=torch.float32):
    return default().empty(*shape, dtype=dtype)


def all_reduce(tensor, op="sum", out=None, **kw):
    return default().all_reduce(tensor, op, out, **kw)


def all_reduce_rmsnorm(x, residual, weight, eps=1e-6, **kw):
    return default().all_reduce_rmsnorm(x, residual, weight, eps, **kw)


def reduce_scatter_rmsnorm(x, residual, weight, eps=1e-6, **kw):
    return default().reduce_scatter_rmsnorm(x, residual, weight, eps, **kw)


def all_gather(out, tensor):
    return default().all_gather(out, tensor)


def reduce_scatter(out, tensor, op="sum"):
    return default().reduce_scatter(out, tensor, op)


def broadcast(tensor, root=0):
    return default().broadcast(tensor, root)


def reduce(tensor, root=0, op="sum"):
    return default().reduce(tensor, root, op)


def all_to_all(out, tensor):
    return default().all_to_all(out, tensor)


def all_to_all_v(out, tensor, send_counts, recv_counts, send_displs=None, recv_displs=None):
    return default().all_to_all_v(out, tensor, send_counts, recv_counts, send_displs, recv_displs)


def send(tensor, dst):
    return default().send(tensor, dst)


def recv(tensor, src):
    return default().recv(tensor, src)


def batch_send_recv(ops):
    return default().batch_send_recv(ops)


def barrier():
    return default().barrier()
