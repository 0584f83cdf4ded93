"""torch.distributed plumbing for cell-sharded runs (one process per GPU, SURVEY section 8e).

Every collective on the hot path is a sum-allreduce of a small replicated object (column
sums [D], A_r^T Y_r [D x l], Gram [l x l], z-score moments [2k]).  With no process group
(single GPU) these are no-ops.
"""
from __future__ import annotations

import torch


def is_distributed() -> bool:
    return torch.distributed.is_available() and torch.distributed.is_initialized() \
        and torch.distributed.get_world_size() > 1


def world_size() -> int:
    return torch.distributed.get_world_size() if is_distributed() else 1


def rank() -> int:
    return torch.distributed.get_rank() if is_distributed() else 0


def all_reduce_sum_(t: torch.Tensor) -> torch.Tensor:
    if is_distributed():
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.SUM)
    return t


def all_reduce_max_(t: torch.Tensor) -> torch.Tensor:
    if is_distributed():
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
    return t


def broadcast_(t: torch.Tensor, src: int = 0) -> torch.Tensor:
    """Make a replicated tensor bit-identical on every rank (guards the replicated d-space basis
    against per-process differences in library kernels)."""
    if is_distributed():
        torch.distributed.broadcast(t, src=src)
    return t


def balanced_row_range(indptr, world: int = None, rank_: int = None):
    """Contiguous row block [r0, r1) of rank ``rank_`` of ``world`` such that every rank holds about the same number of
    stored entries (SURVEY section 8e: "row blocks balanced by nnz, not by row count"; cells differ in depth).
    ``indptr``: CSR row pointer of the WHOLE matrix (numpy array or tensor).  Defaults: the current process group."""
    import numpy as np
    world = world_size() if world is None else int(world)
    rank_ = rank() if rank_ is None else int(rank_)
    ip = indptr.cpu().numpy() if isinstance(indptr, torch.Tensor) else np.asarray(indptr)
    n = ip.shape[0] - 1
    nnz = int(ip[-1]) - int(ip[0])
    cuts = [0] + [int(np.searchsorted(ip, int(ip[0]) + (nnz * i) // world, side="left")) for i in range(1, world)] + [n]
    for i in range(1, len(cuts)):
        cuts[i] = min(n, max(cuts[i], cuts[i - 1]))
    return cuts[rank_], cuts[rank_ + 1]
