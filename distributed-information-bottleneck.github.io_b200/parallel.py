"""Data-parallel plumbing: one process per GPU, ``torch.distributed`` (NCCL over NVLink/NVSwitch) for the single
exchange step of the path -- a sum all-reduce of the flat [gradients || statistics] buffer between backward and
Adam.  The reference has no multi-GPU code (SURVEY.md section 8e); samples are independent units, every loss term is
a batch mean (models.py:111-112), so each global batch splits into contiguous row ranges per rank."""
from __future__ import annotations

import torch
import torch.distributed as dist


def world_and_rank(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def shard_range(n, rank, world):
    """Rows [lo, hi) of an n-row global batch owned by ``rank``: contiguous, sizes differ by at most one,
    earlier ranks take the remainder.  Covers [0, n) exactly once over all ranks."""
    base, rem = divmod(int(n), int(world))
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


def all_gather_rows_(buf: torch.Tensor, group=None):
    """In-place all-gather of a rank-contiguous buffer: ``buf`` holds world equal row blocks, rank r has filled block r, and
    afterwards every rank holds all of them.  No-op for a single process."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return buf
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if buf.shape[0] % world:
        raise ValueError(f"all_gather_rows_: {buf.shape[0]} rows do not split into {world} equal blocks")
    blocks = list(buf.chunk(world))
    if dist.get_backend(group) == "nccl":
        dist.all_gather_into_tensor(buf, blocks[rank], group=group)
    else:                                    # gloo: list all-gather; the own block goes in as a copy
        dist.all_gather(blocks, blocks[rank].clone(), group=group)
    return buf


def allreduce_sum_(flat: torch.Tensor, group=None):
    """In-place sum over the data-parallel group on the current stream; no-op for a single process."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    return flat
