"""Multi-GPU plumbing of the hot path (SURVEY.md 8e): clips are independent, so ranks own contiguous batch
shards with replicated weights and NO data-path collective; the single exchange step is one all-gather of the
int64 token tensors.  A validation epoch ends with one all-reduce of its running sums.  Works with backend
"nccl" (GPU) and "gloo" (CPU tests)."""
from __future__ import annotations

from typing import Optional, Tuple

import torch


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) slice of `n_items` clips owned by `rank` (first `n % world` ranks get one extra)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def all_reduce_sum(t: torch.Tensor, group=None) -> torch.Tensor:
    """Sum `t` over the ranks of `group` in place with one `all_reduce` and return it; unchanged when torch.distributed is not
    initialised.  `unise.Model.validation_epoch` sums its fp64 [Σ B·loss, Σ B·acc, Σ B] with it."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def gather_tokens(tokens: torch.Tensor, n_total: int, group=None, buffers: Optional[dict] = None) -> torch.Tensor:
    """All-gather int64 tokens [b_local, ...] from every rank into [n_total, ...] - the path's single exchange step.

    Equal shards (n_total % world == 0, the benchmarked case): ONE `all_gather_into_tensor` straight into a preallocated
    [n_total, ...] buffer - no padding, no list of per-rank tensors, no concatenation, nothing allocated per call when
    `buffers` (a dict the caller keeps) is given; the call is a single NCCL kernel and can sit inside a captured CUDA graph.
    Ragged shards: padded gather + trim (host-side glue, tests only)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return tokens
    world = dist.get_world_size(group)
    tokens = tokens.contiguous()
    if n_total % world == 0 and tokens.shape[0] * world == n_total:
        key = ("gather", tuple(tokens.shape), tokens.dtype, str(tokens.device), n_total)
        out = buffers.get(key) if buffers is not None else None
        if out is None:
            out = torch.empty((n_total,) + tuple(tokens.shape[1:]), dtype=tokens.dtype, device=tokens.device)
            if buffers is not None:
                buffers[key] = out
        dist.all_gather_into_tensor(out, tokens, group=group)
        return out
    b_max = (n_total + world - 1) // world
    pad = torch.zeros((b_max,) + tuple(tokens.shape[1:]), dtype=tokens.dtype, device=tokens.device)
    pad[: tokens.shape[0]] = tokens
    out = torch.empty((world * b_max,) + tuple(tokens.shape[1:]), dtype=tokens.dtype, device=tokens.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    parts = []
    for r in range(world):
        lo, hi = shard_range(n_total, r, world)
        parts.append(out[r * b_max: r * b_max + hi - lo])
    return torch.cat(parts, 0)
