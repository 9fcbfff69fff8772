"""Multi-GPU plumbing of the hot path (SURVEY.md 8e): clips are independent, so ranks own contiguous batch
shards with replicated weights and NO data-path collective; the single exchange step is one all-gather of the
int64 token tensors.  A validation epoch ends with one all-reduce of its running sums; a data-parallel training
step with one all-reduce of the LM's gradients (`average_gradients`), after the ranks started from one set of
weights (`broadcast_parameters`).  Works with backend "nccl" (GPU) and "gloo" (CPU tests)."""
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


def _world(group) -> int:
    """the size of `group`, or 1 when torch.distributed is not initialised"""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return 1
    return dist.get_world_size(group)


def _flat_parameters(module: torch.nn.Module, what: str, trained_only: bool):
    """the parameters of `module` (those that require grad when `trained_only`), all dense fp32 on one device: what one fp32
    buffer can carry"""
    params = [p for p in module.parameters() if p.requires_grad or not trained_only]
    for p in params:
        if p.dtype != torch.float32 or p.layout != torch.strided or p.device != params[0].device:
            raise TypeError(f"{what}: every parameter must be a dense fp32 tensor on {params[0].device}, got {p.dtype} {p.layout} "
                            f"on {p.device}")
    return params


def broadcast_parameters(module: torch.nn.Module, group=None, src: int = 0) -> None:
    """Copy rank `src`'s parameters into every rank's, in place, as DistributedDataParallel does when it is constructed: one
    broadcast of a flat fp32 buffer, then `copy_` into each parameter.  The copy moves every parameter's version counter (on `src`
    too), so a face that packs its weights (`LLM_SFT`) repacks them at its next call.  No-op when torch.distributed is not
    initialised or the group has one rank.  `src` is a global rank."""
    import torch.distributed as dist
    if _world(group) == 1:
        return
    params = _flat_parameters(module, "broadcast_parameters", trained_only=False)
    if not params:
        return
    flat = torch.cat([p.detach().reshape(-1) for p in params])
    dist.broadcast(flat, src=src, group=group)
    with torch.no_grad():
        for p, v in zip(params, flat.split([p.numel() for p in params])):
            p.copy_(v.view_as(p))


def average_gradients(module: torch.nn.Module, group=None) -> None:
    """Average the `.grad` of `module`'s parameters across the ranks of `group`, leaving in `.grad` what
    DistributedDataParallel(module, find_unused_parameters=True) and its default all-reduce leave there.  Call it after
    `loss.backward()` and before clipping.

    Each rank multiplies its fp32 gradients by 1 / world (as DDP's reducer does while it fills a bucket) and the ranks sum them.  A
    parameter whose `.grad` is None on this rank contributes zeros.  A parameter with a gradient on at least one rank gets the
    average on every rank; where it was None locally it gets a new tensor.  A parameter with no gradient on any rank keeps `.grad
    is None` everywhere, so the optimizer skips it (AdamW: no weight decay, no moment update), as DDP leaves it.  A gradient left
    over from an earlier, un-zeroed backward is averaged like a fresh one, as DDP averages it.  `.grad` cannot tell a leftover from a
    fresh gradient, so one case differs from DDP: a parameter that no rank used in this backward but that holds a leftover `.grad` on
    some rank.  DDP leaves each rank's leftover as it is; this averages them.

    One collective per call: the flattened gradients and one "has a gradient" count per parameter go into a single fp32 buffer,
    all-reduced once, and are copied back.  No gradient value is read on the host.  The counts are read on the host (one small
    device-to-host copy after the all-reduce) only when a parameter has no gradient on this rank, to decide which of them get one.
    No-op when torch.distributed is not initialised or the group has one rank."""
    import torch.distributed as dist
    world = _world(group)
    if world == 1:
        return
    params = _flat_parameters(module, "average_gradients", trained_only=True)
    if not params:
        return
    flat = _pack_gradients(params, world)
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    _unpack_gradients(params, flat)


def _pack_gradients(params, world: int) -> torch.Tensor:
    """[every gradient flattened and multiplied by 1 / world (zeros for a None), then one has-a-gradient flag per parameter]"""
    grads = [p.grad for p in params]
    for g in grads:
        if g is not None and (g.dtype != torch.float32 or g.layout != torch.strided):
            raise TypeError(f"average_gradients: gradients must be dense fp32, got {g.dtype} {g.layout}")
    total = sum(p.numel() for p in params)
    has = torch.tensor([0.0 if g is None else 1.0 for g in grads], dtype=torch.float32).to(params[0].device)
    flat = torch.cat([g.reshape(-1) if g is not None else p.new_zeros(p.numel()) for p, g in zip(params, grads)] + [has])
    flat[:total].mul_(1.0 / world)
    return flat


def _unpack_gradients(params, flat: torch.Tensor) -> None:
    """copy the summed buffer back into `.grad`; a None `.grad` gets a tensor when some rank had a gradient"""
    sizes = [p.numel() for p in params]
    total = sum(sizes)
    counts = flat[total:].tolist() if any(p.grad is None for p in params) else None     # the only host read, and only when needed
    with torch.no_grad():
        for i, (p, v) in enumerate(zip(params, flat[:total].split(sizes))):
            if p.grad is not None:
                p.grad.copy_(v.view_as(p.grad))
            elif counts[i] > 0:
                p.grad = v.view_as(p).clone()
