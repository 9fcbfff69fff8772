"""parallel.average_gradients and parallel.broadcast_parameters on gloo (CPU), pinned against torch's own
DistributedDataParallel(find_unused_parameters=True) at world 2 and 3; world 1 and an uninitialised process group are no-ops."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp
from torch import nn


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


class Toy(nn.Module):
    """`shared` is used on every rank, `first` on rank 0 only, `some` on the odd ranks, `unused` never"""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.shared = nn.Linear(4, 3)
        with torch.no_grad():
            self.shared.weight.copy_(torch.randn(3, 4, generator=g))
            self.shared.bias.copy_(torch.randn(3, generator=g))
        self.some = nn.Parameter(torch.randn(3, generator=g))
        self.unused = nn.Parameter(torch.randn(3, generator=g))
        self.first = nn.Parameter(torch.randn(3, generator=g))

    def forward(self, x, rank: int):
        y = self.shared(x)
        if rank == 0:
            y = y + self.first
        if rank % 2 == 1:
            y = y * self.some
        return (y.tanh() * torch.linspace(-1, 2, 3)).sum()


def _step(model, rank):
    """one rank's backward on its own inputs, with leftover gradients from an earlier, un-zeroed backward on `some` at rank 0
    (where this backward does not use it) and on `shared.bias` at rank 1"""
    g = torch.Generator().manual_seed(100 + rank)
    x = torch.randn(5, 4, generator=g)
    inner = getattr(model, "module", model)
    if rank == 0:
        inner.some.grad = torch.randn(3, generator=g)
    if rank == 1:
        inner.shared.bias.grad = torch.randn(3, generator=g)
    model(x, rank=rank).backward()


def _grads(module):
    return {n: (None if p.grad is None else p.grad.clone()) for n, p in module.named_parameters()}


def _worker(rank, world, port, ret):
    import torch.distributed as dist
    from unified_audio_b200.parallel import average_gradients, broadcast_parameters
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    errors = []
    # DDP's reducer and ours, from the same weights and the same per-rank backward
    ddp = nn.parallel.DistributedDataParallel(Toy(), find_unused_parameters=True)
    _step(ddp, rank)
    want = _grads(ddp.module)
    ours = Toy()
    _step(ours, rank)
    average_gradients(ours)
    got = _grads(ours)
    for n in want:
        if (want[n] is None) != (got[n] is None):
            errors.append(f"{n}: DDP grad is {'None' if want[n] is None else 'set'}, ours is {'None' if got[n] is None else 'set'}")
        elif want[n] is not None:
            # world 2: 0.5 g0 + 0.5 g1 is one rounding whatever the order, so bit for bit.  World 3: gloo sums three terms in an
            # order that depends on where the value sits in the buffer, and DDP's buffer is laid out differently: fp32
            # summation-order differences only.
            same = torch.equal(got[n], want[n]) if world == 2 else torch.allclose(got[n], want[n], rtol=1e-6, atol=1e-7)
            if not same:
                errors.append(f"{n}: {got[n].tolist()} vs DDP {want[n].tolist()}")
    if want["unused"] is not None or want["first"] is None or want["some"] is None:
        errors.append("the case does not exercise a parameter unused everywhere and ones used on some ranks")
    # every rank holds the same average: rank 0's, broadcast (one broadcast per parameter on every rank, whatever it holds)
    for n, p in ours.named_parameters():
        t = torch.cat([torch.tensor([float(got[n] is None)]), torch.zeros(p.numel()) if got[n] is None else got[n].reshape(-1)])
        r0 = t.clone()
        dist.broadcast(r0, 0)
        if not torch.equal(r0, t):
            errors.append(f"{n}: differs from rank 0's")
    # broadcast_parameters from rank src: every rank ends with src's values, and every version counter moves
    for src in (0, world - 1):
        m = Toy()
        with torch.no_grad():
            for p in m.parameters():
                p.add_(rank)
        versions = [p._version for p in m.parameters()]
        broadcast_parameters(m, src=src)
        want = {n: p.detach() + src for n, p in Toy().named_parameters()}
        for (n, p), v in zip(m.named_parameters(), versions):
            if not torch.equal(p.detach(), want[n]):
                errors.append(f"broadcast from {src}: {n} differs from rank {src}'s")
            if p._version == v:
                errors.append(f"broadcast from {src}: {n}'s version counter did not move")
    ret[rank] = errors
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_average_gradients_matches_ddp_gloo(world):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert all(ret[r] == [] for r in range(world)), dict(ret)


def _noop_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ret[rank] = _noop_errors()
    dist.destroy_process_group()


def _noop_errors():
    """average_gradients and broadcast_parameters leave the same tensors with the same bits and the same version counters"""
    from unified_audio_b200.parallel import average_gradients, broadcast_parameters
    m = Toy()
    _step(m, 1)
    before = {n: (p.grad, None if p.grad is None else p.grad.clone(), p.detach().clone(), p._version) for n, p in m.named_parameters()}
    average_gradients(m)
    broadcast_parameters(m)
    errors = []
    for n, p in m.named_parameters():
        grad, bits, value, version = before[n]
        if p.grad is not grad or (grad is not None and not torch.equal(p.grad, bits)):
            errors.append(f"{n}: .grad changed")
        if not torch.equal(p.detach(), value) or p._version != version:
            errors.append(f"{n}: parameter changed")
    return errors


def test_world1_and_uninitialised_are_noops():
    import torch.distributed as dist
    assert not dist.is_initialized()
    assert _noop_errors() == []
    ret = mp.Manager().dict()
    mp.spawn(_noop_worker, args=(1, _free_port(), ret), nprocs=1, join=True)
    assert ret[0] == []
