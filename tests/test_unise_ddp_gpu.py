"""Data-parallel UniSE training on the GPU: unise.Model.broadcast_parameters / sync_gradients across two processes, against the same
steps emulated in one process.

Two ranks share the one H100 through gloo on CUDA tensors (NCCL refuses two ranks on one device); with two or more GPUs visible the
mixed-mode case runs again over NCCL, one rank per GPU.  Reduced widths (tests/test_unise_validation_gpu.build_small), B = 4 per rank,
a fixed dropout seed per rank and step.  The backward is deterministic, so 0.5 g0 + 0.5 g1 computed in one process from the same two
backward passes is what the all-reduce must give, bit for bit (two fp32 terms: one rounding, whatever the order)."""
import os
import socket
from datetime import timedelta

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

B = 4
CONF = dict(opt=dict(lr=1e-3), sch=dict(warmup_steps=0, step_decay=0.9, min_factor=0.02))    # lr > 0 from the first step
MIXED = ("se", "tse")                         # rank 0's mode, rank 1's mode
STEPS = [("se", "tse"), ("tse", "tse"), ("se", "se")]
ENROLL_SOS = "enroll_sos_embedding.weight"


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def fresh_model():
    from test_unise_validation_gpu import build_small
    model = build_small()[0]
    model.config = dict(CONF)
    return model


def batch_for(mode, seed):
    from test_unise_validation_gpu import small_batch, to_cuda
    wav = 0.1 * torch.randn(B, 6400, generator=torch.Generator().manual_seed(seed))
    return to_cuda(small_batch(mode, wav, seed))


def seed_of(case, step, rank):
    return 1000 * case + 10 * step + rank


def backward(model, mode, seed):
    """one rank's training_step + backward from zeroed gradients"""
    model.dnn.zero_grad(set_to_none=True)
    model.training_step(batch_for(mode, seed), dropout_seed=seed + 7)["loss"].backward()


def grads(model):
    return {n: None if p.grad is None else p.grad.detach().cpu().clone() for n, p in model.dnn.named_parameters()}


def params(model):
    return {n: p.detach().cpu().clone() for n, p in model.dnn.named_parameters()}


def optimizer_step(model, opt, sch):
    torch.nn.utils.clip_grad_norm_(model.dnn.parameters(), 5.0)
    opt.step()
    sch["scheduler"].step()


def _worker(rank, world, port, backend, cases, out):
    import torch.distributed as dist
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=timedelta(minutes=5))
    res = {}
    # broadcast: rank 1 starts from other weights, packs them for the inference path, then receives rank 0's
    model = fresh_model()
    probe = batch_for("tse", 1)
    if rank:
        with torch.no_grad():
            for p in model.dnn.parameters():
                p.mul_(1.25)
    before = float(model.validation_step(probe)["valid_loss"])
    model.broadcast_parameters()
    res["broadcast"] = dict(before=before, after=float(model.validation_step(probe)["valid_loss"]), params=params(model))
    # mixed modes: rank 0 'se', rank 1 'tse'
    model.configure_optimizers()
    backward(model, MIXED[rank], seed_of(1, 0, rank))
    res["mixed_local"] = grads(model)
    model.sync_gradients()
    res["mixed"] = grads(model)
    if "all_se" in cases:
        model = fresh_model()
        [opt], [sch] = model.configure_optimizers()
        backward(model, "se", seed_of(2, 0, rank))
        model.sync_gradients()
        res["all_se"] = grads(model)
        optimizer_step(model, opt, sch)
        sos = dict(model.dnn.named_parameters())[ENROLL_SOS]
        res["all_se_params"], res["all_se_sos_state"] = params(model), len(opt.state[sos])
    if "steps" in cases:
        model = fresh_model()
        [opt], [sch] = model.configure_optimizers()
        res["steps"] = []
        for step, modes in enumerate(STEPS):
            opt.zero_grad(set_to_none=True)
            model.training_step(batch_for(modes[rank], seed_of(3, step, rank)), dropout_seed=seed_of(3, step, rank) + 7)["loss"].backward()
            model.sync_gradients()
            optimizer_step(model, opt, sch)
            res["steps"].append(params(model))
    torch.save(res, os.path.join(out, f"rank{rank}.pt"))
    dist.destroy_process_group()


def run_ranks(backend, cases, out):
    mp.spawn(_worker, args=(2, _free_port(), backend, cases, str(out)), nprocs=2, join=True)
    return [torch.load(os.path.join(str(out), f"rank{r}.pt")) for r in range(2)]


def averaged(g0, g1):
    """0.5 g0 + 0.5 g1 per parameter; a None side contributes zero, and None on both sides stays None"""
    out = {}
    for n in g0:
        a, b = g0[n], g1[n]
        out[n] = None if a is None and b is None else (0.5 * a if b is None else 0.5 * b if a is None else 0.5 * a + 0.5 * b)
    return out


def assert_same(got, want, what):
    for n in want:
        assert (got[n] is None) == (want[n] is None), (what, n, got[n] is None)
        assert got[n] is None or torch.equal(got[n], want[n]), (what, n, float((got[n] - want[n]).abs().max()))


@pytest.fixture(scope="module")
def gloo_ranks(lib, tmp_path_factory):
    return run_ranks("gloo", ("all_se", "steps"), tmp_path_factory.mktemp("ddp_gloo"))


def check_mixed(ranks):
    model = fresh_model()
    model.configure_optimizers()
    local = []
    for rank, mode in enumerate(MIXED):
        backward(model, mode, seed_of(1, 0, rank))
        local.append(grads(model))
    assert local[0][ENROLL_SOS] is None and local[1][ENROLL_SOS] is not None
    for rank in range(2):                           # the backward passes the ranks ran are the ones emulated here
        assert_same(ranks[rank]["mixed_local"], local[rank], f"rank {rank}'s own backward")
    want = averaged(*local)
    for rank in range(2):
        assert_same(ranks[rank]["mixed"], want, f"rank {rank} after sync_gradients")
        assert torch.equal(ranks[rank]["mixed"][ENROLL_SOS], local[1][ENROLL_SOS] / 2)


def test_broadcast_parameters_repacks(gloo_ranks):
    model = fresh_model()
    want = float(model.validation_step(batch_for("tse", 1))["valid_loss"])
    assert gloo_ranks[1]["broadcast"]["before"] != want                 # rank 1 packed other weights first
    for rank in range(2):
        assert_same(gloo_ranks[rank]["broadcast"]["params"], params(model), f"rank {rank} after broadcast_parameters")
        assert gloo_ranks[rank]["broadcast"]["after"] == want


def test_sync_gradients_mixed_modes(gloo_ranks):
    check_mixed(gloo_ranks)


def test_sync_gradients_all_se_skips_enroll_sos(gloo_ranks):
    model = fresh_model()
    start = params(model)
    for rank in range(2):
        assert gloo_ranks[rank]["all_se"][ENROLL_SOS] is None
        assert gloo_ranks[rank]["all_se_sos_state"] == 0                  # AdamW kept no moments for it
        after = gloo_ranks[rank]["all_se_params"]
        assert torch.equal(after[ENROLL_SOS], start[ENROLL_SOS])        # no weight decay either
        assert not torch.equal(after["mix_sos_embedding.weight"], start["mix_sos_embedding.weight"])
    assert_same(gloo_ranks[0]["all_se_params"], gloo_ranks[1]["all_se_params"], "ranks after the all-'se' step")


def test_three_steps_match_single_process_emulation(gloo_ranks):
    model = fresh_model()
    [opt], [sch] = model.configure_optimizers()
    for step, modes in enumerate(STEPS):
        local = []
        for rank, mode in enumerate(modes):
            backward(model, mode, seed_of(3, step, rank))
            local.append(grads(model))
        avg = averaged(*local)
        for n, p in model.dnn.named_parameters():
            p.grad = None if avg[n] is None else avg[n].cuda()
        optimizer_step(model, opt, sch)
        want = params(model)
        for rank in range(2):
            assert_same(gloo_ranks[rank]["steps"][step], want, f"rank {rank} after step {step}")


def test_sync_gradients_mixed_modes_nccl(lib, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip(f"NCCL needs one GPU per rank: {torch.cuda.device_count()} visible")
    check_mixed(run_ranks("nccl", (), tmp_path))
