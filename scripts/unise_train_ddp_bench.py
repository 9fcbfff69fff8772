"""Time data-parallel UniSE training: one rank per GPU, each running training_step + loss.backward() + Model.sync_gradients +
clip_grad_norm_(5.0) + AdamW + LambdaLR on B clips of 5 s (modes 'se' and 'tse', shipped widths, seeded weights: the models of
scripts/unise_validation_bench.py; every rank tokenizes the same seeded batch, which does not change the timing).

    torchrun --nproc_per_node=<GPUs> scripts/unise_train_ddp_bench.py [--batch 32 --iters 10 --warmup 3]

Without torchrun it runs as one rank.  Per mode, CUDA events give, as the median over the timed steps (and the largest of the
ranks' medians):
  - `step_ms`: the full step at this world size;
  - `sync_ms`: `sync_gradients` alone (a no-op at world 1);
  - `pack_unpack_ms`: the device work `sync_gradients` does besides the all-reduce (flatten + scale into one fp32 buffer, copy
    back), timed on rank 0 outside the step;
  - `world1_step_ms`: the same step on rank 0 alone (a one-rank group, so no collective) while the other ranks wait;
  - clips/s overall (world x B / step_ms) and the scaling efficiency world1_step_ms / step_ms.
Rank 0 prints one JSON line with the card and its power limit; fails without a GPU."""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bicodec_global_bench import card  # noqa: E402
from scripts.unise_train_bench import CONF  # noqa: E402
from scripts.unise_validation_bench import build_model, make_batch  # noqa: E402


def timed_steps(model, opt, sch, batch, iters, warmup, group):
    """median full-step ms and median sync_gradients ms over `iters` steps after `warmup`"""
    step_ms, sync_ms = [], []
    for i in range(warmup + iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        opt.zero_grad(set_to_none=True)
        model.training_step(batch)["loss"].backward()
        ev[1].record()
        model.sync_gradients(group)
        ev[2].record()
        torch.nn.utils.clip_grad_norm_(model.dnn.parameters(), 5.0)
        opt.step()
        sch.step()
        ev[3].record()
        torch.cuda.synchronize()
        if i >= warmup:
            step_ms.append(ev[0].elapsed_time(ev[3]))
            sync_ms.append(ev[1].elapsed_time(ev[2]))
    return statistics.median(step_ms), statistics.median(sync_ms)


def pack_unpack_ms(model, iters):
    """the flatten + scale + copy-back of average_gradients on this rank's gradients, without the collective"""
    from unified_audio_b200.parallel import _flat_parameters, _pack_gradients, _unpack_gradients
    params = _flat_parameters(model.dnn, "pack_unpack_ms", trained_only=True)
    out = []
    for _ in range(iters + 1):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        _unpack_gradients(params, _pack_gradients(params, 2))
        t1.record()
        torch.cuda.synchronize()
        out.append(t0.elapsed_time(t1))
    return statistics.median(out[1:]), sum(p.numel() for p in params)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--modes", nargs="+", default=["se", "tse"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unise_train_ddp_bench: needs a CUDA device")
    distributed = "WORLD_SIZE" in os.environ
    rank = int(os.environ.get("RANK", 0))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if distributed:
        dist.init_process_group("nccl", device_id=dev)
    world = dist.get_world_size() if distributed else 1
    alone = dist.new_group([0]) if distributed else None          # rank 0 by itself: the world-1 step
    model = build_model(dev)
    model.config = dict(CONF)
    [opt], [sch] = model.configure_optimizers()
    model.broadcast_parameters()
    legs = []
    for mode in args.modes:
        batch = make_batch(mode, args.batch, dev)
        ms, sync = timed_steps(model, opt, sch["scheduler"], batch, args.iters, args.warmup, None)
        mine = torch.tensor([ms, sync], dtype=torch.float64, device=dev)
        per_rank = [mine.clone() for _ in range(world)]
        if distributed:
            dist.all_gather(per_rank, mine)
        per_rank = [t.tolist() for t in per_rank]
        if rank == 0:
            ms1 = ms if world == 1 else timed_steps(model, opt, sch["scheduler"], batch, args.iters, args.warmup, alone)[0]
            pu, n = pack_unpack_ms(model, args.iters)
        if distributed:
            dist.barrier()
        if rank == 0:
            step = max(r[0] for r in per_rank)
            legs.append(dict(mode=mode, batch_per_rank=args.batch, world=world, step_ms=round(step, 3),
                             step_ms_per_rank=[round(r[0], 3) for r in per_rank], sync_ms=round(max(r[1] for r in per_rank), 3),
                             sync_share_of_step=round(max(r[1] for r in per_rank) / step, 5), pack_unpack_ms=round(pu, 3),
                             gradient_mb=round(4 * n / 1e6, 1), world1_step_ms=round(ms1, 3),
                             clips_per_s=round(world * args.batch / step * 1e3, 2), scaling_efficiency=round(ms1 / step, 4)))
    if rank == 0:
        print(json.dumps(dict(metric="unise_ddp_training_step", seconds_per_clip=5.0, world=world, legs=legs, card=card())))
    if distributed:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
