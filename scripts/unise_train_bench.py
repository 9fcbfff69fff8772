"""Time UniSE's training step on the GPU: unise.Model.training_step + loss.backward() + clip_grad_norm_(5.0) + AdamW (configure_optimizers)
over B clips of 5 s in modes 'se' and 'tse', shipped widths, seeded weights (the models of scripts/unise_validation_bench.py), attention
dropout 0.1.  After `--warmup` steps, CUDA events give:
  - ms per full step and its split: tokenize, WavLM (mix + enroll), LM forward, LM backward, optimizer (clip + AdamW + LambdaLR);
  - LM forward + backward ms and its algorithmic TFLOP/s (FLOPs counted from shapes by `lm_flops`, not measured);
  - peak device memory of a step;
  - the same LM loss and gradients from torch eager fp32 autograd of oracle/llama_train.py on the same GPU (no dropout: its mask is
    NumPy), as a yardstick.
Prints one JSON line with the card and its power limit; fails without a GPU."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bicodec_global_bench import card  # noqa: E402
from scripts.unise_validation_bench import build_model, make_batch  # noqa: E402

CONF = dict(opt=dict(lr=5e-4), sch=dict(warmup_steps=2000, step_decay=0.99998, min_factor=0.02))   # U/conf/config.yaml:108-118


def lm_flops(lm, B, L, Lt, n_feat_rows):
    """multiply-adds x 2 of the LM's forward and backward at these shapes: every GEMM three times (forward, data and weight gradient),
    causal attention as L(L+1)/2 score / value products per head forward and 2.5x that backward (P and dP recomputed, dV, dK, dQ)"""
    H, I, V, nl, heads = lm.hidden, 4 * lm.hidden, lm.vocab_size, lm.n_layers, lm.heads
    M = B * L
    gemm = nl * 2 * M * (3 * H * H + H * H + 2 * I * H + I * H) + 2 * B * Lt * V * H + 2 * n_feat_rows * lm.adapter.weight.shape[1] * H
    att = nl * B * heads * (L * (L + 1) // 2) * 64 * 2 * 2
    return dict(forward=gemm + att, backward=2 * gemm + 2.5 * att)


def eager_yardstick(lm, kw, iters):
    """torch eager fp32 autograd of the oracle on this GPU: ms for forward + backward, and the loss"""
    from oracle import llama_train
    cfg = dict(num_tasks=lm.task_embedding.weight.shape[0], task_map=lm.task_map, feats_dim=lm.adapter.weight.shape[1],
               llm_base_config=lm.cfg)
    sd = {n: p.detach().clone().requires_grad_(True) for n, p in lm.named_parameters()}
    args = (sd, cfg, kw["task_name"], kw["enroll_feats"], kw["mix_feats"], kw["global_ids"], kw["semantic_ids"])
    try:
        llama_train.sft_forward(*args)[0].backward()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            for t in sd.values():
                t.grad = None
            loss = llama_train.sft_forward(*args)[0]
            loss.backward()
        t1.record()
        torch.cuda.synchronize()
        return dict(ms=round(t0.elapsed_time(t1) / iters, 3), loss=round(float(loss), 5))
    except torch.cuda.OutOfMemoryError:
        return dict(ms=None, loss=None, note="out of memory")
    finally:
        del sd
        torch.cuda.empty_cache()


def run(model, opt, sch, mode, B, iters, warmup, dev):
    batch = make_batch(mode, B, dev)
    seen = []
    hook = model.dnn.register_forward_pre_hook(lambda mod, args, kwargs: seen.append(dict(kwargs)), with_kwargs=True)

    def step(ev=None):
        rec = (lambda i: ev[i].record()) if ev else (lambda i: None)
        mode_, enroll, mix, speech, interf = batch[:5]
        rec(0)
        g, s = model.tokenizer.tokenize(speech)
        rec(1)
        mf = model.extract_semantic_features(mix)
        ef = model.extract_semantic_features(enroll) if enroll is not None else None
        rec(2)
        model.dnn.train()
        loss, acc = model.dnn(task_name=mode_, enroll_mel=None if enroll is None else model.mel_like(enroll), enroll_feats=ef,
                              mix_mel=model.mel_like(mix), mix_feats=mf, global_ids=g.squeeze(1), semantic_ids=s)
        model.dnn.eval()
        rec(3)
        loss.backward()
        rec(4)
        torch.nn.utils.clip_grad_norm_(model.dnn.parameters(), 5.0)
        opt.step()
        sch.step()
        opt.zero_grad(set_to_none=True)
        rec(5)
        return loss

    def full():
        out = model.training_step(batch)
        out["loss"].backward()
        torch.nn.utils.clip_grad_norm_(model.dnn.parameters(), 5.0)
        opt.step()
        sch.step()
        opt.zero_grad(set_to_none=True)
        return out

    for _ in range(warmup):
        full()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    out = full()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    hook.remove()
    kw = seen[-1]
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        full()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    split = [0.0] * 5
    for _ in range(iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        step(ev)
        torch.cuda.synchronize()
        for i in range(5):
            split[i] += ev[i].elapsed_time(ev[i + 1]) / iters
    lm = model.dnn
    Lt = kw["semantic_ids"].shape[1] + 34
    Te = 0 if kw["enroll_feats"] is None else kw["enroll_feats"].shape[1]
    Tm = kw["mix_feats"].shape[1]
    L = Lt + 2 + Tm + (1 + Te if Te else 0)
    fl = lm_flops(lm, B, L, Lt, B * (Tm + Te))
    lm_ms = split[2] + split[3]
    eager = eager_yardstick(lm, kw, max(1, iters // 2))
    return dict(mode=mode, batch=B, L=L, ms_per_step=round(ms, 3), clips_per_s=round(B / ms * 1e3, 2),
                stage_ms=dict(tokenize=round(split[0], 3), wavlm=round(split[1], 3), lm_forward=round(split[2], 3),
                              lm_backward=round(split[3], 3), optimizer=round(split[4], 3)),
                lm_fwd_bwd_ms=round(lm_ms, 3), lm_algorithmic_tflops=round((fl["forward"] + fl["backward"]) / lm_ms / 1e9, 2),
                peak_memory_gb=round(peak / 2 ** 30, 2), train_loss=round(float(out["loss"]), 5), eager_fp32_autograd=eager)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--modes", nargs="+", default=["se", "tse"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unise_train_bench: needs a CUDA device")
    dev = torch.device("cuda")
    model = build_model(dev)
    model.config = dict(CONF)
    [opt], [sch] = model.configure_optimizers()
    legs = [run(model, opt, sch["scheduler"], mode, args.batch, args.iters, args.warmup, dev) for mode in args.modes]
    print(json.dumps(dict(metric="unise_training_step", seconds_per_clip=5.0, dropout_p=model.dnn.cfg.get("dropout_p", 0.1), legs=legs,
                          card=card())))


if __name__ == "__main__":
    main()
