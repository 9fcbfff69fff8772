"""Time sampled UniSE decoding on the GPU, shipped widths, seeded weights (the model of scripts/unise_validation_bench.py).

1. `LLM_SFT.generate` at the SR shape - B = 32 rows, prefix 252 (task, mix_sos, 250 frames of 5 s), 283 decode steps (32 global + 1 +
   250 semantic) - greedy and sampled with top_k 50 (the reference's default), 1024 (the largest top_k of the one-thread sampler)
   and 0 (no filter: every survivor of the 4096 / 8192-token range is sorted and scanned), top_p 0.95, temperature 0.8.  Reported as
   the generate time and that time over the 283 steps (prefill included); sampled minus greedy is the sampler's share.
2. The same generate with one random stream per row (`row_seeds`) against the call's stream (`seed`), at B = 32 and B = 64 (two
   chunks on lanes).
3. Sampled `enhance_batch` ('se', 'tse') with per-utterance seeds against greedy `enhance_batch`, on the utterance set of
   scripts/unise_enhance_bench.py.
Each configuration is warmed up, then timed `--reps` times with CUDA events; the best is kept.  Prints one JSON line with the card
and its power limit.  Fails without a GPU."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bicodec_global_bench import card  # noqa: E402
from scripts.unise_enhance_bench import SR, make_set  # noqa: E402
from scripts.unise_validation_bench import build_model  # noqa: E402


def best_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        ms.append(t0.elapsed_time(t1))
    return round(min(ms), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lm_sampling_bench: needs a CUDA device")
    dev = torch.device("cuda")
    model = build_model(dev)
    lm = model.dnn
    g = torch.Generator().manual_seed(7)
    frames, steps = 250, 32 + 1 + 250
    mix = torch.randn(64, frames, 768, generator=g).to(dev)           # WavLM-base-plus features of 5 s
    mel = torch.zeros(64, frames, 80, device=dev)
    gen = lambda B, **kw: lm.generate("se", None, None, mel[:B], mix[:B], **kw)
    sr = {}
    for name, kw in (("greedy", dict(do_sample=False)), ("top_k_50", dict(top_k=50, seed=1)), ("top_k_1024", dict(top_k=1024, seed=1)),
                     ("top_k_0", dict(top_k=0, seed=1))):
        ms = best_ms(lambda: gen(32, **kw), args.reps)
        sr[name] = dict(generate_ms=ms, ms_per_step=round(ms / steps, 3))
    rows = {}
    for B in (32, 64):
        seeds = list(range(1000, 1000 + B))
        rows[f"B{B}"] = dict(seed_ms=best_ms(lambda: gen(B, seed=1), args.reps),
                             row_seeds_ms=best_ms(lambda: gen(B, row_seeds=seeds), args.reps))
    srcs, enrolls = make_set(args.utterances, 2026, dev)
    audio_s = sum(s.size(-1) for s in srcs) / SR
    useeds = list(range(len(srcs)))
    enh = {}
    for mode in ("se", "tse"):
        enr = enrolls if mode == "tse" else None
        greedy = best_ms(lambda: model.enhance_batch(mode, enr, srcs), args.reps)
        sampled = best_ms(lambda: model.enhance_batch(mode, enr, srcs, do_sample=True, utterance_seeds=useeds), args.reps)
        enh[mode] = dict(greedy_ms=greedy, sampled_ms=sampled, greedy_audio_s_per_s=round(audio_s / greedy * 1e3, 1),
                         sampled_audio_s_per_s=round(audio_s / sampled * 1e3, 1))
    print(json.dumps(dict(metric="lm_sampling", sr_shape=dict(B=32, prefix=2 + frames, steps=steps, legs=sr), row_seeds=rows,
                          enhance_batch=dict(utterances=len(srcs), audio_seconds=round(audio_s, 2), legs=enh), card=card())))


if __name__ == "__main__":
    main()
