"""Time UniSE inference over a test set on the GPU: `enhance` once per utterance (what `test_step` does for the reference's loader,
one utterance per batch) against `enhance_batch` over the whole set, modes 'se' and 'tse', shipped widths, seeded weights (the model of
scripts/unise_validation_bench.py).  The set: `--utterances` seeded utterances of 2-15 s and, for 'tse', enrollments of 2-8 s.

After a warm-up of both paths, the two are timed alternately, twice each, with CUDA events around each pass over the set.  Prints
one JSON line per run: utterances/s and audio-seconds/s of each path (the better of its two passes) and the speed-up, the peak
device memory of each path, the library's kernel-launch count of one pass, the card and its power limit, and whether both paths'
outputs on the timed inputs are identical (per utterance).  Fails without a GPU."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bicodec_global_bench import card  # noqa: E402
from scripts.unise_validation_bench import build_model  # noqa: E402

SR = 16000


def make_set(n, seed, dev):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(2 * SR, 15 * SR + 1, (n,), generator=g).tolist()
    elens = torch.randint(2 * SR, 8 * SR + 1, (n,), generator=g).tolist()
    srcs = [(0.1 * torch.randn(1, t, generator=g)).to(dev) for t in lens]
    enrolls = [(0.1 * torch.randn(1, t, generator=g)).to(dev) for t in elens]
    return srcs, enrolls


def run(model, mode, srcs, enrolls, max_segments):
    from unified_audio_b200 import ops
    enr = enrolls if mode == "tse" else [None] * len(srcs)
    loop = lambda: [model.enhance(mode, e, s) for s, e in zip(srcs, enr)]
    batch = lambda: model.enhance_batch(mode, enrolls if mode == "tse" else None, srcs, max_segments=max_segments)
    loop(), batch()                                                   # warm-up: captured graphs, workspaces
    torch.cuda.synchronize()
    ms = {"loop": [], "batch": []}
    peak, launches, outs = {}, {}, {}
    for rep in range(2):
        for name, fn in (("loop", loop), ("batch", batch)):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            ops.launch_count_reset()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            outs[name] = fn()
            t1.record()
            torch.cuda.synchronize()
            ms[name].append(t0.elapsed_time(t1))
            launches[name] = ops.launch_count()
            peak[name] = torch.cuda.max_memory_allocated()
    equal = [bool(torch.equal(a, b)) for a, b in zip(outs["loop"], outs["batch"])]
    audio_s = sum(s.size(-1) for s in srcs) / SR
    best = {k: min(v) for k, v in ms.items()}
    leg = dict(mode=mode, utterances=len(srcs), audio_seconds=round(audio_s, 2),
               segments=sum(-(-s.size(-1) // (5 * SR)) for s in srcs), max_segments=max_segments)
    for k in ("loop", "batch"):
        leg[k] = dict(ms=[round(x, 1) for x in ms[k]], utterances_per_s=round(len(srcs) / best[k] * 1e3, 2),
                      audio_seconds_per_s=round(audio_s / best[k] * 1e3, 1), peak_mem_gb=round(peak[k] / 2 ** 30, 2),
                      launches=launches[k])
    leg["speedup"] = round(best["loop"] / best["batch"], 2)
    leg["outputs_equal"] = all(equal)
    leg["utterances_equal"] = sum(equal)
    return leg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=64)
    ap.add_argument("--modes", nargs="+", default=["se", "tse"])
    ap.add_argument("--max-segments", type=int, default=None, help="default: unise.MAX_SEGMENTS")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unise_enhance_bench: needs a CUDA device")
    from unified_audio_b200.unise import MAX_SEGMENTS
    dev = torch.device("cuda")
    model = build_model(dev)
    srcs, enrolls = make_set(args.utterances, 2026, dev)
    ms = args.max_segments or MAX_SEGMENTS
    legs = [run(model, mode, srcs, enrolls, ms) for mode in args.modes]
    print(json.dumps(dict(metric="unise_enhance_batch", legs=legs, card=card())))


if __name__ == "__main__":
    main()
