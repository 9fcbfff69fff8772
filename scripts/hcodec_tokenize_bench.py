"""Time the H-Codec-1.0 and H-Codec-1.5 tokenizers on the GPU: `HCodecTokenizerH1.tokenize` (HuBERT-base -> CodecH1.encode) and
`HCodecTokenizerH15.tokenize` (wav2vec2-XLSR-53, 16 of 24 layers -> the adaptive CodecH15.encode), shipped widths, seeded weights,
B clips of 10 s at 16 kHz (the clip shape of bench.py's h15 leg; B = 32 as there, and B = 1).  After `--warmup` calls, CUDA events
around `--iters` calls give ms per call and clips/s; a second timed loop puts an event between the two stages (SSL features, then
encode).  `launches` is the library's own kernel-launch count for one call (torch's small glue kernels are not counted).  For 1.5,
`mean_token_frames` (25 Hz frames per token) sets the aggregator sequence lengths; with random weights and noise it is not what
real speech gives, so it is printed beside the time.  Prints one JSON line with the card and its power limit; fails without a GPU."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bicodec_global_bench import card  # noqa: E402

SECONDS = 10


def build(dev):
    from oracle import hcodec1, hcodec15 as o15, hubert as oh, wav2vec2 as ow
    from unified_audio_b200 import (CodecH1, CodecH15, HCodecTokenizerH1, HCodecTokenizerH15, HUBERT_BASE, SSLFrontEnd,
                                    WAV2VEC2_XLSR53_RAW)
    c1 = CodecH1({}, {}, {})
    c1.load_state_dict(hcodec1.make_state_dict(hcodec1.H1, 0), strict=True)
    hub = SSLFrontEnd(HUBERT_BASE, in_rate=16000, compress=True)
    hub.load_state_dict(oh.make_state_dict(oh.HUBERT_BASE, 0), strict=True)
    c15 = CodecH15()
    c15.load_state_dict(o15.make_state_dict(o15.H15, 0), strict=True)
    w2v = SSLFrontEnd(WAV2VEC2_XLSR53_RAW, in_rate=16000, compress=True)
    w2v.load_state_dict(ow.make_state_dict(ow.WAV2VEC2_XLSR53, 0), strict=True)
    return dict(h1=HCodecTokenizerH1(c1.to(dev), hub.to(dev)), h15=HCodecTokenizerH15(c15.to(dev), w2v.to(dev)))


def stages(name, tok, wav):
    """tokenize's two stages, as the face runs them, with an event after each"""
    from unified_audio_b200 import ops
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    padded = tok.pad_wav(wav)
    src = padded if name == "h1" else ops.pad_wav(padded, 160, padded.shape[-1] + 320)
    feats = tok.feature_extractor(src, channel_first=True)
    ev[1].record()
    tok.model.encode(padded[:, None], feats)
    ev[2].record()
    return ev


def run(name, tok, B, iters, warmup, dev):
    from unified_audio_b200 import adaptive, ops
    g = torch.Generator(device=dev).manual_seed(B)
    wav = 0.1 * torch.randn(B, SECONDS * 16000, generator=g, device=dev)
    for _ in range(warmup):
        out = tok.tokenize(wav)
    torch.cuda.synchronize()
    ops.launch_count_reset()
    out = tok.tokenize(wav)
    launches = ops.launch_count()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        tok.tokenize(wav)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    split = [0.0, 0.0]
    for _ in range(iters):
        ev = stages(name, tok, wav)
        torch.cuda.synchronize()
        for i in range(2):
            split[i] += ev[i].elapsed_time(ev[i + 1]) / iters
    leg = dict(tokenizer=name, batch=B, ms_per_call=round(ms, 3), clips_per_s=round(B / ms * 1e3, 2), launches=launches,
               stage_ms=dict(features=round(split[0], 3), encode=round(split[1], 3)))
    if name == "h15":
        _, lens = adaptive.extract_lengths(out["acoustic_codes"], tok.model.codebook_size)
        leg["mean_token_frames"] = round(float(lens.sum()) / float((lens > 0).sum()), 3)
        leg["tokens_per_clip"] = round(float((lens > 0).sum()) / B, 2)
    return leg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hcodec_tokenize_bench: needs a CUDA device")
    dev = torch.device("cuda")
    toks = build(dev)
    legs = [run(name, tok, B, args.iters, args.warmup, dev) for name, tok in toks.items() for B in args.batches]
    print(json.dumps(dict(metric="hcodec_tokenize", seconds_per_clip=SECONDS, legs=legs, card=card())))


if __name__ == "__main__":
    main()
