"""Time Codec.forward against the encode -> decode round trip, and the semantic decoder alone.

    python scripts/codec_forward_bench.py [--steps 10] [--warmup 3] [--out DIR]

Cases (seeded weights, shipped widths): H-Codec-2.0 at B = 64 x 10 s (forward vs roundtrip ms per call, semantic_decode ms and
TFLOP/s from the decoder's conv shapes); H-Codec-1.0 and 1.5 at B = 32 x 10 s (H-Codec-1.5 with fewer transformer layers,
oracle/hcodec15.py's h15_shallow: the semantic decoder's widths are the shipped ones).  Times are CUDA events around calls that
end in a device synchronise.  Prints one JSON object with the card's name and power limit.  Needs a GPU: there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def sem_dec_flops(cfg, B, N):
    """2 x MACs of the semantic decoder on N codes per clip (cfg: the Decoder kwargs, widths from decode_channels * channel_ratios
    as vq/semantic_module.py:268-289 derives them)"""
    dc, strides = cfg["decode_channels"], cfg["strides"]
    ratios = cfg.get("channel_ratios", [1] * len(strides))
    width = lambda i: int(dc * ratios[i]) if i < len(strides) else dc
    T, cin = N, width(0)
    f = 2 * B * T * cin * cfg["code_dim"] * 3
    for i, st in enumerate(strides):
        co = width(i + 1)
        if st == 1:
            f += 2 * B * T * co * cin * 3
        else:
            f += 2 * B * T * co * cin * 2 * st          # every input frame meets all 2s taps
            T *= st
        f += 2 * (2 * B * T * co * co * 3 + 2 * B * T * co * co)
        cin = co
    return f + 2 * B * T * cfg["output_channels"] * cin * 3


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("codec_forward_bench needs a CUDA device")
    from oracle import hcodec1, hcodec15, weights
    from oracle import semantic_decoder as osd
    from unified_audio_b200.codec import Codec
    from unified_audio_b200.codec_h1 import CodecH1
    from unified_audio_b200.codec_h15 import CodecH15
    res = {}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res["gpu"] = gpu.strip().splitlines()[0] if gpu.strip() else "unknown"

    cfg = weights.H2_FULL
    sd = dict(weights.make_h2_state_dict(cfg, 1), **osd.make_state_dict(cfg["semantic_decoder_config"], 2))
    m = Codec(cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"],
              cfg["semantic_decoder_config"], semantic_decoder=True)
    m.load_state_dict(sd, strict=True)
    del sd
    m = m.cuda()
    B, N = 64, 125
    wav, feat = weights.synth_inputs(cfg, B, N, 3)
    wav, feat = wav.cuda(), feat.cuda()
    _, sc = m.encode(wav, feat)
    ms_sd = timed(lambda: m.semantic_decode(sc), a.steps, a.warmup)
    res["h2_b64_10s"] = dict(forward_ms=timed(lambda: m(wav, feat), a.steps, a.warmup),
                             roundtrip_ms=timed(lambda: m.roundtrip(wav, feat), a.steps, a.warmup), semantic_decode_ms=ms_sd,
                             semantic_decode_tflops=sem_dec_flops(cfg["semantic_decoder_config"], B, N) / ms_sd / 1e9)
    del m
    torch.cuda.empty_cache()

    for name, c, make, build in (("h1_b32_10s", hcodec1.H1, hcodec1.make_state_dict, lambda c: CodecH1(semantic_decoder=True)),
                                 ("h15_shallow_b32_10s", hcodec15.h15_shallow(), hcodec15.make_state_dict,
                                  lambda c: CodecH15(_cfg={k: v for k, v in c.items() if k != "layer_scale"}, semantic_decoder=True))):
        dcfg = osd.h1_config(c)
        m = build(c)
        m.load_state_dict(dict(make(c, 1), **osd.make_state_dict(dcfg, 2)), strict=True)
        m = m.cuda()
        B, T = 32, 160000
        g = torch.Generator().manual_seed(4)
        x = (0.1 * torch.randn(B, 1, T, generator=g)).cuda()
        f = torch.randn(B, c["sem_in"], T // 320, generator=g)
        f = (torch.sign(f) * f.abs() ** 0.3).cuda()
        codes = m.encode(x, f)
        sc = codes["semantic_codes"] if isinstance(codes, dict) else codes[1]
        ms_sd = timed(lambda: m.semantic_decode(sc), a.steps, a.warmup)
        res[name] = dict(forward_ms=timed(lambda: m(x, f), a.steps, a.warmup),
                         roundtrip_ms=timed(lambda: m.roundtrip(x, f), a.steps, a.warmup), semantic_decode_ms=ms_sd,
                         semantic_decode_tflops=sem_dec_flops(dcfg, B, T // 640) / ms_sd / 1e9)
        del m
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "codec_forward_bench.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
