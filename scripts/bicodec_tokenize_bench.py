"""Time BiCodec tokenize on the GPU: unise.BiCodecTokenizer.tokenize over B clips of 5 s (UniSE's segment), shipped configuration,
seeded weights; the reference clip is the 5 s clip tiled to 6 s by get_ref_clip.  CUDA events around `--iters` calls of each stage
after `--warmup` calls: wav2vec2-XLSR-53 features, semantic tokens (Encoder + FVQ), global tokens, and the whole tokenize.  Prints
one JSON line with ms per call, clips/s, the FLOP count derived from the shapes below, the card and its power limit."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bicodec_global_bench import card, flops as global_flops  # noqa: E402


def wav2vec2_flops(c, B, L):
    """conv stack, feature projection, grouped positional conv and the layers up to the last averaged hidden state"""
    f, T = 0, L
    cin = 1
    for co, k, s in zip(c["conv_dim"], c["conv_kernel"], c["conv_stride"]):
        T = (T - k) // s + 1
        f += 2 * B * T * co * cin * k
        cin = co
    H, M = c["hidden"], B * T
    f += 2 * M * H * cin + 2 * M * H * (H // c["pos_groups"]) * c["pos_k"]
    f += max(c["hidden_state_ids"]) * (2 * M * 4 * H * H + 2 * 2 * M * H * c["ffn"] + 2 * 2 * B * T * T * H)
    return f, T


def semantic_flops(cfg, B, T):
    e, q = cfg["encoder"], cfg["quantizer"]
    M, dim, inter = B * T, e["vocos_dim"], e["vocos_intermediate_dim"]

    def backbone(cin, layers):
        return 2 * M * dim * cin * 7 + layers * (2 * 2 * M * dim * inter + 2 * M * dim * 7)
    f = backbone(e["input_channels"], e["vocos_num_layers"]) + len(e["sample_ratios"]) * backbone(dim, 2)
    f += 2 * M * e["out_channels"] * dim
    return f + 2 * M * q["codebook_dim"] * (q["input_dim"] + q["codebook_size"])       # in_project + the fp64 codebook scan


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=5.0)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bicodec_tokenize_bench: needs a CUDA device")
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from oracle import wav2vec2 as ow
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.ssl import WAV2VEC2_XLSR53, SSLFrontEnd
    from unified_audio_b200.unise import BiCodecTokenizer
    cfg = dict(og.BICODEC_GLOBAL_FULL, encoder=osm.ENCODER_PARAMS)
    sd = dict(ob.make_state_dict(cfg, 0))
    sd.update(og.make_speaker_state_dict(cfg, 0))
    sd.update(osm.make_semantic_state_dict(cfg, 0))
    m = BiCodec(cfg, global_tokens=True, semantic_tokens=True)
    m.load_state_dict(sd, strict=True)
    w2v = SSLFrontEnd(WAV2VEC2_XLSR53, in_rate=16000)
    w2v.load_state_dict(ow.make_state_dict(ow.WAV2VEC2_XLSR53, 0), strict=True)
    tok = BiCodecTokenizer(m.cuda(), feature_extractor=w2v.cuda())
    L = int(16000 * args.seconds)
    wav = 0.1 * torch.randn(args.batch, L, generator=torch.Generator().manual_seed(0)).cuda()
    ref = tok.get_ref_clip(wav)
    feat = w2v(wav)
    ms = dict(wav2vec2=timed(lambda: w2v(wav), args.iters, args.warmup),
              semantic_tokens=timed(lambda: m.get_semantic_tokens({"feat": feat}), args.iters, args.warmup),
              global_tokens=timed(lambda: m.get_global_tokens({"ref_wav": ref}), args.iters, args.warmup),
              tokenize=timed(lambda: tok.tokenize(wav), args.iters, args.warmup))
    fw, T = wav2vec2_flops(WAV2VEC2_XLSR53, args.batch, L)
    fl = dict(wav2vec2=fw, semantic_tokens=semantic_flops(cfg, args.batch, T), global_tokens=global_flops(cfg, args.batch, ref.shape[1]))
    fl["tokenize"] = sum(fl.values())
    print(json.dumps(dict(metric="bicodec_tokenize", batch=args.batch, seconds_per_clip=L / 16000, frames=T,
                          ms_per_call={k: round(v, 3) for k, v in ms.items()},
                          clips_per_s={k: round(args.batch / v * 1e3, 1) for k, v in ms.items()},
                          gflop_per_call={k: round(v / 1e9, 2) for k, v in fl.items()},
                          tflops_one_pass={k: round(fl[k] / ms[k] / 1e9, 2) for k in ms}, card=card())))


if __name__ == "__main__":
    main()
