"""Time BiCodec.get_global_tokens on the GPU: B clips of 6 s (UniSE's 5 s segments tiled to BiCodec's reference clip by
get_ref_clip), shipped configuration, seeded weights.  CUDA events around `--iters` calls after `--warmup` calls; prints one JSON
line with ms per call, clips/s, the FLOP count derived from the shapes below, the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def flops(cfg, B, L):
    """multiply-adds x 2 of every contraction as run (one pass; the 3-term split issues 3 tensor-core passes of each)"""
    mp, s = cfg["mel_params"], cfg["speaker"]
    T = 1 + L // mp["hop_length"]
    M, nf, nm = B * T, mp["n_fft"] // 2 + 1, mp["num_mels"]
    P, Q = 64, mp["n_fft"] // 64
    K2 = (nf - 1) // P + 1
    f = 2 * M * Q * 2 * P * 64 + 2 * M * P * 2 * K2 * 128 + 2 * M * nm * nf               # two-stage DFT, filter bank
    f += 2 * M * 512 * nm * 5                                                              # layer1
    f += 3 * (2 * 2 * M * 512 * 512 + 7 * 2 * M * 64 * 64 * 3 + 2 * 2 * B * 512 * 128)   # SE-Res2 blocks
    f += 2 * M * 1536 * 1536                                                               # 1x1 conv over the concat
    D, N, inner = s["latent_dim"], s["token_num"], int(s["latent_dim"] * 8 / 3)
    R, Nk = B * N, N + T
    f += 2 * M * D * 1536
    f += 2 * (2 * R * 512 * D + 2 * B * Nk * 1024 * D + 2 * 2 * B * 8 * N * Nk * 64 + 2 * R * D * 512 + 2 * R * 2 * inner * D
              + 2 * R * D * inner)
    return f


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=6.0)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bicodec_global_bench: needs a CUDA device")
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from unified_audio_b200.bicodec import BiCodec
    cfg = og.BICODEC_GLOBAL_FULL
    sd = dict(ob.make_state_dict(cfg, 0))
    sd.update(og.make_speaker_state_dict(cfg, 0))
    m = BiCodec(cfg, global_tokens=True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    L = int(16000 * args.seconds) // 320 * 320
    wav = 0.1 * torch.randn(args.batch, L, generator=torch.Generator().manual_seed(0)).cuda()
    batch = {"ref_wav": wav}
    for _ in range(args.warmup):
        m.get_global_tokens(batch)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.iters):
        m.get_global_tokens(batch)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.iters
    f = flops(cfg, args.batch, L)
    print(json.dumps(dict(metric="bicodec_get_global_tokens", batch=args.batch, seconds_per_clip=L / 16000, ms_per_call=round(ms, 3),
                          clips_per_s=round(args.batch / ms * 1e3, 1), gflop_per_call=round(f / 1e9, 2),
                          tflops_one_pass=round(f / ms / 1e9, 2), card=card())))


if __name__ == "__main__":
    main()
