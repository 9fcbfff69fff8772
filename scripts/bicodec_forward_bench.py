"""Time BiCodec.forward against tokenize + detokenize, and the two pieces only forward runs: the x-vector and the postnet.

    python scripts/bicodec_forward_bench.py [--steps 10] [--warmup 3] [--out DIR]

Shipped widths, seeded weights, B = 32: feat [32, 250, 1024] (5 s of wav2vec2 frames), ref_wav 6 s (the reference clip length of
BiCodecTokenizer, 301 mel frames), wav 5 s.  The x-vector is timed from the ECAPA latent of that batch, the postnet from its prenet
output.  Times are CUDA events around calls that end in a device synchronise, after warm-up, in ms per call.  Prints one JSON object
with the card's name and power limit.  Needs a GPU: there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
        raise SystemExit("bicodec_forward_bench needs a CUDA device")
    from oracle import bicodec as ob
    from oracle import bicodec_forward as of
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from oracle.make_golden_bicodec_global import synth_wav
    from unified_audio_b200.bicodec import BiCodec
    res = {}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res["gpu"] = gpu.strip().splitlines()[0] if gpu.strip() else "unknown"
    sd = dict(ob.make_state_dict(ob.BICODEC_FULL, 1))
    sd.update(osm.make_semantic_state_dict(osm.BICODEC_SEMANTIC_FULL, 1))
    sd.update(og.make_speaker_state_dict(og.BICODEC_GLOBAL_FULL, 1))
    sd.update(of.make_forward_state_dict(of.BICODEC_FORWARD_FULL, 1))
    m = BiCodec(full=True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    B, T = 32, 250
    batch = {"feat": osm.synth_feat(B, T, 1024, 2).cuda(), "ref_wav": synth_wav(B, 96000, 3).cuda(), "wav": synth_wav(B, 80000, 4).cuda()}

    def roundtrip():
        return m.detokenize(*m.tokenize(batch))

    _, lat32, latp, Tm = m._global_tokens(batch["ref_wav"], keep_latent=True)
    sem, glob = m.tokenize(batch)
    pre, _ = m._prenet(sem, glob)
    res["b32_feat5s_ref6s"] = dict(forward_ms=timed(lambda: m(batch), a.steps, a.warmup),
                                   tokenize_detokenize_ms=timed(roundtrip, a.steps, a.warmup),
                                   x_vector_ms=timed(lambda: m._xvector(lat32, latp, B, Tm), a.steps, a.warmup),
                                   postnet_ms=timed(lambda: m._postnet(pre, B, T), a.steps, a.warmup), mel_frames=Tm)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bicodec_forward_bench.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
