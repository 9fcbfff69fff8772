"""Time UniSE's validation step on the GPU: unise.Model.validation_step over B clips of 5 s in modes 'se' and 'tse', shipped widths,
seeded weights (XLSR-53 + BiCodec both token paths, WavLM-base-plus, the LM as bench.build_lm makes it).  B = 1 is the shipped
validation batch (conf/config.yaml val_kwargs.batch_size), B = 32 the training batch.  After `--warmup` steps, CUDA events around
`--iters` steps give ms per step and clips/s; a second timed loop runs the step's three stages with an event between them
(tokenize, WavLM on mix + enroll, LM forward).  `launches` is the library's own kernel-launch count for one step (torch's small
glue kernels are not counted).  Prints one JSON line with the card and its power limit; fails without a GPU."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bicodec_global_bench import card  # noqa: E402

SEG = 5 * 16000


def build_model(dev):
    import bench
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from oracle import hubert as oh
    from oracle import wav2vec2 as ow
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.ssl import WAV2VEC2_XLSR53, WAVLM_BASE_PLUS, SSLFrontEnd
    from unified_audio_b200.unise import BiCodecTokenizer, Model
    cfg = dict(og.BICODEC_GLOBAL_FULL, encoder=osm.ENCODER_PARAMS)
    sd = dict(ob.make_state_dict(cfg, 0))
    sd.update(og.make_speaker_state_dict(cfg, 0))
    sd.update(osm.make_semantic_state_dict(cfg, 0))
    codec = BiCodec(cfg, global_tokens=True, semantic_tokens=True)
    codec.load_state_dict(sd, strict=True)
    w2v = SSLFrontEnd(WAV2VEC2_XLSR53, in_rate=16000)
    w2v.load_state_dict(ow.make_state_dict(ow.WAV2VEC2_XLSR53, 0), strict=True)
    wavlm = SSLFrontEnd(WAVLM_BASE_PLUS, in_rate=16000, compress=False)
    wavlm.load_state_dict(oh.wavlm_make_state_dict(oh.WAVLM_BASE_PLUS, 0), strict=True)
    return Model(None, tokenizer=BiCodecTokenizer(codec.to(dev), feature_extractor=w2v.to(dev)), dnn=bench.build_lm(dev),
                 semantic_model=wavlm.to(dev))


def make_batch(mode, B, dev):
    g = torch.Generator().manual_seed(B)
    w = lambda: 0.1 * torch.randn(B, SEG, generator=g).to(dev)
    speech, noise = w(), w()
    enroll = w() if mode == "tse" else None
    return (mode, enroll, speech + 0.5 * noise, speech, noise if mode == "tse" else None, torch.full((B,), 16000, device=dev),
            torch.full((B,), SEG, device=dev), ["x"] * B)


def stages(model, batch):
    """the step's three stages, as _validation_step runs them, with an event after each"""
    mode, enroll, mix, speech = batch[:4]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    g, s = model.tokenizer.tokenize(speech)
    ev[1].record()
    mf = model.extract_semantic_features(mix)
    ef = model.extract_semantic_features(enroll) if enroll is not None else None
    ev[2].record()
    model.dnn(task_name=mode, enroll_mel=None if enroll is None else model.mel_like(enroll), enroll_feats=ef, mix_mel=model.mel_like(mix),
              mix_feats=mf, global_ids=g.squeeze(1), semantic_ids=s)
    ev[3].record()
    return ev


def run(model, mode, B, iters, warmup, dev):
    from unified_audio_b200 import ops
    batch = make_batch(mode, B, dev)
    for _ in range(warmup):
        model.validation_step(batch)
    torch.cuda.synchronize()
    ops.launch_count_reset()
    out = model.validation_step(batch)
    launches = ops.launch_count()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        model.validation_step(batch)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    split = [0.0, 0.0, 0.0]
    for _ in range(iters):
        ev = stages(model, batch)
        torch.cuda.synchronize()
        for i in range(3):
            split[i] += ev[i].elapsed_time(ev[i + 1]) / iters
    return dict(mode=mode, batch=B, ms_per_step=round(ms, 3), clips_per_s=round(B / ms * 1e3, 2), launches=launches,
                stage_ms=dict(tokenize=round(split[0], 3), wavlm=round(split[1], 3), lm_forward=round(split[2], 3)),
                valid_loss=round(float(out["valid_loss"]), 5), valid_acc=round(float(out["valid_acc"]), 5))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unise_validation_bench: needs a CUDA device")
    dev = torch.device("cuda")
    model = build_model(dev)
    legs = [run(model, mode, B, args.iters, args.warmup, dev) for B in args.batches for mode in ("se", "tse")]
    print(json.dumps(dict(metric="unise_validation_step", seconds_per_clip=SEG / 16000, legs=legs, card=card())))


if __name__ == "__main__":
    main()
