"""Pin oracle/bicodec_global.py against the reference's own classes and write the golden fixture of BiCodec's global tokens.

Run in the build container only (reads the reference tree):  python -m oracle.make_golden_bicodec_global
Builds QuarkAudio-UniSE/model/bicodec's SpeakerEncoder with the oracle's hyper-parameters, gives a `BiCodec.__new__` instance
that speaker encoder and the mel transformer of the reference's own `BiCodec.init_mel_transformer`, loads the seeded weights and
runs the reference's unmodified `BiCodec.get_global_tokens` (bicodec.py:174-178) and `BiCodecTokenizer.get_ref_clip`
(audio_tokenizer.py:54-72).  The omegaconf / einx stubs are those of oracle/make_golden_bicodec.py; audio_tokenizer.py's
transformers import is satisfied by the image's transformers, its audio loader's soxr / soundfile by empty modules.
Outputs: tests/golden/bicodec_global_small.npz (ref_wav, mel, latent, perceiver output, z, tokens, a get_ref_clip case),
tests/golden/bicodec_global_keys.json (reference state-dict keys + shapes of the global path, shipped configuration),
tests/golden/bicodec_global_pinning_report.json.
"""
import importlib.machinery
import json
import os
import sys
import types

import numpy as np
import torch

from oracle.make_golden_bicodec import ROOT, _stub_modules

SMALL_SEED, SMALL_B, SMALL_L = 23, 4, 3200        # seed chosen: every FSQ level visited, smallest margin 1.4e-2


def build_reference(cfg, sd):
    _stub_modules()
    from model.bicodec.bicodec import BiCodec
    from model.bicodec.modules.speaker.speaker_encoder import SpeakerEncoder
    s = cfg["speaker"]
    speaker = SpeakerEncoder(input_dim=cfg["mel_params"]["num_mels"], out_dim=s["out_dim"], latent_dim=s["latent_dim"],
                             token_num=s["token_num"], fsq_levels=s["fsq_levels"], fsq_num_quantizers=s["fsq_num_quantizers"])
    model = BiCodec.__new__(BiCodec)
    torch.nn.Module.__init__(model)
    model.speaker_encoder = speaker
    model.init_mel_transformer(cfg["mel_params"])
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    xvec = ("speaker_encoder.speaker_encoder.pool.", "speaker_encoder.speaker_encoder.bn.", "speaker_encoder.speaker_encoder.linear.",
            "speaker_encoder.quantizer.project_out.", "speaker_encoder.project.", "mel_transformer.")
    bad = [k for k in missing if not k.startswith(xvec) and not k.endswith("num_batches_tracked")]
    assert not bad, bad
    return model.eval()


def ref_get_ref_clip(wav, cfg, ref_segment_duration):
    for name in ("soxr", "soundfile"):           # imported by utils/audio.py's load_audio, which get_ref_clip does not use
        try:
            __import__(name)
        except ImportError:
            sys.modules[name] = types.ModuleType(name)
            sys.modules[name].__spec__ = importlib.machinery.ModuleSpec(name, None)
    from model.bicodec.audio_tokenizer import BiCodecTokenizer
    tok = BiCodecTokenizer.__new__(BiCodecTokenizer)
    torch.nn.Module.__init__(tok)
    tok.config = dict(sample_rate=cfg["mel_params"]["sample_rate"], ref_segment_duration=ref_segment_duration, latent_hop_length=320)
    return tok.get_ref_clip(wav)


def synth_wav(B, L, seed):
    """noise plus a few partials per clip, peak ~0.5"""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / 16000
    f0 = 100 + 200 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    w = sum(torch.sin(2 * np.pi * f0 * k * t + k) / k for k in range(1, 6))
    w = w + 0.3 * torch.randn(B, L, generator=g, dtype=torch.float64)
    return (0.5 * w / w.abs().amax(dim=1, keepdim=True)).float()


def run_reference(model, wav):
    with torch.no_grad():
        tokens = model.get_global_tokens({"ref_wav": wav})
        mel = model.mel_transformer(wav).squeeze(1)
        _, latent = model.speaker_encoder.speaker_encoder(mel.transpose(1, 2), True)
        x = model.speaker_encoder.perceiver_sampler(latent.transpose(1, 2))
        z = model.speaker_encoder.quantizer.project_in(x)
    return dict(tokens=tokens, mel=mel, latent=latent, perceiver=x, z=z)


def calibrate_project_in(sd, cfg, wav):
    """Untrained perceiver outputs share a large common part, so a seeded project_in leaves most FSQ dimensions on one level.
    For the small fixture, project_in is rescaled and re-centred on the fixture's own perceiver outputs so that every dimension
    spreads over its levels (std 1.5 around bound's centre); the calibrated weight and bias are stored in the fixture."""
    from oracle import bicodec_global as og
    sd64 = {k: v.double() for k, v in sd.items()}
    taps = {}
    og.get_global_tokens(sd64, cfg, wav.double(), taps)
    z = taps["z"].reshape(-1, taps["z"].shape[-1])
    w, b = sd64["speaker_encoder.quantizer.project_in.weight"], sd64["speaker_encoder.quantizer.project_in.bias"]
    gain = 1.5 / z.std(0)
    w = w * gain[:, None]
    b = (b - z.mean(0)) * gain - 0.3466      # bound(z) = -0.5 at z = -atanh(0.5 / 1.5015): the middle of levels -2..1
    sd["speaker_encoder.quantizer.project_in.weight"] = w.float()
    sd["speaker_encoder.quantizer.project_in.bias"] = b.float()


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def main():
    from oracle import bicodec_global as og
    gold = os.path.join(ROOT, "tests", "golden")
    report = {}
    for name, cfg, B, L, seed in (("small", og.bicodec_global_small(), SMALL_B, SMALL_L, SMALL_SEED),
                                  ("full", og.BICODEC_GLOBAL_FULL, 2, 96000, 21)):
        sd = og.make_speaker_state_dict(cfg, seed)
        wav = synth_wav(B, L, seed + 100)
        if name == "small":
            calibrate_project_in(sd, cfg, wav)
        model = build_reference(cfg, sd)
        ref = run_reference(model, wav)
        sd64 = {k: v.double() for k, v in sd.items()}
        taps = {}
        got = og.get_global_tokens(sd64, cfg, wav.double(), taps)
        levels = cfg["speaker"]["fsq_levels"]
        margins = og.fsq_margins(taps["z"], levels)
        visits = [sorted(set(int(v) for v in torch.round(og.fsq_bound(taps["z"], levels))[..., j].reshape(-1))) for j in range(len(levels))]
        r = dict(tokens_equal=bool(torch.equal(got, ref["tokens"])), dtype=str(ref["tokens"].dtype), shape=list(ref["tokens"].shape),
                 mel_rel=rel(taps["mel"], ref["mel"]), latent_rel=rel(taps["latent"], ref["latent"]),
                 perceiver_rel=rel(taps["perceiver"], ref["perceiver"]), z_rel=rel(taps["z"], ref["z"]),
                 z_absmax_err=float((taps["z"] - ref["z"].double()).abs().max()), min_margin=float(margins.min()),
                 levels_visited=visits, frames=int(ref["mel"].shape[-1]))
        report[name] = r
        print(name, r)
        assert r["tokens_equal"] and ref["tokens"].dtype == torch.int32
        assert ref["tokens"].shape == (B, 1, cfg["speaker"]["token_num"])
        assert max(r["mel_rel"], r["latent_rel"], r["perceiver_rel"], r["z_rel"]) < 1e-5      # the reference runs in fp32
        if name == "small":
            assert all(len(v) == levels[j] for j, v in enumerate(visits)), visits
            assert r["min_margin"] > 1e-3, r["min_margin"]
            short = synth_wav(1, 1000, seed + 200)
            long_ = synth_wav(1, 4000, seed + 300)
            seg = 0.2                        # 3200 samples at 16 kHz
            clips = [ref_get_ref_clip(w, cfg, seg) for w in (short, long_)]
            assert torch.equal(clips[0], og.get_ref_clip(short, 3200)) and torch.equal(clips[1], og.get_ref_clip(long_, 3200))
            np.savez_compressed(os.path.join(gold, "bicodec_global_small.npz"),
                                meta=json.dumps(dict(seed=seed, wav_seed=seed + 100, B=B, L=L, ref_segment_length=3200)),
                                ref_wav=wav.numpy(), mel=ref["mel"].numpy(), latent=ref["latent"].numpy(),
                                perceiver=ref["perceiver"].numpy(), z=ref["z"].numpy(), tokens=ref["tokens"].numpy(),
                                project_in_weight=sd["speaker_encoder.quantizer.project_in.weight"].numpy(),
                                project_in_bias=sd["speaker_encoder.quantizer.project_in.bias"].numpy(), short_wav=short.numpy(), short_clip=clips[0].numpy(), long_wav=long_.numpy(), long_clip=clips[1].numpy())
        else:
            keys = {k: list(v.shape) for k, v in model.state_dict().items() if k.startswith("speaker_encoder.") and
                    not k.startswith(("speaker_encoder.quantizer.project_out.", "speaker_encoder.project."))}
            json.dump(keys, open(os.path.join(gold, "bicodec_global_keys.json"), "w"), indent=0)
    json.dump(report, open(os.path.join(gold, "bicodec_global_pinning_report.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
