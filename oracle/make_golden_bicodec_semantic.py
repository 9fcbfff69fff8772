"""Pin oracle/bicodec_semantic.py against the reference's own classes and write the golden fixture of BiCodec's semantic tokens.

Run in the build container only (reads the reference tree):  python -m oracle.make_golden_bicodec_semantic
Builds QuarkAudio-UniSE/model/bicodec's Encoder and FactorizedVectorQuantize with the oracle's hyper-parameters on a
`BiCodec.__new__` instance that also carries the SpeakerEncoder and the mel transformer of the reference's own
`BiCodec.init_mel_transformer`, loads the seeded weights and runs the reference's unmodified `BiCodec.get_semantic_tokens` and
`BiCodec.tokenize` (bicodec.py:151-172), then its unmodified `BiCodecTokenizer.tokenize` (audio_tokenizer.py:92-105) with
processor = transformers.Wav2Vec2FeatureExtractor() and feature_extractor = a seeded transformers.Wav2Vec2Model at the small
wav2vec2 width (64), built as oracle/make_golden_wav2vec2.py builds it.  The small wav2vec2 keeps one 64-wide attention head: the
product's attention kernels take head_dim 64.  The speaker side is that of tests/golden/bicodec_global_small.npz (seed and
calibrated project_in).  The stubs are those of oracle/make_golden_bicodec.py and make_golden_bicodec_global.py.
Outputs: tests/golden/bicodec_semantic_small.npz (feats, encoder output, z_e, tokens, an end-to-end wav -> (global, semantic)
case), tests/golden/bicodec_semantic_keys.json (reference keys + shapes of the semantic path, shipped configuration),
tests/golden/bicodec_semantic_pinning_report.json.
"""
import json
import os

import numpy as np
import torch

from oracle.make_golden_bicodec import ROOT, _stub_modules
from oracle.make_golden_bicodec_global import ref_get_ref_clip, synth_wav

GOLD = os.path.join(ROOT, "tests", "golden")
SMALL_SEED, SMALL_B, SMALL_T = 48, 3, 40          # seed chosen: every margin >= 1e-3 and >= 64 distinct codes
E2E_SEED, E2E_B, E2E_L, E2E_REF = 40, 2, 6400, 9600   # seed chosen: every semantic and FSQ margin >= 5e-3


def small_config():
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    return dict(og.bicodec_global_small(), encoder=osm.bicodec_semantic_small()["encoder"])


def e2e_wav2vec2_config():
    from oracle import wav2vec2 as ow
    return dict(ow.wav2vec2_small(), conv_dim=[64] * 7, heads=1)


def small_state_dict(cfg, seed):
    """detokenize-path weights (codebook, out_project, ...) + the semantic path + the global fixture's speaker weights"""
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    g = np.load(os.path.join(GOLD, "bicodec_global_small.npz"))
    sd = dict(ob.make_state_dict(cfg, seed))
    sd.update(osm.make_semantic_state_dict(cfg, seed))
    sd.update(og.make_speaker_state_dict(cfg, int(json.loads(str(g["meta"]))["seed"])))
    sd["speaker_encoder.quantizer.project_in.weight"] = torch.from_numpy(g["project_in_weight"])
    sd["speaker_encoder.quantizer.project_in.bias"] = torch.from_numpy(g["project_in_bias"])
    return sd


def build_reference(cfg, sd, with_speaker=True):
    _stub_modules()
    from model.bicodec.bicodec import BiCodec
    from model.bicodec.modules.encoder_decoder.feat_encoder import Encoder
    from model.bicodec.modules.speaker.speaker_encoder import SpeakerEncoder
    from model.bicodec.modules.vq.factorized_vector_quantize import FactorizedVectorQuantize
    q, s = cfg["quantizer"], cfg["speaker"]
    model = BiCodec.__new__(BiCodec)
    torch.nn.Module.__init__(model)
    model.encoder = Encoder(**cfg["encoder"])
    model.quantizer = FactorizedVectorQuantize(q["input_dim"], q["codebook_size"], q["codebook_dim"], commitment=0.25)
    if with_speaker:
        model.speaker_encoder = SpeakerEncoder(input_dim=cfg["mel_params"]["num_mels"], out_dim=s["out_dim"], latent_dim=s["latent_dim"],
                                               token_num=s["token_num"], fsq_levels=s["fsq_levels"], fsq_num_quantizers=s["fsq_num_quantizers"])
        model.init_mel_transformer(cfg["mel_params"])
    own = model.state_dict()
    missing, unexpected = model.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
    assert not unexpected, unexpected
    ok = ("quantizer.cluster_size", "speaker_encoder.speaker_encoder.pool.", "speaker_encoder.speaker_encoder.bn.",
          "speaker_encoder.speaker_encoder.linear.", "mel_transformer.")
    bad = [k for k in missing if not k.startswith(ok) and not k.endswith("num_batches_tracked")]
    assert not bad, bad
    return model.eval()


def ref_tokenizer(model, w2v_cfg, w2v_sd, ref_segment_duration):
    import importlib.machinery
    import sys
    import types
    from transformers import Wav2Vec2FeatureExtractor
    from oracle.make_golden_wav2vec2 import hf_model
    for name in ("soxr", "soundfile"):           # imported by utils/audio.py's load_audio, which tokenize does not use
        try:
            __import__(name)
        except ImportError:
            sys.modules[name] = types.ModuleType(name)
            sys.modules[name].__spec__ = importlib.machinery.ModuleSpec(name, None)
    from model.bicodec.audio_tokenizer import BiCodecTokenizer
    tok = BiCodecTokenizer.__new__(BiCodecTokenizer)
    torch.nn.Module.__init__(tok)
    tok.config = dict(sample_rate=16000, ref_segment_duration=ref_segment_duration, latent_hop_length=320)
    tok.model = model
    tok.processor = Wav2Vec2FeatureExtractor()
    tok.feature_extractor = hf_model(w2v_cfg, w2v_sd)
    tok.feature_extractor.config.output_hidden_states = True
    return tok


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def run_small(seed):
    from oracle import bicodec_semantic as osm
    cfg = small_config()
    sd = small_state_dict(cfg, seed)
    feat = osm.synth_feat(SMALL_B, SMALL_T, cfg["encoder"]["input_channels"], seed + 100)
    sd64 = {k: v.double() for k, v in sd.items()}
    taps = {}
    got = osm.get_semantic_tokens(sd64, cfg, feat.double(), taps)
    margins = osm.fvq_margins(sd64, taps["encoder"])
    return cfg, sd, feat, got, taps, margins


def main():
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from oracle import wav2vec2 as ow
    report = {}
    # ---- small: reference Encoder + FVQ + tokenize
    cfg, sd, feat, got, taps, margins = run_small(SMALL_SEED)
    model = build_reference(cfg, sd)
    with torch.no_grad():
        want = model.get_semantic_tokens({"feat": feat})
        enc = model.encoder(feat.transpose(1, 2)).transpose(1, 2)
        z_e = model.quantizer.in_project(enc.transpose(1, 2)).transpose(1, 2)
    distinct = len(set(want.reshape(-1).tolist()))
    r = dict(tokens_equal=bool(torch.equal(got, want)), dtype=str(want.dtype), shape=list(want.shape), encoder_rel=rel(taps["encoder"], enc),
             z_e_rel=rel(taps["z_e"], z_e), min_margin=float(margins.min()), distinct_codes=distinct, frames=SMALL_B * SMALL_T)
    report["small"] = r
    print("small", r)
    assert r["tokens_equal"] and want.dtype == torch.int64 and max(r["encoder_rel"], r["z_e_rel"]) < 1e-5
    assert r["min_margin"] >= 1e-3 and distinct >= 64, (r["min_margin"], distinct)
    # the reference's BiCodec.tokenize on the same features and a reference clip
    ref_wav = synth_wav(SMALL_B, 3200, SMALL_SEED + 200)
    with torch.no_grad():
        sem_t, glob_t = model.tokenize({"feat": feat, "ref_wav": ref_wav})
    assert torch.equal(sem_t, want)
    assert torch.equal(glob_t, og.get_global_tokens({k: v.double() for k, v in sd.items()}, cfg, ref_wav.double()))
    # ---- end to end: the reference's BiCodecTokenizer.tokenize with a seeded wav2vec2
    wc = e2e_wav2vec2_config()
    wsd = ow.make_state_dict(wc, E2E_SEED)
    tok = ref_tokenizer(model, wc, wsd, E2E_REF / 16000)
    wav = synth_wav(E2E_B, E2E_L, E2E_SEED + 300)
    with torch.no_grad():
        g_ref, s_ref = tok.tokenize(wav)
    sd64 = {k: v.double() for k, v in sd.items()}
    w_feat = ow.extract_wav2vec2_features(wsd, wc, wav)
    etaps, gtaps = {}, {}
    s_or = osm.get_semantic_tokens(sd64, cfg, w_feat.double(), etaps)
    clip = og.get_ref_clip(wav, E2E_REF)
    assert torch.equal(clip, ref_get_ref_clip(wav, cfg, E2E_REF / 16000))
    g_or = og.get_global_tokens(sd64, cfg, clip.double(), gtaps)
    e2e = dict(global_equal=bool(torch.equal(g_or, g_ref)), semantic_equal=bool(torch.equal(s_or, s_ref)),
               semantic_min_margin=float(osm.fvq_margins(sd64, etaps["encoder"]).min()),
               fsq_min_margin=float(og.fsq_margins(gtaps["z"], cfg["speaker"]["fsq_levels"]).min()),
               global_shape=list(g_ref.shape), semantic_shape=list(s_ref.shape), wav2vec2=dict(wc, conv_dim=wc["conv_dim"][0]))
    report["end_to_end"] = e2e
    print("end_to_end", e2e)
    assert e2e["global_equal"] and e2e["semantic_equal"] and g_ref.dtype == torch.int32 and s_ref.dtype == torch.int64
    assert min(e2e["semantic_min_margin"], e2e["fsq_min_margin"]) >= 5e-3, e2e
    np.savez_compressed(os.path.join(GOLD, "bicodec_semantic_small.npz"),
                        meta=json.dumps(dict(seed=SMALL_SEED, feat_seed=SMALL_SEED + 100, B=SMALL_B, T=SMALL_T, w2v_seed=E2E_SEED,
                                             ref_segment_length=E2E_REF)),
                        feat=feat.numpy(), encoder=enc.numpy(), z_e=z_e.numpy(), tokens=want.numpy(), ref_wav=ref_wav.numpy(),
                        global_tokens=glob_t.numpy(), e2e_wav=wav.numpy(), e2e_global=g_ref.numpy(), e2e_semantic=s_ref.numpy())
    # ---- shipped configuration: reference keys and a full-width pin on a few frames
    full = osm.BICODEC_SEMANTIC_FULL
    fsd = dict(osm.make_semantic_state_dict(full, 5))
    from oracle import bicodec as ob
    fsd.update({k: v for k, v in ob.make_state_dict(full, 5).items() if k.startswith("quantizer.")})
    fmodel = build_reference(full, fsd, with_speaker=False)
    ff = osm.synth_feat(1, 12, full["encoder"]["input_channels"], 6)
    with torch.no_grad():
        fwant = fmodel.get_semantic_tokens({"feat": ff})
        fenc = fmodel.encoder(ff.transpose(1, 2)).transpose(1, 2)
    ftaps = {}
    fgot = osm.get_semantic_tokens({k: v.double() for k, v in fsd.items()}, full, ff.double(), ftaps)
    report["full"] = dict(tokens_equal=bool(torch.equal(fgot, fwant)), encoder_rel=rel(ftaps["encoder"], fenc), frames=12)
    print("full", report["full"])
    assert report["full"]["tokens_equal"] and report["full"]["encoder_rel"] < 1e-5
    keys = {k: list(v.shape) for k, v in fmodel.state_dict().items() if k.startswith(("encoder.", "quantizer.in_project."))}
    json.dump(keys, open(os.path.join(GOLD, "bicodec_semantic_keys.json"), "w"), indent=0)
    json.dump(report, open(os.path.join(GOLD, "bicodec_semantic_pinning_report.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
