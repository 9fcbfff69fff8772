"""Pin the oracle's wav -> codes chains against the REFERENCE'S OWN H-Codec-1.0 and H-Codec-1.5 `HCodecTokenizer`s.

TEST INFRASTRUCTURE.  Run in the build container only:  python -m oracle.make_golden_hcodec_tokenizers

Both reference files are imported unmodified:
  * HCodec-1.0/audio_tokenizer.py uses a package-relative import (`from .vq import Codec`): the HCodec-1.0 directory is loaded as
    a package;
  * HCodec-1.5/audio_tokenizer.py imports `librosa` (stubbed: unused on this path) and `from vq import Codec`, resolved to the
    `vq` package oracle/make_golden_h15.build_reference has just imported (with its stubs).
Each `HCodecTokenizer` is built WITHOUT its `__init__` (which reads a checkpoint and downloads the SSL model) and given
    model             = the reference's own `Codec`, seeded: H-Codec-1.0 at the shipped widths (its `Codec(None, None, None)`
                        hard-codes them), H-Codec-1.5 at `oracle.hcodec15.h15_shallow()` (shipped widths, fewer layers);
    feature_extractor = a seeded `transformers.HubertModel` (768 wide, 2 layers of 12 heads x 64) or `Wav2Vec2Model` (1024 wide,
                        4 layers of 16 heads x 64): reduced in depth only, because the front end's width is the codec's
                        semantic-encoder input.  The 1.5 reference reads hidden_states[11] / [14] / [16] of the 24-layer model;
                        `_StatesAt` puts the reduced model's states 1 / 2 / 3 at those positions (hidden_state_ids (1, 2, 3));
    hop_length / config as the reference's `__init__` sets them.
Its unmodified `pad_wav`, `extract_wav2vec2_features`, `tokenize` and `detokenize` then run on clips whose length is not a multiple
of 640, and the oracle chain (zero-pad -> oracle/hcodec_features.py -> oracle/hcodec1.py / hcodec15.py) is checked against them.

H-Codec-1.5's grouping is decided by the cosine similarity of adjacent semantic-encoder frames against the threshold.  The clips
alternate stretches of noise with stretches of one 640-sample pattern repeated (frames of nearly one feature), and the reduced
config's threshold is put in the middle of the widest gap between the adjacent similarities in [0.7, 0.8], so that single-frame
tokens, merged tokens and the 8-frame cap all occur and no similarity lies near the threshold.  The reference codec is given the
same threshold (`manual_threshold`, which its `encode` reads).

Writes tests/golden/hcodec_tokenizers_small.npz (the reference's outputs; the clips are regenerated from the seeds in its meta
by `synth_clips`) and tests/golden/hcodec_tokenizers_pinning_report.json.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch
from torch import nn

from oracle.make_golden_h15 import REF10, REF15, _purge, _stubs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
HOP = 640
SEEDS = dict(h1_codec=21, h1_ssl=22, h1_wav=23, h15_codec=31, h15_ssl=32, h15_wav=33)
# clips as stretches of 640-sample frames: ("noise", n) or ("rep", n) = one random 640-sample pattern repeated n times
H1_CLIPS = [[("noise", 15)], [("noise", 15)]]
H15_CLIPS = [[("noise", 4), ("rep", 9), ("noise", 3), ("rep", 4)], [("rep", 5), ("noise", 6), ("rep", 6), ("noise", 3)]]
H1_TRIM, H15_TRIM = 213, 301                 # samples cut from the end: lengths are not multiples of 640


def hubert_cfg():
    from oracle import hubert as oh
    return dict(oh.HUBERT_BASE, layers=2)


def wav2vec2_cfg():
    from oracle import wav2vec2 as ow
    return dict(ow.WAV2VEC2_XLSR53, layers=4, hidden_state_ids=(1, 2, 3))


def synth_clips(clips, trim, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for clip in clips:
        parts = [0.1 * torch.randn(n * HOP, generator=g) if kind == "noise" else (0.1 * torch.randn(HOP, generator=g)).repeat(n)
                 for kind, n in clip]
        out.append(torch.cat(parts))
    wav = torch.stack(out)
    return wav[:, : wav.shape[1] - trim].contiguous()


class _StatesAt(nn.Module):
    """a reduced-depth Wav2Vec2Model whose hidden states `ids` are returned at the positions (11, 14, 16) the reference reads"""

    def __init__(self, model, ids, at=(11, 14, 16)):
        super().__init__()
        self.model, self.ids, self.at = model, ids, at

    def forward(self, wavs, output_hidden_states=True):
        hs = self.model(wavs, output_hidden_states=output_hidden_states).hidden_states
        states = [None] * (max(self.at) + 1)
        for a, i in zip(self.at, self.ids):
            states[a] = hs[i]
        return types.SimpleNamespace(hidden_states=tuple(states))


def _load_h1_package():
    _stubs()
    _purge({"vq", "adaptive", "hcodec10_ref"})
    spec = importlib.util.spec_from_file_location("hcodec10_ref", os.path.join(REF10, "__init__.py"), submodule_search_locations=[REF10])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["hcodec10_ref"] = mod
    spec.loader.exec_module(mod)
    return mod


def _load_h15_tokenizer_module():
    sys.modules.setdefault("librosa", types.ModuleType("librosa"))
    spec = importlib.util.spec_from_file_location("hcodec15_ref_audio_tokenizer", os.path.join(REF15, "audio_tokenizer.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _new(cls):
    tok = cls.__new__(cls)
    nn.Module.__init__(tok)
    return tok


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def feats_away_from_zero(got, ref):
    """sign(x)|x|^0.3 has an infinite slope at 0: compare where |ref| > 0.2 max"""
    big = ref.abs() > 0.2 * ref.abs().max()
    return float((got - ref).abs()[big].max() / ref.abs().max())


def run_h1():
    from oracle import hcodec1, hubert as oh
    from oracle.hcodec_features import extract_hcodec1_features
    from oracle.make_golden_hubert import hf_model
    hc = hubert_cfg()
    sd = hcodec1.make_state_dict(hcodec1.H1, SEEDS["h1_codec"])
    fsd = oh.make_state_dict(hc, SEEDS["h1_ssl"])
    pkg = _load_h1_package()
    codec = pkg.vq.Codec(None, None, None).eval()
    missing, unexpected = codec.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith("semantic_decoder.") for k in missing), (missing[:5], unexpected[:5])
    tok = _new(pkg.HCodecTokenizer)
    tok.model, tok.feature_extractor, tok.hop_length = codec, hf_model(hc, fsd), HOP
    wav = synth_clips(H1_CLIPS, H1_TRIM, SEEDS["h1_wav"])
    with torch.no_grad():
        padded_r = tok.pad_wav(wav)
        feats_r = tok.extract_wav2vec2_features(padded_r)
        ac_r, sc_r = tok.tokenize(wav)
        rec_r = tok.detokenize(ac_r, sc_r)
    padded_o = torch.nn.functional.pad(wav, (0, padded_r.shape[-1] - wav.shape[-1]))
    feats_o = extract_hcodec1_features(fsd, hc, padded_o)
    ac_o, sc_o = hcodec1.codec_encode(sd, hcodec1.H1, padded_o[:, None], feats_o.transpose(1, 2))
    rec_o = hcodec1.codec_decode(sd, hcodec1.H1, ac_r, sc_r)
    report = dict(batch=int(wav.shape[0]), samples=int(wav.shape[1]), padded=int(padded_r.shape[1]),
                  padded_equal=bool(torch.equal(padded_r, padded_o)), feature_frames=int(feats_r.shape[1]),
                  feats_rel_away_from_zero=feats_away_from_zero(feats_o, feats_r),
                  acoustic_identical=bool(torch.equal(ac_r, ac_o)), semantic_identical=bool(torch.equal(sc_r, sc_o)),
                  rec_rel=rel(rec_o.reshape(rec_r.shape), rec_r), codes_shape=list(ac_r.shape), rec_shape=list(rec_r.shape))
    print("h1", report)
    assert report["padded_equal"] and report["feats_rel_away_from_zero"] < 1e-4
    assert report["acoustic_identical"] and report["semantic_identical"] and report["rec_rel"] < 1e-5
    arrays = dict(h1_padded_len=torch.tensor(padded_r.shape[-1]), h1_feats=feats_r, h1_acoustic=ac_r, h1_semantic=sc_r,
                  h1_rec=rec_r)
    return report, arrays


def pick_threshold(sim):
    """the middle of the widest gap between adjacent-frame similarities inside [0.7, 0.8], rounded to 1e-3"""
    s = torch.cat([torch.tensor([0.7]), sim.flatten().double().sort().values, torch.tensor([0.8])])
    s = s[(s >= 0.7) & (s <= 0.8)]
    gaps = s[1:] - s[:-1]
    k = int(gaps.argmax())
    return round(float(s[k] + s[k + 1]) / 2, 3)


def run_h15():
    from oracle import adaptive as ad
    from oracle import hcodec1, hcodec15 as o15, wav2vec2 as ow
    from oracle.hcodec_features import extract_hcodec15_features
    from oracle.make_golden_h15 import build_reference, reference_kwargs
    from oracle.make_golden_wav2vec2 import hf_model
    wc = wav2vec2_cfg()
    c = o15.h15_shallow()
    sd = o15.make_state_dict(c, SEEDS["h15_codec"])
    fsd = ow.make_state_dict(wc, SEEDS["h15_ssl"])
    wav = synth_clips(H15_CLIPS, H15_TRIM, SEEDS["h15_wav"])
    padded_o = torch.nn.functional.pad(wav, (0, -wav.shape[-1] % HOP))
    feats_o = extract_hcodec15_features(fsd, wc, padded_o)
    sem = hcodec1.semantic_encoder(sd, c, feats_o.transpose(1, 2))
    sim = torch.nn.functional.cosine_similarity(sem[:, :, :-1], sem[:, :, 1:], dim=1)
    thr = pick_threshold(sim)
    ref = build_reference(c, sd)                         # yaml's manual_threshold (0.6) checked against c, then ours set
    ref.manual_threshold = thr
    c = dict(c, threshold=thr)
    mod = _load_h15_tokenizer_module()
    tok = _new(mod.HCodecTokenizer)
    tok.config = reference_kwargs(o15.h15_shallow())
    tok.model, tok.feature_extractor, tok.hop_length = ref, _StatesAt(hf_model(wc, fsd), wc["hidden_state_ids"]), HOP
    with torch.no_grad():
        padded_r = tok.pad_wav(wav)
        feats_r = tok.extract_wav2vec2_features(padded_r)
        out_r = tok.tokenize(wav)
        ac_r, sc_r = out_r["acoustic_codes"], out_r["semantic_codes"]
        rec_r = tok.detokenize(**out_r)
    taps = {}
    ac_o, sc_o = o15.codec_encode(sd, c, padded_o[:, None], feats_o.transpose(1, 2), taps)
    rec_o = o15.codec_decode(sd, c, ac_r, sc_r)
    K = c["codebook_size"]
    _, lens_r = ad.extract_lengths(ac_r, K)
    lens_o = ad.token_lengths(taps["align"])
    real = lens_r[lens_r > 0]
    margin = float((sim - thr).abs().min())
    report = dict(batch=int(wav.shape[0]), samples=int(wav.shape[1]), padded=int(padded_r.shape[1]), threshold=thr,
                  padded_equal=bool(torch.equal(padded_r, padded_o)), feature_frames=int(feats_r.shape[1]),
                  feats_rel_away_from_zero=feats_away_from_zero(feats_o, feats_r),
                  token_lengths_identical=bool(torch.equal(lens_r, lens_o)), groups_per_item=taps["n_groups"].tolist(),
                  token_length_histogram=torch.bincount(real, minlength=9).tolist(),
                  single_frame_tokens=int((real == 1).sum()), merged_tokens=int((real >= 2).sum()), capped_tokens=int((real == 8).sum()),
                  min_abs_similarity_minus_threshold=margin,
                  acoustic_identical=bool(torch.equal(ac_r, ac_o)), semantic_identical=bool(torch.equal(sc_r, sc_o)),
                  rec_rel=rel(rec_o.reshape(rec_r.shape), rec_r), codes_shape=list(ac_r.shape), rec_shape=list(rec_r.shape))
    print("h15", report)
    assert report["padded_equal"] and report["feats_rel_away_from_zero"] < 1e-4 and report["token_lengths_identical"]
    assert report["acoustic_identical"] and report["semantic_identical"] and report["rec_rel"] < 1e-5
    assert report["single_frame_tokens"] > 0 and report["merged_tokens"] > 0 and report["capped_tokens"] > 0 and margin > 5e-3
    arrays = dict(h15_padded_len=torch.tensor(padded_r.shape[-1]), h15_feats=feats_r, h15_acoustic=ac_r,
                  h15_semantic=sc_r, h15_token_lengths=lens_r, h15_seg=taps["align"].argmax(1), h15_rec=rec_r)
    return report, arrays


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    r1, a1 = run_h1()
    r15, a15 = run_h15()
    meta = dict(seeds=SEEDS, hubert=hubert_cfg(), wav2vec2=wav2vec2_cfg(), h15_threshold=r15["threshold"], hop=HOP,
                h1_clips=H1_CLIPS, h15_clips=H15_CLIPS, h1_trim=H1_TRIM, h15_trim=H15_TRIM,
                reference="QuarkAudio-HCodec/HCodec-1.0/audio_tokenizer.py:18-66 and HCodec-1.5/audio_tokenizer.py:38-86 "
                          "(unmodified pad_wav / extract_wav2vec2_features / tokenize / detokenize)")
    path = os.path.join(GOLD, "hcodec_tokenizers_small.npz")
    np.savez_compressed(path, meta=np.array(json.dumps(meta)), **{k: v.numpy() for k, v in {**a1, **a15}.items()})
    json.dump(dict(h1=r1, h15=r15), open(os.path.join(GOLD, "hcodec_tokenizers_pinning_report.json"), "w"), indent=1)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
