"""H-Codec-1.0 / 1.5 tokenizer faces without a GPU: the oracle chain reproduces the reference tokenizers' fixture
(tests/golden/hcodec_tokenizers_small.npz, written by oracle/make_golden_hcodec_tokenizers.py from the reference's own classes),
the constructors refuse front ends that would give wrong codes, bad input is refused, and the package exports the faces."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _fixture():
    z = np.load(os.path.join(GOLD, "hcodec_tokenizers_small.npz"))
    return z, json.loads(str(z["meta"]))


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max())


def _away_from_zero(got, ref):
    big = ref.abs() > 0.2 * ref.abs().max()
    return float((got - ref).abs()[big].max() / ref.abs().max())


def test_oracle_chain_reproduces_reference_tokenizers():
    from oracle import adaptive as ad
    from oracle import hcodec1, hcodec15 as o15, hubert as oh, wav2vec2 as ow
    from oracle.hcodec_features import extract_hcodec1_features, extract_hcodec15_features
    from oracle.make_golden_hcodec_tokenizers import synth_clips
    z, meta = _fixture()
    s = meta["seeds"]
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    # H-Codec-1.0
    wav = synth_clips(meta["h1_clips"], meta["h1_trim"], s["h1_wav"])
    padded = torch.nn.functional.pad(wav, (0, -wav.shape[-1] % meta["hop"]))
    assert padded.shape[-1] == int(z["h1_padded_len"])
    hc = meta["hubert"]
    feats = extract_hcodec1_features(oh.make_state_dict(hc, s["h1_ssl"]), hc, padded)
    ref = torch.from_numpy(z["h1_feats"])
    assert feats.shape == ref.shape == (2, padded.shape[-1] // 320, 768) and _away_from_zero(feats, ref) < 1e-4
    sd = hcodec1.make_state_dict(hcodec1.H1, s["h1_codec"])
    ac, sc = hcodec1.codec_encode(sd, hcodec1.H1, padded[:, None], ref.transpose(1, 2))
    assert torch.equal(ac, torch.from_numpy(z["h1_acoustic"])) and torch.equal(sc, torch.from_numpy(z["h1_semantic"]))
    rec = hcodec1.codec_decode(sd, hcodec1.H1, ac, sc)
    assert _rel(rec.reshape(z["h1_rec"].shape), torch.from_numpy(z["h1_rec"])) < 1e-5
    # H-Codec-1.5
    wav = synth_clips(meta["h15_clips"], meta["h15_trim"], s["h15_wav"])
    padded = torch.nn.functional.pad(wav, (0, -wav.shape[-1] % meta["hop"]))
    assert padded.shape[-1] == int(z["h15_padded_len"])
    wc = meta["wav2vec2"]
    feats = extract_hcodec15_features(ow.make_state_dict(wc, s["h15_ssl"]), wc, padded)
    ref = torch.from_numpy(z["h15_feats"])
    assert feats.shape == ref.shape == (2, padded.shape[-1] // 320, 1024) and _away_from_zero(feats, ref) < 1e-4
    c = dict(o15.h15_shallow(), threshold=meta["h15_threshold"])
    sd = o15.make_state_dict(c, s["h15_codec"])
    taps = {}
    ac, sc = o15.codec_encode(sd, c, padded[:, None], ref.transpose(1, 2), taps)
    assert torch.equal(taps["align"].argmax(1), torch.from_numpy(z["h15_seg"]))
    assert torch.equal(ad.token_lengths(taps["align"]), torch.from_numpy(z["h15_token_lengths"]))
    assert torch.equal(ac, torch.from_numpy(z["h15_acoustic"])) and torch.equal(sc, torch.from_numpy(z["h15_semantic"]))
    rec = o15.codec_decode(sd, c, ac, sc)
    assert _rel(rec.reshape(z["h15_rec"].shape), torch.from_numpy(z["h15_rec"])) < 1e-5
    # the fixture exercises the adaptive path: single-frame tokens, merged tokens and the 8-frame cap
    lens = torch.from_numpy(z["h15_token_lengths"])
    assert int((lens == 1).sum()) > 0 and int((lens >= 2).sum()) > 0 and int((lens == c["max_group"]).sum()) > 0


def _small_codecs():
    from oracle import hcodec15 as o15
    from unified_audio_b200 import CodecH1, CodecH15
    h15 = {k: v for k, v in o15.h15_shallow().items() if k != "layer_scale"}
    return CodecH1({}, {}, {}), CodecH15(_cfg=h15)


def _hubert(**kw):
    from unified_audio_b200 import HUBERT_BASE, SSLFrontEnd
    kw.setdefault("in_rate", 16000)
    kw.setdefault("compress", True)
    return SSLFrontEnd(dict(HUBERT_BASE, layers=1, **kw.pop("cfg", {})), **kw)


def _w2v(**kw):
    from unified_audio_b200 import WAV2VEC2_XLSR53_RAW, SSLFrontEnd
    kw.setdefault("in_rate", 16000)
    kw.setdefault("compress", True)
    cfg = dict(WAV2VEC2_XLSR53_RAW, layers=2, hidden_state_ids=(1,))
    cfg.update(kw.pop("cfg", {}))
    return SSLFrontEnd(cfg, **kw)


def test_constructors_check_the_front_end():
    from unified_audio_b200 import HCodecTokenizerH1, HCodecTokenizerH15
    h1, h15 = _small_codecs()
    tok1, tok15 = HCodecTokenizerH1(h1, _hubert()), HCodecTokenizerH15(h15, _w2v())
    assert tok1.hop_length == 640 and tok15.hop_length == 640
    bad_h1 = [("wav2vec2", lambda: HCodecTokenizerH1(h1, _w2v(cfg=dict(hidden=768, heads=12, ffn=3072)))),
              ("in_rate", lambda: HCodecTokenizerH1(h1, _hubert(in_rate=48000))),
              ("compress", lambda: HCodecTokenizerH1(h1, _hubert(compress=False))),
              ("hidden width", lambda: HCodecTokenizerH1(h1, _hubert(cfg=dict(hidden=512, heads=8, ffn=2048)))),
              ("CodecH1", lambda: HCodecTokenizerH1(h15, _hubert()))]
    bad_h15 = [("hubert", lambda: HCodecTokenizerH15(h15, _hubert(cfg=dict(hidden=1024, heads=16, ffn=4096)))),
               ("in_rate", lambda: HCodecTokenizerH15(h15, _w2v(in_rate=48000))),
               ("compress", lambda: HCodecTokenizerH15(h15, _w2v(compress=False))),
               ("normalisation", lambda: HCodecTokenizerH15(h15, _w2v(cfg=dict(do_normalize=True)))),
               ("hidden width", lambda: HCodecTokenizerH15(h15, _w2v(cfg=dict(hidden=768, heads=12, ffn=3072)))),
               ("CodecH15", lambda: HCodecTokenizerH15(h1, _w2v()))]
    for what, make in bad_h1 + bad_h15:
        with pytest.raises(ValueError, match=what):
            make()


def test_bad_input_is_refused_before_the_device():
    from unified_audio_b200 import HCodecTokenizerH1, HCodecTokenizerH15
    h1, h15 = _small_codecs()
    for tok in (HCodecTokenizerH1(h1, _hubert()), HCodecTokenizerH15(h15, _w2v())):
        for wav in (torch.zeros(640), torch.zeros(1, 1, 640)):
            with pytest.raises(ValueError, match=r"\[B, T\]"):
                tok.tokenize(wav)
            with pytest.raises(ValueError, match=r"\[B, T\]"):
                tok.extract_wav2vec2_features(wav)
        with pytest.raises(RuntimeError, match="CUDA only"):
            tok.tokenize(torch.zeros(1, 640))
        with pytest.raises(RuntimeError, match="CUDA only"):
            tok.extract_wav2vec2_features(torch.zeros(1, 640))


def test_package_exports_the_faces():
    import unified_audio_b200 as ua
    from unified_audio_b200 import ssl
    assert ua.HCodecTokenizerH1 is ssl.HCodecTokenizerH1 and ua.HCodecTokenizerH15 is ssl.HCodecTokenizerH15
    assert ua.WAV2VEC2_XLSR53_RAW == dict(ua.WAV2VEC2_XLSR53, do_normalize=False)
    assert ua.WAV2VEC2_XLSR53["do_normalize"] is True                   # BiCodec's front end is unchanged
