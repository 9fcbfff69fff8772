"""H-Codec-1.0 / 1.5 tokenizers on the GPU (`HCodecTokenizerH1`, `HCodecTokenizerH15`) against the reference tokenizers' own
outputs (tests/golden/hcodec_tokenizers_small.npz, written by oracle/make_golden_hcodec_tokenizers.py) and, at the shipped widths,
against the oracle chain (oracle/hcodec_features.py -> oracle/hcodec1.py / hcodec15.py)."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _decompress(y):
    return torch.sign(y) * y.abs() ** (1 / 0.3)


def _feature_errors(got, ref):
    """sign(x)|x|^0.3 has an infinite slope at 0: compare after undoing the compression, and directly away from zero"""
    got, ref = got.double().cpu(), ref.double().cpu()
    mean = _decompress(ref)
    big = mean.abs() > 1e-2 * mean.abs().max()
    return rel(_decompress(got), mean), float((got - ref).abs()[big].max() / ref.abs().max())


def _codebooks(sd, name, nq):
    return torch.stack([sd[f"{name}.layers.{i}._codebook.embed"][0] for i in range(nq)], 0)


def _fixture():
    z = np.load(os.path.join(GOLD, "hcodec_tokenizers_small.npz"))
    return z, json.loads(str(z["meta"]))


def _h1(hubert_cfg, seed_codec, seed_ssl):
    from oracle import hcodec1, hubert as oh
    from unified_audio_b200 import CodecH1, HCodecTokenizerH1, SSLFrontEnd
    sd, fsd = hcodec1.make_state_dict(hcodec1.H1, seed_codec), oh.make_state_dict(hubert_cfg, seed_ssl)
    codec = CodecH1({}, {}, {})
    codec.load_state_dict(sd, strict=True)
    fe = SSLFrontEnd(dict(hubert_cfg, kind="hubert"), in_rate=16000, compress=True)
    fe.load_state_dict(fsd, strict=True)
    return HCodecTokenizerH1(codec.cuda(), fe.cuda()), sd, fsd


def _h15(c, w2v_cfg, seed_codec, seed_ssl):
    from oracle import hcodec15 as o15, wav2vec2 as ow
    from unified_audio_b200 import CodecH15, HCodecTokenizerH15, SSLFrontEnd
    sd, fsd = o15.make_state_dict(c, seed_codec), ow.make_state_dict(w2v_cfg, seed_ssl)
    codec = CodecH15(_cfg={k: v for k, v in c.items() if k != "layer_scale"})
    codec.load_state_dict(sd, strict=True)
    fe = SSLFrontEnd(w2v_cfg, in_rate=16000, compress=True)
    fe.load_state_dict(fsd, strict=True)
    return HCodecTokenizerH15(codec.cuda(), fe.cuda()), sd, fsd


def _audit(tag, got, want, rows_got, rows_ref, codebooks):
    from oracle.parity import audit_codes
    a = audit_codes(got, want, rows_got, rows_ref, codebooks)
    print(f"  {tag}: {a}")
    assert a["explained"], f"{tag}: an index differs at a numerically safe decision"
    return a


def _rows(t):
    """[B, D, N] -> [B*N, D]"""
    return t.double().cpu().transpose(1, 2).reshape(-1, t.shape[1])


def _by_hand_h1(tok, wav, taps=None):
    """pad -> front end (channel-first) -> CodecH1.encode: the existing faces called one after the other"""
    from unified_audio_b200.ssl import pad_wav
    padded = pad_wav(wav, 640)
    return tok.model.encode(padded[:, None], tok.feature_extractor(padded, channel_first=True), taps=taps)


def _by_hand_h15(tok, wav, taps=None):
    from unified_audio_b200 import ops
    from unified_audio_b200.ssl import pad_wav
    padded = pad_wav(wav, 640)
    feats = tok.feature_extractor(ops.pad_wav(padded, 160, padded.shape[-1] + 320), channel_first=True)
    return tok.model.encode(padded[:, None], feats, taps=taps)


def test_h1_tokenizer_vs_reference_fixture(lib):
    from oracle import hcodec1
    from oracle.make_golden_hcodec_tokenizers import synth_clips
    z, meta = _fixture()
    s = meta["seeds"]
    tok, sd, _ = _h1(meta["hubert"], s["h1_codec"], s["h1_ssl"])
    wav = synth_clips(meta["h1_clips"], meta["h1_trim"], s["h1_wav"])
    padded = tok.pad_wav(wav.cuda())
    assert padded.shape[-1] == int(z["h1_padded_len"]) and torch.equal(padded.cpu(), torch.nn.functional.pad(wav, (0, padded.shape[-1] - wav.shape[-1])))
    feats = tok.extract_wav2vec2_features(padded)
    e_dec, e_big = _feature_errors(feats, torch.from_numpy(z["h1_feats"]))
    print(f"[h1 fixture] features: decompressed rel {e_dec:.2e}, direct away from zero {e_big:.2e}")
    assert feats.shape == z["h1_feats"].shape and max(e_dec, e_big) < TOL
    ac, sc = tok.tokenize(wav.cuda())
    want_a, want_s = torch.from_numpy(z["h1_acoustic"]), torch.from_numpy(z["h1_semantic"])
    assert ac.shape == want_a.shape == (2, 4, padded.shape[-1] // 640) and ac.dtype == torch.int64
    taps = {}
    _by_hand_h1(tok, wav.cuda(), taps)
    x = padded.cpu()[:, None]
    ref_feats = torch.from_numpy(z["h1_feats"]).transpose(1, 2)
    emb_ref, sem_ref = hcodec1.seanet_encoder(sd, hcodec1.H1, x), hcodec1.semantic_encoder(sd, hcodec1.H1, ref_feats)
    _audit("h1 fixture acoustic", ac, want_a, _rows(taps["enc.out"]), _rows(emb_ref), _codebooks(sd, "quantizer", 4))
    _audit("h1 fixture semantic", sc, want_s, _rows(taps["sem.out"]), _rows(sem_ref), _codebooks(sd, "semantic_quantizer", 4))
    rec = tok.detokenize(want_a.cuda(), want_s.cuda())
    e_wav = rel(rec, torch.from_numpy(z["h1_rec"]))
    print(f"[h1 fixture] detokenize of the reference's codes: rel {e_wav:.2e}")
    assert rec.shape == z["h1_rec"].shape and e_wav < TOL


def test_h15_tokenizer_vs_reference_fixture(lib):
    from oracle import adaptive as oad
    from oracle import hcodec15 as o15
    from oracle.make_golden_hcodec_tokenizers import synth_clips
    from unified_audio_b200 import WAV2VEC2_XLSR53_RAW
    z, meta = _fixture()
    s = meta["seeds"]
    c = dict(o15.h15_shallow(), threshold=meta["h15_threshold"])
    w2v = dict(WAV2VEC2_XLSR53_RAW, layers=meta["wav2vec2"]["layers"], hidden_state_ids=tuple(meta["wav2vec2"]["hidden_state_ids"]))
    tok, sd, _ = _h15(c, w2v, s["h15_codec"], s["h15_ssl"])
    wav = synth_clips(meta["h15_clips"], meta["h15_trim"], s["h15_wav"])
    padded = tok.pad_wav(wav.cuda())
    assert padded.shape[-1] == int(z["h15_padded_len"]) and torch.equal(padded.cpu(), torch.nn.functional.pad(wav, (0, padded.shape[-1] - wav.shape[-1])))
    feats = tok.extract_wav2vec2_features(padded)
    e_dec, e_big = _feature_errors(feats, torch.from_numpy(z["h15_feats"]))
    print(f"[h15 fixture] features: decompressed rel {e_dec:.2e}, direct away from zero {e_big:.2e}")
    assert feats.shape == z["h15_feats"].shape and max(e_dec, e_big) < TOL
    out = tok.tokenize(wav.cuda())
    assert set(out) == {"acoustic_codes", "semantic_codes"}
    taps = {}
    _by_hand_h15(tok, wav.cuda(), taps)
    K, nq = c["codebook_size"], c["nq"]
    margin = float((taps["sim"].cpu() - c["threshold"]).abs().min())
    print(f"[h15 fixture] groups per item {taps['n_groups'].tolist()}; closest similarity to the threshold {margin:.2e}")
    assert torch.equal(taps["seg"].cpu().long(), torch.from_numpy(z["h15_seg"])), "grouping differs from the reference"
    assert torch.equal(taps["token_lengths"].cpu(), torch.from_numpy(z["h15_token_lengths"]))
    otaps = {}
    o15.codec_encode(sd, c, padded.cpu()[:, None], torch.from_numpy(z["h15_feats"]).transpose(1, 2), otaps)
    for tag, key, qname, tap in (("acoustic", "acoustic_codes", "quantizer", "ac_agg.out"),
                                 ("semantic", "semantic_codes", "semantic_quantizer", "sem_agg.out")):
        got, want = out[key].cpu(), torch.from_numpy(z[f"h15_{tag}"])
        assert got.shape == want.shape and got.dtype == torch.int64
        gp, gl = oad.extract_lengths(got, K)
        wp, wl = oad.extract_lengths(want, K)
        assert torch.equal(gl, wl), "token lengths packed into the indices differ"
        _audit(f"h15 fixture {tag}", gp, wp, _rows(taps[tap]), _rows(otaps[tap]), _codebooks(sd, qname, nq))
    rec = tok.detokenize(torch.from_numpy(z["h15_acoustic"]).cuda(), torch.from_numpy(z["h15_semantic"]).cuda())
    e_wav = rel(rec, torch.from_numpy(z["h15_rec"]))
    print(f"[h15 fixture] detokenize of the reference's codes: rel {e_wav:.2e}")
    assert rec.shape == z["h15_rec"].shape and e_wav < TOL
    rec_l = tok.detokenize(*(oad.extract_lengths(torch.from_numpy(z[f"h15_{t}"]), K)[0].cuda() for t in ("acoustic", "semantic")),
                           token_lengths=torch.from_numpy(z["h15_token_lengths"]).cuda())
    assert torch.equal(rec_l, rec)


def test_tokenize_is_the_composition_of_the_faces(lib):
    """tokenize adds no arithmetic: bit-identical to pad -> front end -> encode called by hand, and to itself on a second call"""
    from oracle import hcodec15 as o15
    from oracle.make_golden_hcodec_tokenizers import synth_clips
    from unified_audio_b200 import WAV2VEC2_XLSR53_RAW
    z, meta = _fixture()
    s = meta["seeds"]
    tok1, _, _ = _h1(meta["hubert"], s["h1_codec"], s["h1_ssl"])
    wav = synth_clips(meta["h1_clips"], meta["h1_trim"], s["h1_wav"]).cuda()
    ac, sc = tok1.tokenize(wav)
    ha, hs = _by_hand_h1(tok1, wav)
    assert torch.equal(ac, ha) and torch.equal(sc, hs)
    ac2, sc2 = tok1.tokenize(wav)
    assert torch.equal(ac, ac2) and torch.equal(sc, sc2)
    c = dict(o15.h15_shallow(), threshold=meta["h15_threshold"])
    w2v = dict(WAV2VEC2_XLSR53_RAW, layers=meta["wav2vec2"]["layers"], hidden_state_ids=tuple(meta["wav2vec2"]["hidden_state_ids"]))
    tok15, _, _ = _h15(c, w2v, s["h15_codec"], s["h15_ssl"])
    wav = synth_clips(meta["h15_clips"], meta["h15_trim"], s["h15_wav"]).cuda()
    out = tok15.tokenize(wav)
    hand = _by_hand_h15(tok15, wav)
    assert all(torch.equal(out[k], hand[k]) for k in ("acoustic_codes", "semantic_codes"))
    feats = tok15.extract_wav2vec2_features(tok15.pad_wav(wav))
    torch.cuda.synchronize()
    assert feats.shape == (2, tok15.pad_wav(wav).shape[-1] // 320, 1024)
    with pytest.raises(ValueError, match=r"\[B, T\]"):
        tok15.tokenize(wav[:, None])
    with pytest.raises(RuntimeError, match="CUDA only"):
        tok1.tokenize(wav.cpu())


def test_h1_tokenizer_shipped_widths_vs_oracle(lib):
    """HUBERT_BASE + the CodecH1 default config, B = 2 x ~2 s, against the oracle chain"""
    from oracle import hcodec1, hubert as oh
    from oracle.hcodec_features import extract_hcodec1_features
    from unified_audio_b200 import HUBERT_BASE
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    tok, sd, fsd = _h1(HUBERT_BASE, 41, 42)
    g = torch.Generator().manual_seed(43)
    wav = 0.1 * torch.randn(2, 32000 - 123, generator=g)
    padded = torch.nn.functional.pad(wav, (0, 123))
    ref_feats = extract_hcodec1_features(fsd, oh.HUBERT_BASE, padded)
    feats = tok.extract_wav2vec2_features(tok.pad_wav(wav.cuda()))
    e_dec, e_big = _feature_errors(feats, ref_feats)
    print(f"[h1 shipped] features: decompressed rel {e_dec:.2e}, direct away from zero {e_big:.2e}")
    assert feats.shape == ref_feats.shape == (2, 100, 768) and max(e_dec, e_big) < TOL
    ac, sc = tok.tokenize(wav.cuda())
    taps = {}
    _by_hand_h1(tok, wav.cuda(), taps)
    oa, os_ = hcodec1.codec_encode(sd, hcodec1.H1, padded[:, None], ref_feats.transpose(1, 2))
    assert ac.shape == oa.shape == (2, 4, 50)
    emb_ref = hcodec1.seanet_encoder(sd, hcodec1.H1, padded[:, None])
    sem_ref = hcodec1.semantic_encoder(sd, hcodec1.H1, ref_feats.transpose(1, 2))
    _audit("h1 shipped acoustic", ac, oa, _rows(taps["enc.out"]), _rows(emb_ref), _codebooks(sd, "quantizer", 4))
    a = _audit("h1 shipped semantic", sc, os_, _rows(taps["sem.out"]), _rows(sem_ref), _codebooks(sd, "semantic_quantizer", 4))
    assert a["index_match_rate"] > 0.9
    rec = tok.detokenize(ac, sc)
    torch.cuda.synchronize()
    assert rec.shape == (2, 32000)


def test_h15_tokenizer_shipped_widths_vs_oracle(lib):
    """WAV2VEC2_XLSR53_RAW (16 of 24 layers computed) + the CodecH15 default config, B = 2 x ~2 s, against the oracle chain"""
    from oracle import adaptive as oad
    from oracle import hcodec15 as o15, wav2vec2 as ow
    from oracle.hcodec_features import extract_hcodec15_features
    from unified_audio_b200 import WAV2VEC2_XLSR53_RAW
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    c = o15.H15
    tok, sd, fsd = _h15(c, WAV2VEC2_XLSR53_RAW, 51, 52)
    g = torch.Generator().manual_seed(53)
    wav = 0.1 * torch.randn(2, 32000 - 301, generator=g)
    padded = torch.nn.functional.pad(wav, (0, 301))
    ref_feats = extract_hcodec15_features(fsd, ow.WAV2VEC2_XLSR53, padded)
    feats = tok.extract_wav2vec2_features(tok.pad_wav(wav.cuda()))
    e_dec, e_big = _feature_errors(feats, ref_feats)
    print(f"[h15 shipped] features: decompressed rel {e_dec:.2e}, direct away from zero {e_big:.2e}")
    assert feats.shape == ref_feats.shape == (2, 100, 1024) and max(e_dec, e_big) < TOL
    out = tok.tokenize(wav.cuda())
    taps, otaps = {}, {}
    _by_hand_h15(tok, wav.cuda(), taps)
    oa, osem = o15.codec_encode(sd, c, padded[:, None], ref_feats.transpose(1, 2), otaps)
    margin = float((taps["sim"].cpu() - c["threshold"]).abs().min())
    lens = oad.token_lengths(otaps["align"])
    print(f"[h15 shipped] groups per clip {otaps['n_groups'].tolist()} of 50 frames, token lengths "
          f"{torch.bincount(lens[lens > 0], minlength=9).tolist()}; closest similarity to the threshold {margin:.2e}")
    assert torch.equal(taps["seg"].cpu().long(), otaps["align"].argmax(1)), "grouping differs from the oracle"
    K, nq = c["codebook_size"], c["nq"]
    for tag, got, want, qname, key in (("acoustic", out["acoustic_codes"], oa, "quantizer", "ac_agg.out"),
                                       ("semantic", out["semantic_codes"], osem, "semantic_quantizer", "sem_agg.out")):
        assert got.shape == want.shape and got.dtype == torch.int64
        gp, gl = oad.extract_lengths(got.cpu(), K)
        wp, wl = oad.extract_lengths(want, K)
        assert torch.equal(gl, wl)
        a = _audit(f"h15 shipped {tag}", gp, wp, _rows(taps[key]), _rows(otaps[key]), _codebooks(sd, qname, nq))
        assert a["index_match_rate"] > 0.9
    rec = tok.detokenize(out["acoustic_codes"], out["semantic_codes"])
    torch.cuda.synchronize()
    assert rec.shape == (2, 32000)
