"""H-Codec-1.5 adaptive frame-rate codec (SURVEY.md 8f.4) on the GPU against the golden outputs of the reference's own modules
(tests/golden/h15_*.npz, written by oracle/make_golden_h15.py) and against the oracle's intermediate taps."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3


# the hyper-parameters of HCodec-1.5/conf/config_adaptive_v3.yaml that the reference's constructors read
_AGG = dict(dim=512, in_out_dim=512, num_heads=8, num_layers=32, dim_feedforward=2048, causal=False, use_mean_pooling_init=True,
            context_frames=16)
SHIPPED_CONFIG = dict(
    encoder_config=dict(encoder=dict(n_filters=32, dimension=512, ratios=[2, 4, 5, 8]),
                        semantic_encoder=dict(input_channels=1024, encode_channels=1024, out_channels=512, strides=[2, 1])),
    decoder_config=dict(decoder=dict(input_channels=1024, dim=1024, intermediate_dim=2304)),
    quantizer_config=dict(quantizer=dict(dim=512, codebook_size=1024, num_quantizers=4)),
    adaptive_config=dict(use_similarity_alignment=True, similarity_threshold=0.7, max_tokens_per_group=8, manual_threshold=0.6,
                         use_query_token_aggregator=True, use_bottleneck_transformer=True,
                         aggregators=dict(semantic_aggregator=dict(_AGG), acoustic_aggregator=dict(_AGG)),
                         transformer_kwargs=dict(d_model=1024, num_heads=8, num_layers=32, causal=False, layer_scale=0.01, context=16,
                                                 conv_layout=True, gating="none", norm="layer_norm", positional_embedding="rope",
                                                 dim_feedforward=2048, input_dimension=1024, output_dimensions=[1024])))


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _setup(name, precision):
    from oracle import hcodec15 as o15
    from oracle.make_golden_h15 import synth
    from unified_audio_b200.codec_h15 import CodecH15
    z = np.load(os.path.join(GOLD, f"h15_{name}.npz"))
    meta = json.loads(str(z["meta"]))
    c = o15.h15_shallow() if name == "shallow" else o15.H15
    sd = o15.make_state_dict(c, meta["seed_w"])
    cfg = {k: v for k, v in c.items() if k != "layer_scale"}
    m = CodecH15(precision=precision, _cfg=cfg)
    m.load_state_dict(sd, strict=True)
    wav, feat = synth(c, meta["batch"], meta["frames"], meta["seed_x"])
    return z, c, sd, m.cuda(), wav, feat


def _codebooks(sd, name, nq):
    return torch.stack([sd[f"{name}.layers.{i}._codebook.embed"][0] for i in range(nq)], 0)


@pytest.mark.parametrize("name,precision", [("shallow", "mixed"), ("shallow", "accurate"), ("full", "mixed")])
def test_h15_encode_decode_against_reference_golden(lib, name, precision):
    from oracle import adaptive as oad
    from oracle.parity import audit_codes
    z, c, sd, m, wav, feat = _setup(name, precision)
    B, K, nq = wav.shape[0], c["codebook_size"], c["nq"]
    taps = {}
    out = m.encode(wav.cuda(), feat.cuda(), taps=taps)
    torch.cuda.synchronize()
    e_emb, e_sem = rel(taps["enc.out"], torch.from_numpy(z["emb"])), rel(taps["sem.out"], torch.from_numpy(z["sem"]))
    print(f"[h15 {name}/{precision}] emb rel {e_emb:.2e} sem rel {e_sem:.2e}")
    assert e_emb < TOL and e_sem < TOL
    # grouping: the frame -> token map must reproduce the reference's alignment matrix (a flip needs a cosine similarity within
    # float error of the threshold; report the closest one)
    align = torch.from_numpy(z["align"]).float()
    seg_ref = align.argmax(1)
    margin = float((taps["sim"].cpu() - c["threshold"]).abs().min())
    print(f"[h15 {name}] groups per item {taps['n_groups'].tolist()} (reference {z['n_groups'].tolist()}); closest similarity to the "
          f"threshold: {margin:.2e}")
    assert torch.equal(taps["seg"].cpu().long(), seg_ref), "grouping differs from the reference"
    assert torch.equal(taps["n_groups"].cpu(), torch.from_numpy(z["n_groups"]))
    assert torch.equal(taps["token_lengths"].cpu(), oad.token_lengths(align))
    e_st, e_at = rel(taps["sem_agg.out"], torch.from_numpy(z["sem_tok"])), rel(taps["ac_agg.out"], torch.from_numpy(z["ac_tok"]))
    print(f"[h15 {name}/{precision}] aggregator tokens: semantic rel {e_st:.2e} acoustic rel {e_at:.2e}")
    assert e_st < TOL and e_at < TOL
    G = align.shape[1]
    for tag, key, qname, tok_key, tok_ref in (("acoustic", "acoustic_codes", "quantizer", "ac_agg.out", "ac_tok"),
                                              ("semantic", "semantic_codes", "semantic_quantizer", "sem_agg.out", "sem_tok")):
        got, want = out[key].cpu(), torch.from_numpy(z[key])
        assert got.shape == want.shape == (B, nq, G) and got.dtype == torch.int64
        gp, gl = oad.extract_lengths(got, K)
        wp, wl = oad.extract_lengths(want, K)
        assert torch.equal(gl, wl), "token lengths packed into the indices differ"
        rows = lambda t: t.double().cpu().transpose(1, 2).reshape(B * G, -1)
        a = audit_codes(gp, wp, rows(taps[tok_key]), rows(torch.from_numpy(z[tok_ref])), _codebooks(sd, qname, nq))
        print(f"[h15 {name}/{precision}] {tag}: {a}")
        assert a["explained"], f"{tag} index differs at a numerically safe decision"
        assert a["index_match_rate"] > 0.97
    # decode the REFERENCE's codes
    dtaps = {}
    rec = m.decode(torch.from_numpy(z["acoustic_codes"]).cuda(), torch.from_numpy(z["semantic_codes"]).cuda(), taps=dtaps)
    torch.cuda.synchronize()
    assert rel(dtaps["dec.z"], torch.from_numpy(z["z"])) < 1e-6
    e_bn, e_wav = rel(dtaps["bottleneck.out"], torch.from_numpy(z["bottleneck"])), rel(rec, torch.from_numpy(z["wav_rec"]))
    print(f"[h15 {name}/{precision}] bottleneck rel {e_bn:.2e} wav rel {e_wav:.2e}")
    assert rec.shape == tuple(z["wav_rec"].shape)
    assert e_bn < TOL and e_wav < TOL


def test_h15_taps_vs_oracle_and_reference_surface(lib):
    """layer-level taps of the aggregator / bottleneck stacks against the oracle; constructor from the reference's config blocks"""
    from oracle import hcodec15 as o15
    from unified_audio_b200.codec_h15 import CodecH15, H15, config_from_kwargs
    z, c, sd, m, wav, feat = _setup("shallow", "mixed")
    otaps, gtaps = {}, {}
    o15.codec_encode(sd, c, wav, feat, otaps)
    m.encode(wav.cuda(), feat.cuda(), taps=gtaps)
    for k in ("sem_agg.interleaved", "sem_agg.layer0", f"sem_agg.layer{c['agg']['layers'] - 1}", "ac_agg.interleaved", "ac_agg.layer0"):
        e = rel(gtaps[k], otaps[k])
        print(f"  tap {k}: {e:.2e}")
        assert e < TOL
    # threshold argument (codec_adaptive.py:153-161): a higher threshold merges less
    out_hi = m.encode(wav.cuda(), feat.cuda(), threshold=0.95)
    oa, _ = o15.codec_encode(sd, c, wav, feat, threshold=0.95)
    assert out_hi["acoustic_codes"].shape == oa.shape
    with pytest.raises(ValueError):
        m.encode(wav.cuda(), feat.cuda(), threshold=1.5)
    y = SHIPPED_CONFIG
    cfg = config_from_kwargs(y["encoder_config"], y["decoder_config"], y["quantizer_config"], y["adaptive_config"])
    assert cfg == {k: v for k, v in H15.items()}
    full = CodecH15(y["encoder_config"], y["decoder_config"], y["quantizer_config"], y["adaptive_config"])
    assert set(full.state_dict()) == set(o15.param_specs(o15.H15))


def test_h15_bench_shape_vs_oracle(lib):
    """the shipped config at the bench leg's clip length (10 s -> 250 frames, T + G ~ 350 rows per aggregator sequence), 2 clips,
    bench-style inputs, against the oracle on the same weights: every float tap < 1e-3, grouping identical, indices audited"""
    from oracle import adaptive as oad
    from oracle import hcodec15 as o15
    from oracle.make_golden_h15 import synth
    from oracle.parity import audit_codes
    from unified_audio_b200.codec_h15 import CodecH15
    c = o15.H15
    sd = o15.make_state_dict(c, 31)
    m = CodecH15(precision="mixed", _cfg={k: v for k, v in c.items() if k != "layer_scale"})
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    B, N = 2, 250
    wav, feat = synth(c, B, N, 32)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    otaps, gtaps = {}, {}
    oa, osem = o15.codec_encode(sd, c, wav, feat, otaps)
    out = m.encode(wav.cuda(), feat.cuda(), taps=gtaps)
    torch.cuda.synchronize()
    align = otaps["align"]
    assert torch.equal(gtaps["seg"].cpu().long(), align.argmax(1)), "grouping differs from the oracle"
    G = align.shape[1]
    print(f"[h15 bench shape] groups per clip {otaps['n_groups'].tolist()} of {N} frames; sequences of {N + G} rows")
    for k in ("enc.out", "sem.out", "sem_agg.layer0", "sem_agg.layer31", "ac_agg.layer31", "sem_agg.out", "ac_agg.out"):
        e = rel(gtaps[k], otaps[k])
        print(f"  [h15 bench shape] tap {k}: {e:.2e}")
        assert e < TOL
    K, nq = c["codebook_size"], c["nq"]
    rows = lambda t: t.double().cpu().transpose(1, 2).reshape(B * G, -1)
    for tag, got, want, qname, key in (("acoustic", out["acoustic_codes"], oa, "quantizer", "ac_agg.out"),
                                       ("semantic", out["semantic_codes"], osem, "semantic_quantizer", "sem_agg.out")):
        gp, gl = oad.extract_lengths(got.cpu(), K)
        wp, wl = oad.extract_lengths(want, K)
        assert torch.equal(gl, wl)
        a = audit_codes(gp, wp, rows(gtaps[key]), rows(otaps[key]), _codebooks(sd, qname, nq))
        print(f"[h15 bench shape] {tag}: {a}")
        assert a["explained"] and a["index_match_rate"] > 0.97
    dt_o, dt_g = {}, {}
    ref = o15.codec_decode(sd, c, oa, osem, dt_o)
    rec = m.decode(oa.cuda(), osem.cuda(), taps=dt_g)
    torch.cuda.synchronize()
    for k in ("bottleneck.layer0", "bottleneck.out", "dec.tf", "dec.post"):
        e = rel(dt_g[k], dt_o[k])
        print(f"  [h15 bench shape] tap {k}: {e:.2e}")
        assert e < TOL
    e_wav = rel(rec, ref)
    print(f"[h15 bench shape] wav rel {e_wav:.2e}")
    assert rec.shape == ref.shape == (B, N * 640) and e_wav < TOL


def _shallow_codec():
    from oracle import hcodec15 as o15
    from unified_audio_b200.codec_h15 import CodecH15
    c = o15.h15_shallow()
    sd = o15.make_state_dict(c, 11)
    m = CodecH15(precision="mixed", _cfg={k: v for k, v in c.items() if k != "layer_scale"})
    m.load_state_dict(sd, strict=True)
    return c, sd, m.cuda()


def _agg_taps(c):
    last = c["agg"]["layers"] - 1
    return [f"{a}.{k}" for a in ("sem_agg", "ac_agg") for k in ("interleaved", "layer0", f"layer{last}", "out")]


def test_h15_one_frame_clips(lib):
    """640 samples per clip (the shortest clip the tokenizer makes: it pads anything up to 640 samples to that) give one frame and
    one token per clip: the frame -> token map handed to the aggregator kernels is int32 zeros, every tap matches the oracle, the
    packed codes equal the oracle's and decode of them matches the oracle's decode.  The seed keeps every RVQ decision at least
    5e-4 |token| from a tie."""
    from oracle import hcodec15 as o15
    from oracle.make_golden_h15 import synth
    c, sd, m = _shallow_codec()
    wav, feat = synth(c, 2, 1, 62)
    assert wav.shape == (2, 1, 640)
    otaps, gtaps = {}, {}
    oa, osem = o15.codec_encode(sd, c, wav, feat, otaps)
    out = m.encode(wav.cuda(), feat.cuda(), taps=gtaps)
    torch.cuda.synchronize()
    seg = gtaps["seg"]
    assert seg.dtype == torch.int32 and tuple(seg.shape) == (2, 1) and not bool(seg.any())
    assert gtaps["n_groups"].tolist() == [1, 1] and gtaps["token_lengths"].tolist() == [[1], [1]]
    for k in ["enc.out", "sem.out"] + _agg_taps(c):
        e = rel(gtaps[k], otaps[k])
        print(f"  [h15 one frame] tap {k}: {e:.2e}")
        assert e < TOL
    assert torch.equal(out["acoustic_codes"].cpu(), oa) and torch.equal(out["semantic_codes"].cpu(), osem)
    rec = m.decode(out["acoustic_codes"], out["semantic_codes"])
    torch.cuda.synchronize()
    ref = o15.codec_decode(sd, c, oa, osem)
    e_wav = rel(rec, ref)
    print(f"[h15 one frame] codes {oa[:, :, 0].tolist()}, wav rel {e_wav:.2e}")
    assert rec.shape == ref.shape == (2, 640) and e_wav < TOL


def _grouping_spread_inputs(c, N, seed):
    """B = 3 clips of N frames whose features group very differently: clip 0 constant over time (its interior semantic frames are
    identical and merge up to the cap), clip 1 random, clip 2 constant for the first half and random for the second"""
    from oracle.make_golden_h15 import synth
    wav, feat = synth(c, 3, N, seed)
    g = torch.Generator().manual_seed(seed + 1)
    T50 = 2 * N
    col = torch.randn(c["sem_in"], 1, generator=g)
    r = torch.randn(c["sem_in"], T50, generator=g)
    feat[0] = (torch.sign(col) * col.abs() ** 0.3).expand(-1, T50)
    feat[1] = torch.sign(r) * r.abs() ** 0.3
    feat[2, :, : T50 // 2] = feat[0, :, : T50 // 2]
    feat[2, :, T50 // 2:] = feat[1, :, T50 // 2:]
    return wav, feat


def test_h15_batch_with_padded_groups(lib):
    """a batch whose clips have 3, 24 and about 14 tokens of 24 frames: the shorter clips carry padded groups (query rows that are
    the bare embedding on the way in, zero tokens on the way out, length 0 packed as negative codes).  Grouping identical to the
    oracle, every aggregator tap < 1e-3, the packed codes equal the oracle's (the seed keeps every RVQ decision of a live group at
    least 1.8e-4 |token| from a tie, and every similarity 0.07 from the threshold) and decode of the oracle's codes < 1e-3."""
    from oracle import adaptive as oad
    from oracle import hcodec15 as o15
    c, sd, m = _shallow_codec()
    N = 24
    wav, feat = _grouping_spread_inputs(c, N, 57)
    otaps, gtaps = {}, {}
    oa, osem = o15.codec_encode(sd, c, wav, feat, otaps)
    out = m.encode(wav.cuda(), feat.cuda(), taps=gtaps)
    torch.cuda.synchronize()
    align, ng = otaps["align"], otaps["n_groups"]
    G = align.shape[1]
    print(f"[h15 padded groups] groups per clip {ng.tolist()} of {N} frames")
    assert int(ng.max()) >= 3 * int(ng.min()) and int(ng.min()) < G
    assert torch.equal(gtaps["n_groups"].cpu(), ng)
    assert torch.equal(gtaps["seg"].cpu().long(), align.argmax(1)), "grouping differs from the oracle"
    assert torch.equal(gtaps["token_lengths"].cpu(), oad.token_lengths(align))
    for k in ["enc.out", "sem.out"] + _agg_taps(c):
        e = rel(gtaps[k], otaps[k])
        print(f"  [h15 padded groups] tap {k}: {e:.2e}")
        assert e < TOL
    pad = torch.arange(G)[None] >= ng[:, None]
    for t in ("sem_agg.out", "ac_agg.out"):
        assert not bool(gtaps[t].cpu().transpose(1, 2)[pad].any()), f"{t}: padded groups must be zero tokens"
    assert bool((oa.transpose(1, 2)[pad] < 0).all())
    assert torch.equal(out["acoustic_codes"].cpu(), oa) and torch.equal(out["semantic_codes"].cpu(), osem)
    rec = m.decode(oa.cuda(), osem.cuda())
    torch.cuda.synchronize()
    ref = o15.codec_decode(sd, c, oa, osem)
    e_wav = rel(rec, ref)
    print(f"[h15 padded groups] wav rel {e_wav:.2e}")
    assert rec.shape == ref.shape == (3, N * 640) and e_wav < TOL
