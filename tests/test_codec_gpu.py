"""GPU parity of unified_audio_b200.Codec (through the C ABI) against the CPU oracle and the golden
fixtures generated from the reference's own modules (oracle/make_golden.py)."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3     # north_star: floats within 1e-3 relative


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def build(cfg, seed, precision):
    from oracle import weights
    from unified_audio_b200.codec import Codec
    sd = weights.make_h2_state_dict(cfg, seed)
    m = Codec(cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"],
              cfg["semantic_decoder_config"], precision=precision)
    missing, unexpected = m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def golden(name):
    z = np.load(os.path.join(GOLD, f"h2_{name}.npz"))
    meta = json.loads(str(z["meta"]))
    return z, meta


def check_codes(tag, got, want, x_rows, codebooks):
    """indices must equal the oracle's wherever the fp64 margin of the decision is numerically safe"""
    from oracle import rvq
    B, nq, N = want.shape
    got_r = got.cpu().transpose(1, 2).reshape(B * N, nq)
    want_r = want.transpose(1, 2).reshape(B * N, nq)
    _, margin = rvq.rvq_margin_audit(x_rows, codebooks, want_r)
    first_bad = torch.full((B * N,), nq, dtype=torch.long)
    for q in range(nq - 1, -1, -1):
        first_bad[got_r[:, q] != want_r[:, q]] = q
    n_tok_bad = int((first_bad < nq).sum())
    worst = [float(margin[i, first_bad[i]]) for i in range(B * N) if first_bad[i] < nq]
    print(f"[{tag}] tokens with a differing index: {n_tok_bad}/{B*N}; margins at first divergence: {worst[:8]}")
    return n_tok_bad, worst


@pytest.mark.parametrize("name,precision", [("small", "accurate"), ("small", "mixed"), ("mid", "mixed")])
def test_h2_golden(lib, name, precision):
    from oracle import hcodec2, weights
    z, meta = golden(name)
    cfg = meta["cfg"]
    model, sd = build(cfg, meta["seed_w"], precision)
    wav, feat = weights.synth_inputs(cfg, meta["batch"], meta["n_tokens"], meta["seed_x"])
    # stage-wise taps vs the oracle (diagnostic + assertion)
    otaps = {}
    hcodec2.codec_encode(sd, cfg, wav, feat, taps=otaps)
    gtaps = {}
    ac, sc = model.encode(wav.cuda(), feat.cuda(), taps=gtaps)
    torch.cuda.synchronize()
    for k in otaps:
        if k in gtaps:
            a, b = gtaps[k].float().cpu(), otaps[k]
            if k == "enc.feat":   # conditioning-aware metric (tests/test_bench_shape_gpu.py::feat_tap_error), asserted
                from oracle.parity import feat_tap_error
                assert feat_tap_error(a, b) < TOL
            else:
                print(f"  tap {k}: max-rel {rel(a, b):.2e}  l2-rel {l2(a, b):.2e}")
                assert rel(a, b) < TOL, f"tap {k}"
    emb_ref, sem_ref = torch.from_numpy(z["emb"]), torch.from_numpy(z["sem"])
    e_emb, e_sem = rel(gtaps["enc.out"], emb_ref), rel(gtaps["sem.out"], sem_ref)
    print(f"[{name}/{precision}] emb rel {e_emb:.2e} sem rel {e_sem:.2e}")
    assert e_emb < TOL and e_sem < TOL
    # codes: RVQ on the ORACLE embedding must be bit-exact; end-to-end codes reported with margins
    B, D, N = emb_ref.shape
    cb_a, cb_s = hcodec2._codebooks(sd, "quantizer"), hcodec2._codebooks(sd, "semantic_quantizer")
    rows_a = emb_ref.transpose(1, 2).reshape(B * N, D)
    ia, _ = model.quantizer.encode_rows(rows_a.cuda())
    want_a = torch.from_numpy(z["acoustic_codes"])
    nbad, worst = check_codes("rvq on oracle emb", ia.reshape(B, N, -1).transpose(1, 2), want_a, rows_a, cb_a)
    assert nbad == 0 or max(worst) < 1e-5
    # end-to-end codes: every index equal to the reference's, or explained by the embedding tolerance (oracle/parity.py)
    from oracle.parity import audit_codes
    grow = lambda t: t.float().cpu().transpose(1, 2).reshape(B * N, D)
    for tag, got, want, g_, o_, cb in (("acoustic", ac, want_a, gtaps["enc.out"], emb_ref, cb_a),
                                       ("semantic", sc, torch.from_numpy(z["semantic_codes"]), gtaps["sem.out"], sem_ref, cb_s)):
        a_ = audit_codes(got, want, grow(g_), grow(o_), cb)
        print(f"[{name}/{precision}] end-to-end {tag} codes: {a_}")
        assert a_["explained"], f"{tag}: index differs beyond the reach of the embedding tolerance"
    # decode from the reference's codes
    dtaps, odtaps = {}, {}
    rec = model.decode(want_a.cuda(), torch.from_numpy(z["semantic_codes"]).cuda(), taps=dtaps)
    torch.cuda.synchronize()
    hcodec2.codec_decode(sd, cfg, want_a, torch.from_numpy(z["semantic_codes"]), taps=odtaps)
    for k in odtaps:
        if k in dtaps:
            print(f"  tap {k}: max-rel {rel(dtaps[k].float(), odtaps[k]):.2e}  l2-rel {l2(dtaps[k].float(), odtaps[k]):.2e}")
    e_wav = rel(rec, torch.from_numpy(z["wav_rec"]))
    print(f"[{name}/{precision}] wav rel {e_wav:.2e}  l2 {l2(rec, torch.from_numpy(z['wav_rec'])):.2e}")
    assert rec.shape == z["wav_rec"].shape
    assert e_wav < TOL


def test_h2_full_config_vs_oracle(lib):
    """Shipped 48 kHz config (large_12.5hz_config.yaml), B=2 x 8 tokens, mixed precision policy."""
    from oracle import hcodec2, weights
    cfg = weights.H2_FULL
    model, sd = build(cfg, 0, "mixed")
    wav, feat = weights.synth_inputs(cfg, 2, 8, 2000)
    otaps, gtaps = {}, {}
    oa, os_ = hcodec2.codec_encode(sd, cfg, wav, feat, taps=otaps)
    ac, sc = model.encode(wav.cuda(), feat.cuda(), taps=gtaps)
    torch.cuda.synchronize()
    for k in otaps:
        if k in gtaps and k != "enc.feat":
            print(f"  tap {k}: max-rel {rel(gtaps[k].float(), otaps[k]):.2e}")
    assert rel(gtaps["enc.out"], otaps["enc.out"]) < TOL and rel(gtaps["sem.out"], otaps["sem.out"]) < TOL
    B, D, N = otaps["enc.out"].shape
    from oracle.parity import audit_codes
    grow = lambda t: t.float().cpu().transpose(1, 2).reshape(B * N, D)
    for tag, got, want, key, q in (("acoustic", ac, oa, "enc.out", "quantizer"), ("semantic", sc, os_, "sem.out", "semantic_quantizer")):
        a_ = audit_codes(got, want, grow(gtaps[key]), grow(otaps[key]), hcodec2._codebooks(sd, q))
        print(f"[full] end-to-end {tag} codes: {a_}")
        assert a_["explained"]
    rec = model.decode(oa.cuda(), os_.cuda())
    torch.cuda.synchronize()
    ref = hcodec2.codec_decode(sd, cfg, oa, os_)
    print(f"[full/mixed] wav rel {rel(rec, ref):.2e} l2 {l2(rec, ref):.2e}")
    assert rel(rec, ref) < TOL


def test_h2_ragged_sizes_vs_oracle(lib):
    """odd batch / token counts (partial M tiles, LSTM groups with < 32 rows, CTA-pair fallbacks), at the small config and at
    a mid-width one (512 channels, 16 quantisers of 1024 codes)"""
    from oracle import hcodec2, weights
    for widths, shapes in ((dict(), ((1, 1), (3, 5), (33, 2))),
                           (dict(dim=512, inter=1536, enc_layers=3, dec_layers=4, tf_layers=2, sem_ch=512, nq=16, cb=1024, qdim=512),
                            ((1, 4),))):
        cfg = weights.h2_small(**widths)
        model, sd = build(cfg, 5, "mixed")
        for B, ntok in shapes:
            wav, feat = weights.synth_inputs(cfg, B, ntok, 77 + B)
            oa, os_ = hcodec2.codec_encode(sd, cfg, wav, feat)
            emb = hcodec2.encoder_forward(sd, cfg["encoder_config"], wav)
            taps = {}
            ac, sc = model.encode(wav.cuda(), feat.cuda(), taps=taps)
            rec = model.decode(oa.cuda(), os_.cuda())
            torch.cuda.synchronize()
            ref = hcodec2.codec_decode(sd, cfg, oa, os_)
            print(f"[ragged dim={cfg['encoder_config']['dim']} B={B} N={ntok}] emb rel {rel(taps['enc.out'], emb):.2e} "
                  f"wav rel {rel(rec, ref):.2e} code match {float((ac.cpu() == oa).float().mean()):.4f}")
            assert rel(taps["enc.out"], emb) < TOL and rel(rec, ref) < TOL and rec.shape == (B, ntok * 3840)
            with pytest.raises(ValueError):
                model.encode(wav[:, :-1].cuda(), feat.cuda())          # length not a multiple of 3840 (pad_wav contract)


def test_h2_full_size_properties(lib):
    """BASELINE-size clips (10 s @ 48 kHz, shipped config): size-independent properties instead of a CPU oracle run -
    run-to-run determinism, batch invariance (clip i of a batch == the same clip alone), output length."""
    from oracle import weights
    cfg = weights.H2_FULL
    model, _ = build(cfg, 0, "mixed")
    B, ntok = 6, 125
    wav, feat = weights.synth_inputs(cfg, B, ntok, 4242)
    wav, feat = wav.cuda(), feat.cuda()
    ac1, sc1 = model.encode(wav, feat)
    rec1 = model.decode(ac1, sc1).clone()
    ac2, sc2 = model.encode(wav, feat)
    rec2 = model.decode(ac2, sc2)
    torch.cuda.synchronize()
    assert torch.equal(ac1, ac2) and torch.equal(sc1, sc2) and torch.equal(rec1, rec2), "non-deterministic"
    assert ac1.shape == (B, 16, ntok) and rec1.shape == (B, ntok * 3840) and bool(torch.isfinite(rec1).all())
    i = 4
    aci, sci = model.encode(wav[i:i + 1].contiguous(), feat[i:i + 1].contiguous())
    reci = model.decode(ac1[i:i + 1].contiguous(), sc1[i:i + 1].contiguous())
    torch.cuda.synchronize()
    match = float((aci == ac1[i:i + 1]).float().mean())
    e = rel(reci, rec1[i:i + 1])
    print(f"[full-size] batch invariance: code match {match:.4f}, wav rel {e:.2e}")
    assert match == 1.0 and e < 1e-5
    assert int(ac1.min()) >= 0 and int(ac1.max()) < 1024


def test_graphed_roundtrip_matches_eager(lib):
    """Codec.graphed('roundtrip'): the CUDA-graph replay returns bit-identical tokens and waveform, also after the static
    inputs are overwritten with a second batch."""
    from oracle import weights
    cfg = weights.h2_small()
    m, _ = build(cfg, 5, "mixed")
    batches = []
    for seed in (1, 2):
        wav, feat = weights.synth_inputs(cfg, 3, 6, seed)
        batches.append((wav.cuda(), feat.cuda()))
    g = m.graphed("roundtrip", *batches[0])
    assert g.launches_per_replay > 50
    for wav, feat in batches + batches[:1]:
        ac, sc, rec = [t.clone() for t in g(wav, feat)]
        ea, es = m.encode(wav, feat)
        er = m.decode(ea, es)
        torch.cuda.synchronize()
        assert torch.equal(ac, ea) and torch.equal(sc, es) and torch.equal(rec, er)


def test_graphed_stream_host_io_matches_eager(lib):
    """GraphedCall.stream: pinned-host inputs / outputs with the copies on a side stream overlapped across steps; every step's host
    outputs equal the eager result for that step's inputs (staging buffers are never overwritten while still in flight)."""
    from oracle import weights
    cfg = weights.h2_small()
    m, _ = build(cfg, 5, "mixed")
    host_in = []
    for seed in (1, 2, 3, 4):
        wav, feat = weights.synth_inputs(cfg, 3, 6, seed)
        host_in.append((wav.pin_memory(), feat.pin_memory()))
    g = m.graphed("roundtrip", host_in[0][0].cuda(), host_in[0][1].cuda())
    outs = [tuple(torch.empty(o.shape, dtype=o.dtype).pin_memory() for o in g.outputs) for _ in host_in]
    for (wav, feat), out in zip(host_in, outs):          # back-to-back, no synchronisation between steps
        g.stream((wav, feat), out)
    g.finish()
    torch.cuda.synchronize()
    for (wav, feat), (ac, sc, rec) in zip(host_in, outs):
        ea, es = m.encode(wav.cuda(), feat.cuda())
        er = m.decode(ea, es)
        torch.cuda.synchronize()
        assert torch.equal(ac, ea.cpu()) and torch.equal(sc, es.cpu()) and torch.equal(rec, er.cpu())
