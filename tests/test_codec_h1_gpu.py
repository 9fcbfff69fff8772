"""GPU parity of unified_audio_b200.CodecH1 (H-Codec-1.0, BASELINE configs[0]: 1 s 16 kHz mono clip round trip)
against the golden outputs of the reference's own modules (tests/golden/h1_full_1s.npz) and the oracle."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("precision", ["mixed", "accurate"])
def test_h1_config1_roundtrip(lib, precision):
    from oracle import hcodec1, rvq
    from unified_audio_b200.codec_h1 import CodecH1
    z = np.load(os.path.join(GOLD, "h1_full_1s.npz"))
    meta = json.loads(str(z["meta"]))
    c = hcodec1.H1
    sd = hcodec1.make_state_dict(c, meta["seed_w"])
    m = CodecH1({}, {}, {}, precision=precision)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    g = torch.Generator().manual_seed(meta["seed_x"])
    x = 0.1 * torch.randn(1, 1, 16000, generator=g)
    g2 = torch.Generator().manual_seed(meta["seed_x"] + 1)
    f = torch.randn(1, 768, 50, generator=g2)
    feat = torch.sign(f) * f.abs() ** 0.3
    otaps, gtaps = {}, {}
    hcodec1.seanet_encoder(sd, c, x, otaps)
    ac, sc = m.encode(x.cuda(), feat.cuda(), taps=gtaps)
    torch.cuda.synchronize()
    for k in otaps:
        if k in gtaps:
            print(f"  tap {k}: max-rel {rel(gtaps[k], otaps[k]):.2e}")
    e_emb, e_sem = rel(gtaps["enc.out"], torch.from_numpy(z["emb"])), rel(gtaps["sem.out"], torch.from_numpy(z["sem"]))
    print(f"[h1/{precision}] emb rel {e_emb:.2e} sem rel {e_sem:.2e}")
    assert e_emb < 1e-3 and e_sem < 1e-3
    want_a, want_s = torch.from_numpy(z["acoustic_codes"]), torch.from_numpy(z["semantic_codes"])
    assert ac.shape == want_a.shape == (1, 4, 25)
    emb_ref = torch.from_numpy(z["emb"])
    rows = emb_ref.transpose(1, 2).reshape(25, 512)
    cb = torch.stack([sd[f"quantizer.layers.{i}._codebook.embed"][0] for i in range(4)], 0)
    _, margin = rvq.rvq_margin_audit(rows, cb, want_a.transpose(1, 2).reshape(25, 4))
    bad = (ac.cpu() != want_a).transpose(1, 2).reshape(25, 4)
    print(f"[h1/{precision}] differing acoustic indices {int(bad.sum())}/100, semantic {int((sc.cpu() != want_s).sum())}/100;"
          f" min margin {float(margin.min()):.2e}")
    for t in range(25):
        if bad[t].any():
            q = int(bad[t].nonzero()[0])
            assert float(margin[t, q]) < 1e-3, "index differs at a numerically safe decision"
    rec = m.decode(want_a.cuda(), want_s.cuda())
    torch.cuda.synchronize()
    e_wav = rel(rec, torch.from_numpy(z["wav_rec"]))
    print(f"[h1/{precision}] wav rel {e_wav:.2e}")
    assert rec.shape == (1, 16000) and e_wav < 1e-3


def test_h1_batch_of_260_matches_batch_of_4(lib):
    """A clip's codes do not depend on the batch it is encoded in: the shipped config at B = 260 (three LSTM launches of at most
    128 rows per transformer layer) gives rows 0-3 the codes those four clips get at B = 4"""
    from oracle import hcodec1
    from unified_audio_b200.codec_h1 import CodecH1
    m = CodecH1({}, {}, {})
    m.load_state_dict(hcodec1.make_state_dict(hcodec1.H1, 5), strict=True)
    m = m.cuda()
    B, T = 260, 3200
    g = torch.Generator().manual_seed(17)
    x = 0.1 * torch.randn(B, 1, T, generator=g)
    f = torch.randn(B, 768, T // 320, generator=g)
    feat = torch.sign(f) * f.abs() ** 0.3
    taps_b, taps_4 = {}, {}
    codes_b = m.encode(x.cuda(), feat.cuda(), taps=taps_b)
    codes_4 = m.encode(x[:4].cuda(), feat[:4].cuda(), taps=taps_4)
    torch.cuda.synchronize()
    diverged = [k for k in taps_4 if not torch.equal(taps_b[k][:4], taps_4[k])]
    print(f"taps of rows 0-3 that differ between B = {B} and B = 4: {diverged or 'none'}")
    for name, cb, c4 in zip(("acoustic", "semantic"), codes_b, codes_4):
        assert torch.equal(cb[:4], c4), f"{name} codes of rows 0-3 differ between B = {B} and B = 4; taps that differ: {diverged}"


def test_h1_small_decoder_width_rejected_at_prepare(lib):
    """oracle.hcodec1.h1_small() has dec_dim 384, which the wgmma recurrence cannot run: encode fails while the weights are
    packed, with a message naming the width, instead of inside a kernel"""
    from oracle import hcodec1
    from unified_audio_b200.codec_h1 import CodecH1
    c = hcodec1.h1_small()
    m = CodecH1(_cfg=c)
    m.load_state_dict(hcodec1.make_state_dict(c, 1), strict=True)
    m = m.cuda()
    with pytest.raises(ValueError, match="LSTM width 384 unsupported by the wgmma recurrence"):
        m.encode(torch.zeros(1, 1, 1280, device="cuda"), torch.zeros(1, c["sem_in"], 4, device="cuda"))
