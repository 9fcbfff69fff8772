"""Codec.forward / semantic_decode on the GPU for H-Codec-2.0, 1.0 and 1.5.

pred_feat against the fp64 oracle (oracle/semantic_decoder.py, pinned to the reference's Decoder by tests/test_codec_forward_host.py)
at the shipped decoder widths, B = 2, the code counts of 10 s clips and odd ones; recon bit-identical to decode(*encode(x, feat)); the
H-Codec-1.5 token lengths; the transposed conv's phase GEMM against fp64; the two C entries through ctypes alone; and a forward after
a call of another shape."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import semantic_decoder as osd

pytestmark = pytest.mark.gpu
TOL = 1e-3


def frob(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def _codes(B, nq, N, K, seed):
    return torch.randint(0, K, (B, nq, N), generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------ faces with the semantic decoder at the shipped widths
def _h2(dec_seed=7):
    from oracle import weights
    from unified_audio_b200.codec import Codec
    cfg = weights.h2_small(qdim=512, sem_ch=1536)          # small encoder / decoder; semantic decoder 512 -> 1536 -> 768, [2, 1, 2]
    sd = dict(weights.make_h2_state_dict(cfg, 5), **osd.make_state_dict(cfg["semantic_decoder_config"], dec_seed))
    m = Codec(cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"],
              cfg["semantic_decoder_config"], semantic_decoder=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd, cfg["semantic_decoder_config"], cfg


def _h1():
    from oracle import hcodec1
    from unified_audio_b200.codec_h1 import CodecH1
    c = hcodec1.H1
    sd = dict(hcodec1.make_state_dict(c, 5), **osd.make_state_dict(osd.h1_config(c), 7))
    m = CodecH1(semantic_decoder=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd, osd.h1_config(c), c


def _h15():
    from oracle import hcodec15
    from unified_audio_b200.codec_h15 import CodecH15
    c = hcodec15.h15_shallow()
    sd = dict(hcodec15.make_state_dict(c, 5), **osd.make_state_dict(osd.h1_config(c), 7))
    m = CodecH15(_cfg={k: v for k, v in c.items() if k != "layer_scale"}, semantic_decoder=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd, osd.h1_config(c), c


FACES = {"h2": (_h2, 125), "h1": (_h1, 250), "h15": (_h15, 250)}      # codes of a 10 s clip


def _oracle_pred(sd, dcfg, codes):
    z = osd._dequantize({k: v.double() for k, v in sd.items() if k.startswith("semantic_quantizer.")}, "semantic_quantizer", codes)
    return osd.semantic_decoder_forward({k: v.double() for k, v in sd.items() if k.startswith("semantic_decoder.")}, dcfg, z)


@pytest.mark.parametrize("face", list(FACES))
def test_semantic_decode_against_fp64_oracle(face):
    make, n10 = FACES[face]
    m, sd, dcfg, _ = make()
    nq, K = m.semantic_quantizer.num_quantizers, m.semantic_quantizer.codebook_size
    up = 1
    for s in dcfg["strides"]:
        up *= s
    errs = {}
    for N in (n10, 37, 1):
        codes = _codes(2, nq, N, K, N)
        if face == "h15":      # length-packed codes of one token per frame: decode's input format
            from unified_audio_b200 import adaptive
            got = m.semantic_decode(adaptive.inject_lengths(codes.cuda(), torch.ones(2, N, dtype=torch.long, device="cuda"), K))
        else:
            got = m.semantic_decode(codes.cuda())
        want = _oracle_pred(sd, dcfg, codes)
        assert got.dtype == torch.float32 and tuple(got.shape) == (2, dcfg["output_channels"], N * up)
        errs[N] = frob(got, want)
    print(face, "pred_feat rel. Frobenius vs fp64:", errs)
    assert max(errs.values()) < TOL, errs


def _inputs_h2(cfg, B, n):
    from oracle import weights
    return weights.synth_inputs(cfg, B, n, 11)


def _inputs_h1(c, B, T, seed=11):
    g = torch.Generator().manual_seed(seed)
    x = 0.1 * torch.randn(B, 1, T, generator=g)
    f = torch.randn(B, c["sem_in"], T // 320, generator=torch.Generator().manual_seed(seed + 1))
    return x, torch.sign(f) * f.abs() ** 0.3


@pytest.mark.parametrize("face", list(FACES))
def test_forward_recon_is_decode_of_encode(face):
    make = FACES[face][0]
    m, _, _, c = make()
    x, feat = _inputs_h2(c, 2, 3) if face == "h2" else _inputs_h1(c, 2, 640 * 5)
    x, feat = x.cuda(), feat.cuda()
    out = m(x, feat)
    if face == "h15":
        codes = m.encode(x, feat)
        recon = m.decode(codes["acoustic_codes"], codes["semantic_codes"])
        from unified_audio_b200 import adaptive
        _, lens = adaptive.extract_lengths(codes["semantic_codes"], m.codebook_size)
        assert set(out) == {"recon", "pred_feat", "commit_loss", "token_lengths"}
        assert out["token_lengths"].dtype == torch.int64 and torch.equal(out["token_lengths"], lens)
        assert torch.equal(out["pred_feat"], m.semantic_decode(codes["semantic_codes"]))
        got_recon, loss = out["recon"], out["commit_loss"]
    else:
        ac, sc = m.encode(x, feat)
        recon = m.decode(ac, sc)
        got_recon, pred, loss = out
        assert torch.equal(pred, m.semantic_decode(sc)) and pred.dtype == torch.float32
    assert torch.equal(got_recon, recon)
    assert loss.dim() == 0 and loss.dtype == torch.float32 and loss.is_cuda and float(loss) == 0.0


@pytest.mark.parametrize("T", [1, 37, 125])
def test_transposed_conv_phase_gemm_against_fp64(T):
    """ConvTranspose1d(1536 -> 1536, k 4, stride 2, padding 1) - the H-Codec-2.0 decoder's first up-sampler - as the 2-tap phase
    GEMM over a one-frame-padded buffer, read back as the cropped channel-last clip, and the ELU planes the next unit reads."""
    from unified_audio_b200 import ops
    from unified_audio_b200.ops import Planes, rowmap
    B, C, s = 4, 1536, 2
    g = torch.Generator().manual_seed(T)
    w = torch.randn(C, C, 2 * s, generator=g, dtype=torch.float64) / (2 * C) ** 0.5
    b = torch.randn(C, generator=g, dtype=torch.float64) * 0.05
    x = torch.randn(B, C, T, generator=g, dtype=torch.float64)
    want = F.conv_transpose1d(x, w, b, stride=s, padding=1)                       # [B, C, 2T]
    wt, J = ops.convt_planes(w.float().cuda(), s, True)
    a = Planes.zeros((B, T + 2, C), True, "cuda")
    ops.rows_to_planes(x.transpose(1, 2).reshape(B * T, C).float().cuda().contiguous(), B, T, C, a, C, T + 2, 1)
    up = torch.zeros(B, T + 1, s * C, device="cuda")
    ops.gemm(a, wt, s * C, a_batch=B, a_rows_per_batch=T + 2, a_ld=C, m_per_batch=T + 1, taps=J,
             bias=b.float().repeat(s).cuda().contiguous(), out_f32=rowmap(up, s * C, T + 1, 0))
    got = up.reshape(B, (T + 1) * s, C)[:, 1:1 + s * T].transpose(1, 2)
    assert J == 2 and frob(got, want) < 1e-4          # 3-term split operands, fp32 accumulation over K = 2 x 1536
    pe = Planes.zeros((B, s * T + 2, C), True, "cuda")
    ops.elu_planes(up.view(-1)[C:], (T + 1) * s * C, B, s * T, C, pe, C, s * T + 2, 1)
    el = pe.float().reshape(B, s * T + 2, C)
    assert bool((el[:, 0] == 0).all()) and bool((el[:, -1] == 0).all())
    assert frob(el[:, 1:-1].transpose(1, 2), F.elu(got.double())) < 1e-6


def test_c_abi_through_ctypes_matches_semantic_decode():
    """qb_codec_load_semantic_decoder / qb_codec_semantic_decode called through ctypes on a handle built without the decoder give
    Codec.semantic_decode's bits; a second load is refused."""
    from unified_audio_b200 import _lib
    from unified_audio_b200.codec import Codec
    from unified_audio_b200.engine import CodecEngine, _tensor_array
    m, sd, dcfg, cfg = _h2()
    plain = Codec(cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"],
                  cfg["semantic_decoder_config"])
    plain.load_state_dict(sd, strict=True)
    eng = plain.cuda().engine()
    assert isinstance(eng, CodecEngine)
    lib = _lib.load()
    dec = {k: v.cuda() for k, v in sd.items() if k.startswith("semantic_decoder.")}
    c = _lib.SemanticDecoderCfg()
    c.code_dim, c.output_channels, c.n_blocks = dcfg["code_dim"], dcfg["output_channels"], len(dcfg["strides"])
    for i, s in enumerate(dcfg["strides"]):
        c.strides[i] = s
    arr, keep = _tensor_array(dec)
    _lib.check(lib.qb_codec_load_semantic_decoder(eng.h, C.byref(c), arr, len(dec)))
    assert lib.qb_codec_load_semantic_decoder(eng.h, C.byref(c), arr, len(dec)) != 0
    codes = _codes(2, m.semantic_quantizer.num_quantizers, 125, m.semantic_quantizer.codebook_size, 3).cuda()
    out = torch.empty(2, dcfg["output_channels"], 500, device="cuda")
    _lib.check(lib.qb_codec_semantic_decode(eng.h, codes.data_ptr(), 2, 125, out.data_ptr(),
                                            C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert torch.equal(out, m.semantic_decode(codes))
    del keep


@pytest.mark.parametrize("face", list(FACES))
def test_forward_after_another_shape_matches_fresh_face(face):
    make = FACES[face][0]
    m, sd, _, c = make()
    if face == "h2":
        (x0, f0), (x1, f1) = _inputs_h2(c, 1, 6), _inputs_h2(c, 2, 3)
    else:
        (x0, f0), (x1, f1) = _inputs_h1(c, 1, 640 * 6), _inputs_h1(c, 2, 640 * 3)
    m.encode(x0.cuda(), f0.cuda())
    m(x0.cuda(), f0.cuda())
    got = m(x1.cuda(), f1.cuda())
    fresh = make()[0](x1.cuda(), f1.cuda())
    if face == "h15":
        assert set(got) == set(fresh) and all(torch.equal(got[k], fresh[k]) for k in got)
    else:
        assert all(torch.equal(a, b) for a, b in zip(got, fresh))


# ------------------------------------------------------------------ the reference's own Codec.forward (fixture, small widths)
@pytest.mark.parametrize("name", ["h2", "h1", "h15"])
def test_forward_against_reference_fixture(name):
    """each face's forward on the inputs and seeded weights of the fixture the reference's unmodified Codec.forward wrote
    (oracle/make_golden_codec_forward.py): recon and pred_feat within the suite's 1e-3, commit_loss 0, token_lengths equal"""
    import os

    import numpy as np
    from oracle.make_golden_codec_forward import forward_case
    from unified_audio_b200.codec import Codec
    from unified_audio_b200.codec_h1 import CodecH1
    from unified_audio_b200.codec_h15 import CodecH15
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "codec_forward_small.npz"))
    cfg, sd, x, feat = forward_case(name)
    if name == "h2":
        m = Codec(cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"],
                  cfg["semantic_decoder_config"], semantic_decoder=True)
    elif name == "h1":
        m = CodecH1(semantic_decoder=True)
    else:
        m = CodecH15(_cfg={k: v for k, v in cfg.items() if k != "layer_scale"}, semantic_decoder=True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    out = m(x.cuda(), feat.cuda())
    if name != "h15":
        out = dict(zip(("recon", "pred_feat", "commit_loss"), out))
    else:
        want_len = torch.from_numpy(z[f"fwd/{name}/token_lengths"])
        assert int(want_len.max()) > 1 and torch.equal(out["token_lengths"].cpu(), want_len)
    errs = {}
    for k in ("recon", "pred_feat"):
        want = torch.from_numpy(z[f"fwd/{name}/{k}"])
        got = out[k].reshape(want.shape) if k == "recon" else out[k]
        assert tuple(out[k].shape)[-1] == want.shape[-1]
        errs[k] = float((got.double().cpu() - want.double()).abs().max() / want.double().abs().max())
    print(name, "forward vs the reference's fixture (max-relative):", errs)
    assert max(errs.values()) < TOL, errs
    assert out["commit_loss"].dim() == 0 and float(out["commit_loss"]) == 0.0


def test_h15_semantic_decode_deaggregates_groups_like_the_oracle():
    """CodecH15.semantic_decode on groups of 1..8 frames (length-packed codes and plain codes + token_lengths) against the fp64
    oracle on the codes de-aggregated by oracle/adaptive.py"""
    from oracle import adaptive as oad
    from unified_audio_b200 import adaptive
    m, sd, dcfg, _ = _h15()
    nq, K = m.semantic_quantizer.num_quantizers, m.semantic_quantizer.codebook_size
    g = torch.Generator().manual_seed(5)
    B, T = 2, 61
    rows = []
    for _ in range(B):
        ln, left = [], T
        while left:
            ln.append(min(left, int(torch.randint(1, 9, (1,), generator=g))))
            left -= ln[-1]
        rows.append(ln)
    G = max(len(r) for r in rows)
    lens = torch.zeros(B, G, dtype=torch.long)
    for b, r in enumerate(rows):
        lens[b, :len(r)] = torch.tensor(r)
    codes = torch.randint(0, K, (B, nq, G), generator=g)
    want = _oracle_pred(sd, dcfg, oad.deaggregate_by_lengths(codes, lens))
    packed = adaptive.inject_lengths(codes.cuda(), lens.cuda(), K)
    got_packed = m.semantic_decode(packed)
    got_plain = m.semantic_decode(codes.cuda(), token_lengths=lens.cuda())
    assert int(lens.max()) > 1 and tuple(got_packed.shape) == (B, dcfg["output_channels"], 2 * T)
    assert torch.equal(got_packed, got_plain)
    err = frob(got_packed, want)
    print("h15 semantic_decode on groups vs fp64:", err)
    assert err < TOL
