"""The handle-level C ABI (include/quark_b200.h "Handle-level contract", SURVEY.md 8b) driven through ctypes ONLY -
qb_init / qb_codec_load / qb_codec_encode / qb_codec_decode / qb_rvq_* - against the golden fixtures generated from
the reference's own modules and against the oracle.  No Python orchestration of kernels on this path: torch only allocates
the device buffers whose pointers are passed."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle.parity import audit_codes, rel

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3


def _tensors(sd):
    from unified_audio_b200._lib import Tensor
    keep, arr = [], (Tensor * len(sd))()
    for i, (k, v) in enumerate(sd.items()):
        t = v.float().contiguous().cuda()
        name = k.encode()
        keep += [t, name]
        arr[i].name, arr[i].data, arr[i].ndim = name, t.data_ptr(), t.dim()
        for j, s in enumerate(t.shape):
            arr[i].shape[j] = s
    return arr, keep


def _check(lib, code):
    assert code == 0, lib.qb_last_error().decode()


def _codec_cfg(cfg, precision=0):
    from unified_audio_b200._lib import CodecCfg
    e, d, q, s = cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"]
    c = CodecCfg()
    c.dim, c.intermediate_dim, c.dimension, c.n_fft, c.hop_length = e["dim"], e["intermediate_dim"], e["dimension"], e["n_fft"], e["hop_length"]
    c.enc_convnext_layers, c.enc_transformer_layers = e["convnext_layers"], e["transformer_layers"]
    c.dec_convnext_layers, c.dec_transformer_layers, c.dec_input_channels = d["convnext_layers"], d["transformer_layers"], d["input_channels"]
    c.frame_stride = int(50 / e["target_frame_rate"])
    c.num_quantizers, c.codebook_size = q["num_quantizers"], q["codebook_size"]
    c.sem_input_channels, c.sem_encode_channels, c.sem_out_channels = s["input_channels"], s["encode_channels"], s["out_channels"]
    c.sem_n_blocks = len(s["strides"])
    for i, st in enumerate(s["strides"]):
        c.sem_strides[i] = st
    c.precision = precision
    return c


@pytest.mark.parametrize("name", ["small", "mid"])
def test_codec_c_abi_roundtrip_against_reference_golden(lib, name):
    """encode -> decode through the C entry points only, against the outputs of the reference's own Codec (tests/golden)."""
    from oracle import hcodec2, weights
    z = np.load(os.path.join(GOLD, f"h2_{name}.npz"))
    meta = json.loads(str(z["meta"]))
    cfg = meta["cfg"]
    sd = weights.make_h2_state_dict(cfg, meta["seed_w"])
    wav, feat = weights.synth_inputs(cfg, meta["batch"], meta["n_tokens"], meta["seed_x"])
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    h, codec = C.c_void_p(), C.c_void_p()
    _check(lib, lib.qb_init(0, C.byref(h)))
    arr, keep = _tensors(sd)
    ccfg = _codec_cfg(cfg)
    _check(lib, lib.qb_codec_load(h, C.byref(ccfg), arr, len(sd), C.byref(codec)))
    del keep                                                    # the handle owns its repacked copies
    B, T = wav.shape
    N, nq = meta["n_tokens"], cfg["quantizer_config"]["num_quantizers"]
    wav_d, feat_d = wav.cuda().contiguous(), feat.cuda().contiguous()
    ac = torch.full((B, nq, N), -1, dtype=torch.int64, device="cuda")
    sc = torch.full((B, nq, N), -1, dtype=torch.int64, device="cuda")
    # taps through the C callback (copied with qb_memcpy_d2d on the same stream)
    from unified_audio_b200._lib import TAP_FN
    taps = {}

    def cb(user, nm, ptr, b, rows, cc):
        buf = torch.empty(b, rows, cc, device="cuda")
        _check(lib, lib.qb_memcpy_d2d(buf.data_ptr(), ptr, b * rows * cc * 4, stream))
        taps[nm.decode()] = buf
    fn = TAP_FN(cb)
    _check(lib, lib.qb_codec_set_tap(codec, fn, None))
    _check(lib, lib.qb_codec_encode(codec, wav_d.data_ptr(), B, T, feat_d.data_ptr(), ac.data_ptr(), sc.data_ptr(), stream))
    _check(lib, lib.qb_codec_set_tap(codec, TAP_FN(0), None))
    torch.cuda.synchronize()
    emb_ref, sem_ref = torch.from_numpy(z["emb"]), torch.from_numpy(z["sem"])           # [B, D, N]
    e_emb = rel(taps["enc.out"].transpose(1, 2), emb_ref)
    e_sem = rel(taps["sem.out"].transpose(1, 2), sem_ref)
    D = emb_ref.shape[1]
    rows = lambda t: t.float().cpu().reshape(B * N, D)
    for tag, got, want, g, o, q in (("acoustic", ac, z["acoustic_codes"], taps["enc.out"], emb_ref, "quantizer"),
                                    ("semantic", sc, z["semantic_codes"], taps["sem.out"], sem_ref, "semantic_quantizer")):
        a = audit_codes(got, torch.from_numpy(want), rows(g), o.transpose(1, 2).reshape(B * N, D), hcodec2._codebooks(sd, q))
        print(f"[c-abi {name}] {tag}: {a}")
        assert a["explained"]
    wav_out = torch.empty(B, N * 3840, device="cuda")
    ra, rs = torch.from_numpy(z["acoustic_codes"]).cuda().contiguous(), torch.from_numpy(z["semantic_codes"]).cuda().contiguous()
    _check(lib, lib.qb_codec_decode(codec, ra.data_ptr(), rs.data_ptr(), B, N, wav_out.data_ptr(), stream))      # no taps: the product call
    torch.cuda.synchronize()
    enc_taps = dict(taps)
    taps.clear()
    wav_tap = torch.empty_like(wav_out)
    _check(lib, lib.qb_codec_set_tap(codec, fn, None))
    _check(lib, lib.qb_codec_decode(codec, ra.data_ptr(), rs.data_ptr(), B, N, wav_tap.data_ptr(), stream))
    _check(lib, lib.qb_codec_set_tap(codec, TAP_FN(0), None))
    torch.cuda.synchronize()
    assert torch.equal(wav_tap, wav_out), "decode with and without debug taps must be bit-identical"
    odt = {}
    hcodec2.codec_decode(sd, cfg, torch.from_numpy(z["acoustic_codes"]), torch.from_numpy(z["semantic_codes"]), taps=odt)
    for k in odt:
        if k in taps:
            ref_t = odt[k] if k == "dec.final_norm" else odt[k].transpose(1, 2)
            print(f"   [c-abi {name}] tap {k}: {rel(taps[k], ref_t):.2e}")
    taps = enc_taps
    e_wav = rel(wav_out, torch.from_numpy(z["wav_rec"]))
    print(f"[c-abi {name}] emb rel {e_emb:.2e} sem rel {e_sem:.2e} wav rel {e_wav:.2e}")
    assert e_emb < TOL and e_sem < TOL and e_wav < TOL
    # error contract: negative code + message, no exception, no crash
    assert lib.qb_codec_encode(codec, wav_d.data_ptr(), B, T - 1, feat_d.data_ptr(), ac.data_ptr(), sc.data_ptr(), stream) < 0
    assert b"multiple" in lib.qb_last_error()
    assert lib.qb_codec_load(h, C.byref(ccfg), arr, 3, C.byref(C.c_void_p())) < 0 and b"missing weight" in lib.qb_last_error()
    big = _codec_cfg(cfg)
    big.n_fft, big.hop_length = 8192, 4096                      # no two-stage factorisation n_fft = P*Q with P, Q <= 64
    assert lib.qb_codec_load(h, C.byref(big), arr, len(sd), C.byref(C.c_void_p())) < 0 and b"n_fft <= 4096" in lib.qb_last_error()
    # row-level quantiser handles of the loaded codec == the oracle on identical rows
    from oracle import rvq as orvq
    q0 = C.c_void_p(lib.qb_codec_rvq(codec, 0))
    x = rows(taps["enc.out"])
    idx = torch.empty(B * N, nq, dtype=torch.int64, device="cuda")
    quant = torch.empty(B * N, D, device="cuda")
    xd = x.cuda()
    _check(lib, lib.qb_rvq_encode_rows(q0, xd.data_ptr(), B * N, idx.data_ptr(), quant.data_ptr(), stream))
    out = torch.empty(B * N, D, device="cuda")
    _check(lib, lib.qb_rvq_decode_rows(q0, idx.data_ptr(), B * N, out.data_ptr(), stream))
    torch.cuda.synchronize()
    cb_a = hcodec2._codebooks(sd, "quantizer")
    oidx, oquant = orvq.rvq_encode(x, cb_a)
    tidx, margin = orvq.rvq_margin_audit(x, cb_a, oidx)
    safe = (margin > 1e-5).all(-1)
    assert bool((idx.cpu()[safe] == oidx[safe]).all())
    assert torch.equal(out.cpu(), orvq.rvq_decode(idx.cpu(), cb_a)) and rel(quant, out) < 1e-6
    lib.qb_codec_free(codec)
    lib.qb_handle_free(h)
