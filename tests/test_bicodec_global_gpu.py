"""GPU parity of BiCodec.get_global_tokens (mel -> ECAPA-TDNN -> perceiver -> FSQ) against the outputs of the reference's own
classes (tests/golden/bicodec_global_small.npz) and the fp64 oracle on the shipped configuration, plus the two GEMM epilogues the
path adds (ReLU + folded BatchNorm, GEGLU), checked in fp64.

Token rule: a token is compared exactly when all of its FSQ decisions lie at least TAU from a rounding boundary in the fp64
oracle; TAU is at least 10x the largest |z_gpu - z_oracle| seen.  Flips are allowed only below TAU and are counted."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
FLOAT_TOL = 5e-5                 # the SSL front ends' budget for fp32-grade (3-term split) taps
TAU_MIN = 1e-4


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def build(cfg, speaker_sd, seed=3):
    from oracle import bicodec as ob
    from unified_audio_b200.bicodec import BiCodec
    sd = dict(ob.make_state_dict(cfg, seed))
    sd.update(speaker_sd)
    m = BiCodec(cfg, global_tokens=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def small_model():
    from oracle import bicodec_global as og
    z = np.load(os.path.join(GOLD, "bicodec_global_small.npz"))
    meta = json.loads(str(z["meta"]))
    cfg = og.bicodec_global_small()
    ssd = og.make_speaker_state_dict(cfg, meta["seed"])
    ssd["speaker_encoder.quantizer.project_in.weight"] = torch.from_numpy(z["project_in_weight"])
    ssd["speaker_encoder.quantizer.project_in.bias"] = torch.from_numpy(z["project_in_bias"])
    m, sd = build(cfg, ssd)
    return z, cfg, m, sd


def compare_tokens(got, want, z_gpu, z_ref, levels, label):
    from oracle import bicodec_global as og
    zerr = float((z_gpu.double().cpu() - z_ref.double().cpu()).abs().max())
    tau = max(10 * zerr, TAU_MIN)
    safe = (og.fsq_margins(z_ref, levels) >= tau).all(-1)                 # [B, N]
    g, w = got.cpu()[:, 0], want.cpu()[:, 0]
    assert torch.equal(g[safe], w[safe]), f"{label}: token differs where every decision has a margin >= tau"
    flips = int((g[~safe] != w[~safe]).sum())
    print(f"[{label}] tau {tau:.2e} (max |dz| {zerr:.2e}), tokens below tau {int((~safe).sum())}, flips {flips}")
    return tau, int((~safe).sum()), flips


def test_small_fixture_matches_reference(lib):
    z, cfg, m, _ = small_model()
    wav = torch.from_numpy(z["ref_wav"]).cuda()
    taps = {}
    tok = m.get_global_tokens({"ref_wav": wav}, taps=taps)
    torch.cuda.synchronize()
    B = wav.shape[0]
    e = dict(mel=rel(taps["mel"].transpose(1, 2), z["mel"]), latent=rel(taps["latent"].transpose(1, 2), z["latent"]),
             perceiver=rel(taps["perceiver"], z["perceiver"]), z=rel(taps["z"], z["z"]))
    print("[bicodec global small] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    assert tok.dtype == torch.int32 and tok.shape == (B, 1, cfg["speaker"]["token_num"])
    assert max(e.values()) < FLOAT_TOL
    tau, below, flips = compare_tokens(tok, torch.from_numpy(z["tokens"]), taps["z"], torch.from_numpy(z["z"]).double(),
                                       cfg["speaker"]["fsq_levels"], "small")
    assert below == 0 and torch.equal(tok.cpu(), torch.from_numpy(z["tokens"]))     # seeds chosen so that this is strict equality
    mel = m.mel_spectrogram(wav[:, None, :])
    assert mel.shape == (B, cfg["mel_params"]["num_mels"], 1 + wav.shape[1] // 320) and rel(mel, z["mel"]) < FLOAT_TOL
    with pytest.raises(ValueError):
        m.get_global_tokens({"ref_wav": wav[:, None, None]})
    with pytest.raises(RuntimeError):
        m.get_global_tokens({"ref_wav": wav.cpu()})


def test_full_config_matches_oracle_and_is_batch_independent(lib):
    from oracle import bicodec_global as og
    from oracle.make_golden_bicodec_global import synth_wav
    cfg = og.BICODEC_GLOBAL_FULL
    ssd = og.make_speaker_state_dict(cfg, 21)
    m, sd = build(cfg, ssd, 4)
    wav = synth_wav(3, 96000, 121)
    sd64 = {k: v.double() for k, v in ssd.items()}
    want_taps = {}
    want = og.get_global_tokens(sd64, cfg, wav[:2].double(), want_taps)
    taps = {}
    got = m.get_global_tokens({"ref_wav": wav[:2].cuda()}, taps=taps)
    torch.cuda.synchronize()
    e = dict(mel=rel(taps["mel"].transpose(1, 2), want_taps["mel"]), latent=rel(taps["latent"].transpose(1, 2), want_taps["latent"]),
             perceiver=rel(taps["perceiver"], want_taps["perceiver"]), z=rel(taps["z"], want_taps["z"]))
    print("[bicodec global full B=2 x 6 s] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    assert got.shape == (2, 1, 32) and got.dtype == torch.int32 and max(e.values()) < FLOAT_TOL
    compare_tokens(got, want, taps["z"], want_taps["z"], cfg["speaker"]["fsq_levels"], "full")
    # a clip's tokens do not depend on its batch, and a call is deterministic
    three = m.get_global_tokens({"ref_wav": wav.cuda()})
    again = m.get_global_tokens({"ref_wav": wav.cuda()})
    alone = torch.cat([m.get_global_tokens({"ref_wav": wav[i:i + 1].cuda()}) for i in range(3)], 0)
    torch.cuda.synchronize()
    assert torch.equal(three, alone) and torch.equal(three, again) and torch.equal(three[:2], got)
    # the tokens are what detokenize takes
    from oracle import bicodec as ob
    sem, _ = ob.synth_tokens(cfg, 2, 9, 77)
    wav_out = m.detokenize(sem.cuda(), got)
    ref_out = ob.detokenize(sd, cfg, sem, got.cpu().long())
    torch.cuda.synchronize()
    assert wav_out.shape == (2, 1, 9 * 320) and rel(wav_out, ref_out) < 1e-3


def test_get_ref_clip_tiles_short_and_cuts_long(lib):
    from unified_audio_b200.unise import BiCodecTokenizer
    z, cfg, m, _ = small_model()
    tok = BiCodecTokenizer(m, ref_segment_length=int(json.loads(str(z["meta"]))["ref_segment_length"]))
    for n in ("short", "long"):
        got = tok.get_ref_clip(torch.from_numpy(z[n + "_wav"]).cuda())
        assert torch.equal(got.cpu(), torch.from_numpy(z[n + "_clip"])), n
    w = torch.randn(2, 40000, device="cuda")
    full = BiCodecTokenizer(m).get_ref_clip(w)
    assert full.shape == (2, 96000) and torch.equal(full.cpu(), torch.tile(w.cpu(), (1, 3))[:, :96000])


def test_relu_bn_epilogue_and_geglu_fp64(lib):
    """ReLU + gamma + broadcast residual row (Conv1dReluBn) in the GEMM epilogue, and the GEGLU kernel after a GEMM, 3-term split,
    ragged shapes; fp64 reference computed from the planes."""
    from unified_audio_b200 import ops
    from unified_audio_b200.ops import ACT_RELU, Planes, rowmap
    g = torch.Generator().manual_seed(9)
    M, K = 301, 192
    A = Planes.from_f32(torch.randn(M, K, generator=g).cuda(), True)
    a64 = A.float().double().cpu()
    for N in (200, 37):
        W = Planes.from_f32(torch.randn(N, K, generator=g).cuda() / K ** 0.5, True)
        w64 = W.float().double().cpu()
        bias, gamma, shift = (torch.randn(N, generator=g) for _ in range(3))
        out = torch.empty(M, N, device="cuda")
        ops.gemm(A, W, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias.cuda(), gamma=gamma.cuda(), act=ACT_RELU,
                 residual=rowmap(shift.cuda(), 0, 0, 0), out_f32=rowmap(out, N, M, 0))
        want = torch.relu(a64 @ w64.t() + bias.double()) * gamma.double() + shift.double()
        e = float((out.double().cpu() - want).abs().max() / want.abs().max())
        print(f"[relu+bn N={N}] rel {e:.2e}")
        assert e < 1e-5
    inner = 171
    W = Planes.from_f32(torch.randn(2 * inner, K, generator=g).cuda() / K ** 0.5, True)
    w64 = W.float().double().cpu()
    bias = torch.randn(2 * inner, generator=g)
    h = torch.empty(M, 2 * inner, device="cuda")
    ops.gemm(A, W, 2 * inner, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias.cuda(), out_f32=rowmap(h, 2 * inner, M, 0))
    hid = Planes.zeros((M, 192), True, "cuda")
    ops.geglu_planes(h, M, inner, hid, 192)
    v = a64 @ w64.t() + bias.double()
    want = torch.nn.functional.gelu(v[:, inner:]) * v[:, :inner]
    got = hid.float().double().cpu()
    e = float((got[:, :inner] - want).abs().max() / want.abs().max())
    print(f"[geglu] rel {e:.2e}")
    assert e < 1e-5 and float(got[:, inner:].abs().max()) == 0.0
