"""GPU checks of BiCodec.forward: the ASTP and codebook-usage kernels against fp64 at the shapes and edges where each can go wrong,
the full face against the outputs of the reference's own BiCodec.forward (tests/golden/bicodec_forward_small.npz), and at the shipped
widths forward's reconstruction against detokenize(*tokenize(batch)) bit for bit, the x-vector and pred_feat against fp64, and the
token paths unchanged by an interleaved forward."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
FACE_TOL = 1e-3                  # the bar of the other BiCodec face tests
STD_FLOOR = np.float32(math.sqrt(1e-7))


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


# ------------------------------------------------------------------------------------------------------------------------- kernels
def _planes(shape):
    from unified_audio_b200.ops import Planes
    return Planes.zeros(shape, True, DEV)


def _context_ref(x):
    """x [B, T, C] fp64 -> [B, 2C] = [mean | sqrt(unbiased var + 1e-7)]"""
    return torch.cat([x.mean(1), torch.sqrt(x.var(1) + 1e-7)], 1)


def _pool_ref(x, logits):
    a = torch.softmax(logits, dim=1)
    mean = (a * x).sum(1)
    return torch.cat([mean, torch.sqrt(((a * x * x).sum(1) - mean ** 2).clamp(min=1e-7))], 1)


def _run_asp(x, logits):
    from unified_audio_b200 import ops
    B, T, C = x.shape
    ctx, cpl = torch.full((B, 2 * C), -1.0, device=DEV), _planes((B, 2 * C + 64))
    ops.asp_context(x.reshape(B * T, C), B, T, C, ctx, cpl, 2 * C + 64)
    pool, ppl = torch.full((B, 2 * C), -1.0, device=DEV), _planes((B, 2 * C + 64))
    ops.asp_pool(x.reshape(B * T, C), logits.reshape(B * T, C), B, T, C, pool, ppl, 2 * C + 64)
    torch.cuda.synchronize()
    for out, pl in ((ctx, cpl), (pool, ppl)):          # the planes carry the fp32 values; columns past 2C stay untouched
        assert torch.equal(pl.hi[:, :2 * C], out.half())
        assert float((pl.float()[:, :2 * C] - out).abs().max()) <= float(out.abs().max()) * 2.0 ** -21
        assert not pl.hi[:, 2 * C:].any()
    return ctx.cpu().double(), pool.cpu().double()


@pytest.mark.parametrize("T", [2, 37, 1501])
def test_astp_kernels_against_fp64(lib, T):
    g = torch.Generator().manual_seed(T)
    B, C = 3, 200                                   # C above the block's 128 channels, not a multiple of it
    x = torch.relu(torch.randn(B, T, C, generator=g)) + 0.1 * torch.randn(B, 1, C, generator=g)
    logits = 4.0 * torch.randn(B, T, C, generator=g)
    ctx, pool = _run_asp(x.to(DEV), logits.to(DEV))
    x64, l64 = x.double(), logits.double()
    e = (rel(ctx, _context_ref(x64)), rel(pool, _pool_ref(x64, l64)))
    print(f"[astp T={T}] context {e[0]:.2e} pool {e[1]:.2e}")
    assert max(e) < 4 * 2.0 ** -24 * 4


def test_astp_pool_one_frame_dominates_and_uniform_logits(lib):
    g = torch.Generator().manual_seed(5)
    B, T, C = 2, 41, 64
    x = torch.randn(B, T, C, generator=g)
    logits = torch.full((B, T, C), -300.0)
    t0 = torch.randint(0, T, (B, C), generator=g)
    logits.scatter_(1, t0[:, None, :], 20.0)
    _, pool = _run_asp(x.to(DEV), logits.to(DEV))
    assert torch.equal(pool[:, :C].float(), x.gather(1, t0[:, None, :])[:, 0])     # alpha is one-hot: mean is that frame
    assert (pool[:, C:].float() == torch.from_numpy(np.array(STD_FLOOR))).all()      # var 0 clamps to 1e-7
    flat = torch.full((B, T, C), 3.25)
    _, pool = _run_asp(x.to(DEV), flat.to(DEV))
    x64 = x.double()
    assert rel(pool[:, :C], x64.mean(1)) < 4 * 2.0 ** -24
    assert rel(pool[:, C:], x64.var(1, unbiased=False).clamp(min=1e-7).sqrt()) < 4 * 2.0 ** -24


def test_astp_constant_channel_clamps(lib):
    g = torch.Generator().manual_seed(6)
    B, T, C = 2, 301, 130
    x = torch.rand(B, T, C, generator=g)
    x[:, :, 7] = 0.7
    x[1, :, 129] = 0.0
    ctx, pool = _run_asp(x.to(DEV), torch.randn(B, T, C, generator=g).to(DEV))
    floor = torch.from_numpy(np.array(STD_FLOOR))
    for b, c in ((0, 7), (1, 7), (1, 129)):
        assert ctx[b, C + c].float() == floor and pool[b, C + c].float() == floor
        assert ctx[b, c].float() == x[b, 0, c] and pool[b, c].float() == x[b, 0, c]


def test_asp_tanh_planes(lib):
    from unified_audio_b200 import ops
    g = torch.Generator().manual_seed(7)
    B, T, N, ld = 3, 19, 128, 192
    h, row = torch.randn(B * T, N, generator=g), torch.randn(B, N, generator=g)
    out = _planes((B * T, ld))
    out.hi.fill_(1.0)
    ops.asp_tanh_planes(h.to(DEV), row.to(DEV), B, T, N, out, ld)
    torch.cuda.synchronize()
    want = torch.tanh(h.double() + row.double().repeat_interleave(T, 0))
    got = out.float().cpu().double()
    assert float((got[:, :N] - want).abs().max()) < 1e-6 and not got[:, N:].any()


def _usage(idx, K):
    from unified_audio_b200 import ops
    p, a = torch.full((), -1.0, device=DEV), torch.full((), -1.0, device=DEV)
    counts = torch.full((K,), 77, dtype=torch.int32, device=DEV)          # stale counts: the entry clears them
    ops.fvq_usage(idx.to(DEV).reshape(-1), K, counts, p, a)
    torch.cuda.synchronize()
    want = torch.bincount(idx.reshape(-1), minlength=K)
    assert torch.equal(counts.cpu().long(), want)
    pr = want.double() / idx.numel()
    return float(p), float(a), float(torch.exp(-(pr * torch.log(pr + 1e-10)).sum())), int((want > 0).sum())


def test_fvq_usage_against_fp64(lib):
    K = 8192
    p, a, _, _ = _usage(torch.full((4, 50), 123), K)
    assert p == 1.0 and a == 1.0
    p, a, _, _ = _usage(torch.full((2, 3), K - 1), K)
    assert p == 1.0 and a == 1.0
    p, a, pw, aw = _usage(torch.randperm(K)[:300].reshape(3, 100), K)
    assert a == 300.0 and abs(p - pw) <= 2e-7 * pw and abs(pw - 300.0) < 1e-3
    g = torch.Generator().manual_seed(8)
    idx = torch.randint(0, K, (32, 250), generator=g)
    idx[0, :100] = K - 1
    p, a, pw, aw = _usage(idx, K)
    assert a == aw and abs(p - pw) <= 2e-7 * pw


def test_new_entries_refuse_bad_shapes(lib):
    from unified_audio_b200 import ops
    x = torch.zeros(2 * 5, 64, device=DEV)
    out, pl = torch.zeros(2, 128, device=DEV), _planes((2, 128))
    with pytest.raises(RuntimeError, match="T >= 2"):
        ops.asp_context(x, 10, 1, 64, out, pl, 128)
    with pytest.raises(RuntimeError, match="asp_context"):
        ops.asp_context(x, 2, 5, 64, out, pl, 127)
    with pytest.raises(RuntimeError, match="asp_pool"):
        ops.asp_pool(x, x, 2, 5, 64, out, pl, 96)
    with pytest.raises(RuntimeError, match="asp_tanh_planes"):
        ops.asp_tanh_planes(x, out, 2, 5, 64, _planes((10, 64)), 32)
    p, a = torch.zeros((), device=DEV), torch.zeros((), device=DEV)
    with pytest.raises(RuntimeError, match="fvq_usage"):
        ops.fvq_usage(torch.zeros(0, dtype=torch.int64, device=DEV), 8, torch.zeros(8, dtype=torch.int32, device=DEV), p, a)
    with pytest.raises(RuntimeError, match="fvq_usage"):
        ops.fvq_usage(torch.zeros(4, dtype=torch.int64, device=DEV), 0, torch.zeros(8, dtype=torch.int32, device=DEV), p, a)
    torch.cuda.synchronize()
    assert float(p) == 0.0 and float(a) == 0.0 and not out.any()


# ------------------------------------------------------------------------------------------------------------------------- face
def test_small_face_matches_reference_forward(lib):
    from oracle.make_golden_bicodec_forward import small_config, small_state_dict
    from unified_audio_b200.bicodec import BiCodec
    z = np.load(os.path.join(GOLD, "bicodec_forward_small.npz"))
    cfg = small_config()
    m = BiCodec(cfg, full=True)
    m.load_state_dict(small_state_dict(cfg), strict=True)
    m = m.cuda()
    batch = {k: torch.from_numpy(z[k]).to(DEV) for k in ("feat", "ref_wav", "wav")}
    out = m(batch)
    torch.cuda.synchronize()
    assert set(out) == {"vq_loss", "perplexity", "cluster_size", "recons", "pred_feat", "x_vector", "d_vector", "audios", "with_speaker_loss"}
    e = {k: rel(out[k], z[k]) for k in ("recons", "pred_feat", "x_vector", "d_vector")}
    print("[bicodec forward small] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    for k in ("recons", "pred_feat", "x_vector", "d_vector", "perplexity", "cluster_size", "vq_loss"):
        assert out[k].dtype == torch.float32 and tuple(out[k].shape) == z[k].shape and out[k].is_cuda, k
    assert max(e.values()) < FACE_TOL
    assert abs(float(out["perplexity"]) - float(z["perplexity"])) <= 1e-5 * float(z["perplexity"])
    assert float(out["cluster_size"]) == float(z["cluster_size"])
    assert torch.isnan(out["vq_loss"]) and out["with_speaker_loss"] is False
    assert out["audios"].data_ptr() == batch["wav"].data_ptr() and out["audios"].shape == (3, 1, z["wav"].shape[-1])
    # the reference's self-test on the face: forward's reconstruction is the round trip's, exactly
    assert torch.equal(out["recons"], m.detokenize(*m.tokenize(batch)))
    with pytest.raises(ValueError):
        m(dict(batch, wav=batch["wav"][:2]))


def full_model(seed):
    from oracle import bicodec as ob
    from oracle import bicodec_forward as of
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from unified_audio_b200.bicodec import BiCodec
    sd = dict(ob.make_state_dict(ob.BICODEC_FULL, seed))
    sd.update(osm.make_semantic_state_dict(osm.BICODEC_SEMANTIC_FULL, seed))
    sd.update(og.make_speaker_state_dict(og.BICODEC_GLOBAL_FULL, seed))
    sd.update(of.make_forward_state_dict(of.BICODEC_FORWARD_FULL, seed))
    m = BiCodec(full=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def test_shipped_widths_forward_is_the_round_trip(lib):
    from oracle import bicodec_forward as of
    from oracle import bicodec_semantic as osm
    from oracle.make_golden_bicodec_global import synth_wav
    cfg = of.BICODEC_FORWARD_FULL
    m, sd = full_model(4)
    B, T = 2, 50
    batch = {"feat": osm.synth_feat(B, T, 1024, 41).to(DEV), "ref_wav": synth_wav(B, 16000, 42).to(DEV), "wav": synth_wav(B, 16000, 43).to(DEV)}
    sem0, glob0 = m.tokenize(batch)
    taps = {}
    rec0 = m.detokenize(sem0, glob0, taps=taps)
    gtaps = {}
    m.get_global_tokens(batch, taps=gtaps)
    out = m(batch)
    sem1, glob1 = m.tokenize(batch)
    rec1 = m.detokenize(sem1, glob1)
    torch.cuda.synchronize()
    assert torch.equal(out["recons"], rec0), "forward's reconstruction must be detokenize(*tokenize(batch)) bit for bit"
    assert torch.equal(sem1, sem0) and torch.equal(glob1, glob0) and torch.equal(rec1, rec0), "forward leaked into the token paths"
    assert torch.equal(out["d_vector"], taps["d_vector"])
    sd64 = {k: v.double() for k, v in sd.items()}
    # the new pieces on the device's own intermediates: x-vector from the latent, pred_feat from the prenet output
    xv_own = of.x_vector(sd64, gtaps["latent"].double().cpu().transpose(1, 2))
    pf_own = of.postnet(sd64, cfg, taps["prenet.out"].double().cpu().reshape(B, T, -1).transpose(1, 2))
    # the x-vector end to end against the fp64 oracle (the latent does not depend on any token decision)
    from oracle import bicodec_global as og
    latent = og.ecapa_latent(sd64, og.mel_spectrogram(batch["ref_wav"].double().cpu(), cfg["mel_params"]))
    e = dict(x_vector_own=rel(out["x_vector"], xv_own), pred_feat_own=rel(out["pred_feat"], pf_own),
             x_vector=rel(out["x_vector"], of.x_vector(sd64, latent)))
    print("[bicodec forward shipped B=2 x 1 s] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    assert out["x_vector"].shape == (B, 1024) and out["pred_feat"].shape == (B, 1024, T)
    assert max(e.values()) < FACE_TOL and e["x_vector_own"] < 1e-4
    p, n = of.fvq_usage(sem0.cpu(), 8192)
    assert float(out["cluster_size"]) == n and abs(float(out["perplexity"]) - float(p)) <= 1e-5 * float(p)
