"""GPU parity of BiCodec.get_semantic_tokens (Encoder -> FVQ tokenize), BiCodec.tokenize and unise.BiCodecTokenizer.tokenize against
the outputs of the reference's own classes (tests/golden/bicodec_semantic_small.npz) and the fp64 oracle on the shipped
configuration, and of qb_fvq_tokenize alone against fp64.

Token rule on the shipped configuration: scores are 2 e.c - |c|^2 with |c| = 1, so a token can only change where the oracle's margin
(best minus second-best score) is below 2 max_row |e_gpu - e_oracle|; TAU = max(20 max_row |e_gpu - e_oracle|, 1e-6) leaves a 10x
safety factor.  Tokens must be equal wherever the margin is >= TAU; flips below TAU are counted and printed."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
FLOAT_TOL = 5e-5                 # the budget of the other 3-term-split paths' float taps


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def small_model():
    from oracle.make_golden_bicodec_semantic import small_config, small_state_dict
    from unified_audio_b200.bicodec import BiCodec
    z = np.load(os.path.join(GOLD, "bicodec_semantic_small.npz"))
    meta = json.loads(str(z["meta"]))
    cfg = small_config()
    sd = small_state_dict(cfg, meta["seed"])
    m = BiCodec(cfg, global_tokens=True, semantic_tokens=True)
    m.load_state_dict(sd, strict=True)
    return z, meta, cfg, m.cuda(), sd


def full_model(seed=1, global_tokens=False):
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from unified_audio_b200.bicodec import BiCodec
    sd = dict(ob.make_state_dict(ob.BICODEC_FULL, seed))
    sd.update(osm.make_semantic_state_dict(osm.BICODEC_SEMANTIC_FULL, seed))
    if global_tokens:
        sd.update(og.make_speaker_state_dict(og.BICODEC_GLOBAL_FULL, seed))
    m = BiCodec(global_tokens=global_tokens, semantic_tokens=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def test_small_fixture_matches_reference(lib):
    z, meta, cfg, m, _ = small_model()
    feat = torch.from_numpy(z["feat"]).cuda()
    taps = {}
    tok = m.get_semantic_tokens({"feat": feat}, taps=taps)
    torch.cuda.synchronize()
    e = dict(encoder=rel(taps["encoder"], z["encoder"]), z_e=rel(taps["z_e"], z["z_e"]))
    print("[bicodec semantic small] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    assert tok.dtype == torch.int64 and tok.shape == (meta["B"], meta["T"])
    assert torch.equal(tok.cpu(), torch.from_numpy(z["tokens"])) and max(e.values()) < FLOAT_TOL
    assert torch.equal(m.get_semantic_tokens(feat).cpu(), tok.cpu())                 # a bare tensor is taken too
    sem, glob = m.tokenize({"feat": feat, "ref_wav": torch.from_numpy(z["ref_wav"]).cuda()})
    assert torch.equal(sem.cpu(), tok.cpu()) and torch.equal(glob.cpu(), torch.from_numpy(z["global_tokens"]))
    # fresh outputs: a later call does not overwrite an earlier result
    m.get_semantic_tokens(feat.flip(1).contiguous())
    torch.cuda.synchronize()
    assert torch.equal(tok.cpu(), torch.from_numpy(z["tokens"]))
    with pytest.raises(ValueError):
        m.get_semantic_tokens(feat[..., :32].contiguous())
    with pytest.raises(RuntimeError):
        m.get_semantic_tokens(feat.cpu())


def compare_tokens(got, z_e_gpu, want, z_e_ref, margins, label):
    e_gpu = torch.nn.functional.normalize(z_e_gpu.double().cpu(), dim=-1)
    e_ref = torch.nn.functional.normalize(z_e_ref.double().cpu(), dim=-1)
    de = float((e_gpu - e_ref).norm(dim=-1).max())
    tau = max(20 * de, 1e-6)
    safe = margins >= tau
    g, w = got.cpu(), want.cpu()
    assert torch.equal(g[safe], w[safe]), f"{label}: token differs where the margin is >= tau"
    flips = int((g[~safe] != w[~safe]).sum())
    print(f"[{label}] tau {tau:.2e} (max |de| {de:.2e}), tokens below tau {int((~safe).sum())} of {g.numel()}, flips {flips}, "
          f"smallest margin {float(margins.min()):.2e}")
    return tau


def test_full_config_matches_oracle_and_is_batch_independent(lib):
    from oracle import bicodec as ob
    from oracle import bicodec_semantic as osm
    cfg = osm.BICODEC_SEMANTIC_FULL
    m, sd = full_model(3)
    feat = osm.synth_feat(3, 299, cfg["encoder"]["input_channels"], 31)
    sd64 = {k: v.double() for k, v in sd.items()}
    want_taps = {}
    want = osm.get_semantic_tokens(sd64, cfg, feat[:2].double(), want_taps)
    taps = {}
    got = m.get_semantic_tokens({"feat": feat[:2].cuda()}, taps=taps)
    torch.cuda.synchronize()
    e = dict(encoder=rel(taps["encoder"], want_taps["encoder"]), z_e=rel(taps["z_e"], want_taps["z_e"]))
    print("[bicodec semantic full B=2 x 299] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    assert got.shape == (2, 299) and got.dtype == torch.int64 and max(e.values()) < FLOAT_TOL
    compare_tokens(got, taps["z_e"], want, want_taps["z_e"], osm.fvq_margins(sd64, want_taps["encoder"]), "full")
    # a clip's tokens do not depend on its batch, and a call is deterministic
    three = m.get_semantic_tokens(feat.cuda())
    again = m.get_semantic_tokens(feat.cuda())
    alone = torch.cat([m.get_semantic_tokens(feat[i:i + 1].cuda()) for i in range(3)], 0)
    torch.cuda.synchronize()
    assert torch.equal(three, alone) and torch.equal(three, again) and torch.equal(three[:2], got)
    # the tokens are what detokenize takes
    _, glob = ob.synth_tokens(cfg, 2, 9, 77)
    wav = m.detokenize(got[:, :9], glob.cuda())
    ref = ob.detokenize(sd, cfg, got[:, :9].cpu(), glob)
    torch.cuda.synchronize()
    assert wav.shape == (2, 1, 9 * 320) and rel(wav, ref) < 1e-3


def fvq_reference(z, w, b, cb):
    """fp64 torch restatement of the kernel's contract (on the device: the largest case has 79 M scores) -> (idx [M], margin of the
    best score over the second best [M], z_e [M, cdim]), on the host"""
    z, w, b, cb = (t.cuda().double() for t in (z, w, b, cb))
    z_e = z @ w.t() + b
    e = torch.nn.functional.normalize(z_e, dim=1)
    cbn = torch.nn.functional.normalize(cb, dim=1)
    s = 2 * e @ cbn.t() - cbn.pow(2).sum(1)
    top = s.topk(min(2, s.shape[1]), dim=1).values
    return s.max(1)[1].cpu(), (top[:, 0] - top[:, -1]).cpu(), z_e.cpu()


def run_fvq(z, w, b, cb, pad=5):
    from unified_audio_b200 import ops
    M, D = z.shape
    K, cdim = cb.shape
    cbn = torch.nn.functional.normalize(cb.double(), dim=1).cuda()
    idx = torch.full((M + pad,), -7, dtype=torch.int64, device="cuda")
    z_e = torch.full(((M + pad) * cdim,), float("nan"), device="cuda")
    ops.fvq_tokenize(z.cuda().contiguous(), M, D, w.cuda().contiguous(), b.cuda().contiguous(), cbn, K, cdim, idx, z_e)
    torch.cuda.synchronize()
    assert bool((idx[M:] == -7).all()) and bool(z_e[M * cdim:].isnan().all()), "written past M"
    return idx[:M].cpu(), z_e[:M * cdim].reshape(M, cdim).cpu()


@pytest.mark.parametrize("K", [256, 1000, 8192])
@pytest.mark.parametrize("M", [1, 37, 9600])
def test_fvq_tokenize_kernel_fp64(lib, K, M):
    g = torch.Generator().manual_seed(K * 7 + M)
    D, cdim = 1024, 8
    z = torch.randn(M, D, generator=g)
    w = torch.randn(cdim, D, generator=g) / D ** 0.5
    b = 0.1 * torch.randn(cdim, generator=g)
    cb = torch.randn(K, cdim, generator=g)
    idx, z_e = run_fvq(z, w, b, cb)
    want, margin, ze_ref = fvq_reference(z, w, b, cb)
    assert float((z_e.double() - ze_ref).abs().max()) <= 1e-6 * float(ze_ref.abs().max())
    safe = margin >= 1e-12                  # both sides are fp64: only the summation order differs
    assert torch.equal(idx[safe], want[safe])
    print(f"[fvq K={K} M={M}] margins below 1e-12: {int((~safe).sum())}, distinct codes {len(set(idx.tolist()))}")


@pytest.mark.parametrize("cdim", [3, 8, 16])
def test_fvq_tokenize_kernel_ties_and_zero_rows(lib, cdim):
    """z_e = z (identity in_project, no bias): rows planted on codebook entries that occur several times, and all-zero rows that
    must pick the first all-zero codebook row; the lowest index wins every exact tie."""
    g = torch.Generator().manual_seed(cdim)
    K = 300
    cb = torch.randn(K, cdim, generator=g)
    cb[100] = 2.0 * cb[3]                   # same direction: normalises to the same code
    cb[200] = cb[3]
    cb[250] = cb[40]
    cb[5] = 0.0
    cb[9] = 0.0
    z = torch.randn(64, cdim, generator=g)
    z[0], z[1], z[2], z[3] = cb[3], cb[200], 3.0 * cb[40], cb[250]
    z[4] = 0.0
    z[5] = 0.0
    w, b = torch.eye(cdim), torch.zeros(cdim)
    idx, z_e = run_fvq(z, w, b, cb)
    assert idx[:6].tolist() == [3, 3, 40, 40, 5, 5]
    want, _, _ = fvq_reference(z, w, b, cb)
    assert torch.equal(idx, want) and torch.equal(z_e, z)


def test_fvq_tokenize_refuses_bad_shapes(lib):
    from unified_audio_b200 import ops
    z, w, b = torch.zeros(4, 17, device="cuda"), torch.zeros(17, 17, device="cuda"), torch.zeros(17, device="cuda")
    cb = torch.zeros(8, 17, dtype=torch.float64, device="cuda")
    idx = torch.zeros(4, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="codebook_dim"):
        ops.fvq_tokenize(z, 4, 17, w, b, cb, 8, 17, idx)
    with pytest.raises(RuntimeError, match="bad args"):
        ops.fvq_tokenize(z, 4, 17, w, b, cb, 0, 8, idx)


def test_tokenizer_end_to_end_small_matches_reference(lib):
    from oracle import wav2vec2 as ow
    from oracle.make_golden_bicodec_semantic import e2e_wav2vec2_config
    from unified_audio_b200.ssl import SSLFrontEnd
    from unified_audio_b200.unise import BiCodecTokenizer
    z, meta, cfg, m, _ = small_model()
    wc = e2e_wav2vec2_config()
    w2v = SSLFrontEnd(dict(wc, kind="wav2vec2", do_normalize=True), in_rate=16000)
    w2v.load_state_dict(ow.make_state_dict(wc, meta["w2v_seed"]), strict=True)
    tok = BiCodecTokenizer(m, ref_segment_length=meta["ref_segment_length"], feature_extractor=w2v.cuda())
    glob, sem = tok.tokenize(torch.from_numpy(z["e2e_wav"]).cuda())
    torch.cuda.synchronize()
    assert glob.dtype == torch.int32 and sem.dtype == torch.int64
    assert torch.equal(glob.cpu(), torch.from_numpy(z["e2e_global"])) and torch.equal(sem.cpu(), torch.from_numpy(z["e2e_semantic"]))


def test_tokenizer_end_to_end_full_config(lib):
    from oracle import wav2vec2 as ow
    from oracle.make_golden_bicodec_global import synth_wav
    from unified_audio_b200.ssl import WAV2VEC2_XLSR53, SSLFrontEnd
    from unified_audio_b200.unise import BiCodecTokenizer
    m, _ = full_model(2, global_tokens=True)
    w2v = SSLFrontEnd(WAV2VEC2_XLSR53, in_rate=16000)
    w2v.load_state_dict(ow.make_state_dict(ow.WAV2VEC2_XLSR53, 5), strict=True)
    w2v = w2v.cuda()
    tok = BiCodecTokenizer(m, feature_extractor=w2v)
    wav = synth_wav(2, 96000, 12).cuda()
    glob, sem = tok.tokenize(wav)
    want_g = m.get_global_tokens({"ref_wav": tok.get_ref_clip(wav)})
    want_s = m.get_semantic_tokens({"feat": w2v(wav)})
    torch.cuda.synchronize()
    assert glob.dtype == torch.int32 and glob.shape == (2, 1, 32) and sem.dtype == torch.int64 and sem.shape == (2, 299)
    assert torch.equal(glob, want_g) and torch.equal(sem, want_s)
    out = tok.detokenize(glob, sem)
    torch.cuda.synchronize()
    assert out.shape == (2, 1, 299 * 320) and bool(torch.isfinite(out).all())
