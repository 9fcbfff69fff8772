"""GPU unit parity of every C-ABI op against plain torch fp32/fp64 math on the same device."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def planes_ref(p):
    return p.hi.double() + (p.lo.double() if p.lo is not None else 0.0)


def relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 128), (300, 384, 192), (1000, 1922, 1536), (4096, 4608, 1536)])
def test_gemm_linear(lib, split, M, N, K):
    from unified_audio_b200 import ops
    x, w, bias = _mk((M, K), 1), _mk((N, K), 2, K ** -0.5), _mk((N,), 3)
    a, wp = ops.Planes.from_f32(x, split), ops.Planes.from_f32(w, split)
    out = torch.full((M, N), float("nan"), device=DEV)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias,
             out_f32=ops.rowmap(out, N, M, 0))
    torch.cuda.synchronize()
    ref = planes_ref(a) @ planes_ref(wp).t() + bias.double()
    if split:  # the kernel omits the lo*lo term
        ref = ref - a.lo.double() @ wp.lo.double().t()
    e = relerr(out, ref)
    print(f"gemm split={split} {M}x{N}x{K} relerr={e:.3e}")
    assert e < 2e-5
    if split:
        e_true = relerr(out, x.double() @ w.double().t() + bias.double())
        print(f"   vs fp64 of the fp32 operands: {e_true:.3e}")
        assert e_true < 1e-5


def test_gemm_matches_simt_crosscheck(lib):
    from unified_audio_b200 import ops
    M, N, K = 200, 320, 128
    x, w = _mk((M, K), 5), _mk((N, K), 6, K ** -0.5)
    a, wp = ops.Planes.from_f32(x, True), ops.Planes.from_f32(w, True)
    o1, o2 = torch.zeros(M, N, device=DEV), torch.zeros(M, N, device=DEV)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, out_f32=ops.rowmap(o1, N, M, 0))
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, out_f32=ops.rowmap(o2, N, M, 0), simt=True)
    torch.cuda.synchronize()
    assert relerr(o1, o2) < 1e-5


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("k,s,Cin,Cout,T,B", [(3, 1, 128, 256, 50, 2), (9, 4, 256, 128, 48, 3), (4, 2, 128, 128, 40, 2),
                                               (5, 1, 1024, 1536, 200, 2), (3, 1, 1984, 1536, 96, 1)])
def test_gemm_conv1d(lib, split, k, s, Cin, Cout, T, B):
    """Conv1d over a zero-padded channel-last buffer == F.conv1d (vq/conv.py:35-57)."""
    import torch.nn.functional as F
    from unified_audio_b200 import ops
    pad = (k - 1) // 2 if s > 1 and k % 2 == 0 else k // 2      # semantic_module.py: (k-1)//2 ; conv.py: k//2
    Tp = T + 2 * pad
    Tp += (-Tp) % s
    T_out = (T + 2 * pad - k) // s + 1
    x = _mk((B, T, Cin), 7)
    w = _mk((Cout, Cin, k), 8, (Cin * k) ** -0.5)
    bias = _mk((Cout,), 9)
    buf = ops.Planes.zeros((B, Tp, Cin), split, DEV)
    ops.rows_to_planes(x.reshape(B * T, Cin), B, T, Cin, buf, Cin, Tp, pad)
    wp = ops.Planes.from_f32(w.permute(0, 2, 1).reshape(Cout, k * Cin), split)
    out = torch.full((B, T_out, Cout), float("nan"), device=DEV)
    ops.gemm(buf, wp, Cout, a_batch=B, a_rows_per_batch=Tp, a_ld=Cin, m_per_batch=T_out, taps=k, stride=s, bias=bias,
             out_f32=ops.rowmap(out, Cout, T_out, 0))
    torch.cuda.synchronize()
    xq = planes_ref(ops.Planes(buf.hi[:, pad:pad + T], buf.lo[:, pad:pad + T] if split else None))
    ref = F.conv1d(xq.transpose(1, 2), planes_ref(wp).reshape(Cout, k, Cin).permute(0, 2, 1), bias.double(), stride=s,
                   padding=pad).transpose(1, 2)
    e = relerr(out, ref)
    print(f"conv k{k}s{s} {Cin}->{Cout} T{T} split={split} relerr={e:.3e}")
    assert out.shape == ref.shape and e < 3e-5


def test_gemm_epilogues(lib):
    """the 3-term <3,128,3> kernel against the fp64 product of the fp32 operands"""
    _gemm_epilogues(True)


def test_gemm_epilogues_single_pass(lib):
    """the same epilogues on the single-pass 256-wide tile (N = 512) against the fp64 product of the fp16 operands it reads"""
    _gemm_epilogues(False)


def _gemm_epilogues(split):
    import torch.nn.functional as F
    from unified_audio_b200 import ops
    M, N, K = 260, 512, 256
    x, w, bias, gamma, res = _mk((M, K), 11), _mk((N, K), 12, K ** -0.5), _mk((N,), 13), _mk((N,), 14), _mk((M, N), 15)
    a, wp = ops.Planes.from_f32(x, split), ops.Planes.from_f32(w, split)
    acc = (x.double() @ w.double().t()) if split else planes_ref(a) @ planes_ref(wp).t()
    # GELU -> planes
    outp = ops.Planes.zeros((M, N), True, DEV)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias, act=ops.ACT_GELU,
             out_planes=outp, out_planes_map=(N, M, 0))
    torch.cuda.synchronize()
    assert relerr(planes_ref(outp), F.gelu(acc + bias.double())) < 2e-5
    # gamma + residual in place
    r2 = res.clone()
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias, gamma=gamma,
             residual=ops.rowmap(r2, N, M, 0), out_f32=ops.rowmap(r2, N, M, 0))
    torch.cuda.synchronize()
    assert relerr(r2, (acc + bias.double()) * gamma.double() + res.double()) < 2e-5
    # SwiGLU pairs
    o = torch.zeros(M, N // 2, device=DEV)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, act=ops.ACT_SWIGLU,
             out_f32=ops.rowmap(o, N // 2, M, 0))
    torch.cuda.synchronize()
    assert relerr(o, F.silu(acc[:, 0::2]) * acc[:, 1::2]) < 2e-5
    # ELU only on the plane output, fp32 output pre-activation, padded destination
    o32 = torch.zeros(M, N, device=DEV)
    dst = ops.Planes.zeros((1, M + 2, N), True, DEV)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, act2=ops.ACT_ELU,
             out_f32=ops.rowmap(o32, N, M, 0), out_planes=dst, out_planes_map=(N, M + 2, 1))
    torch.cuda.synchronize()
    assert relerr(o32, acc) < 2e-5
    assert relerr(planes_ref(dst)[0, 1:-1], F.elu(acc)) < 2e-5
    assert float(dst.hi[0, 0].abs().max()) == 0 and float(dst.hi[0, -1].abs().max()) == 0


def test_norms_and_dwconv(lib):
    import torch.nn.functional as F
    from unified_audio_b200 import ops
    B, T, Cc = 3, 37, 256
    x = _mk((B, T, Cc), 21) * 2 + 0.3
    w, b = _mk((Cc,), 22) * 0.1 + 1, _mk((Cc,), 23) * 0.1
    out = torch.zeros_like(x)
    p = ops.Planes.zeros((B, T, Cc), True, DEV)
    ops.layernorm(x, w, b, B, T, Cc, out_f32=out, out=p)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.double(), (Cc,), w.double(), b.double(), 1e-6)
    assert relerr(out, ref) < 1e-5 and relerr(planes_ref(p), ref) < 1e-5
    p2 = ops.Planes.zeros((B * T, Cc), True, DEV)
    ops.rmsnorm(x, w, B * T, Cc, p2)
    torch.cuda.synchronize()
    assert relerr(planes_ref(p2).reshape(B, T, Cc), F.rms_norm(x.double(), (Cc,), w.double(), 1e-6)) < 1e-5
    dw_w, dw_b = _mk((Cc, 7), 24, 0.3), _mk((Cc,), 25, 0.1)
    p3 = ops.Planes.zeros((B, T, Cc), True, DEV)
    ops.dwconv7_ln(x, dw_w, dw_b, w, b, B, T, Cc, p3)
    torch.cuda.synchronize()
    h = F.conv1d(x.double().transpose(1, 2), dw_w.double()[:, None, :], dw_b.double(), padding=3, groups=Cc).transpose(1, 2)
    assert relerr(planes_ref(p3), F.layer_norm(h, (Cc,), w.double(), b.double(), 1e-6)) < 1e-5
    # group norm (+swish) into a padded buffer
    stats = torch.zeros(B, 32, 2, device=DEV)
    ops.groupnorm_stats(x, B, T, Cc, stats)
    dst = ops.Planes.zeros((B, T + 2, Cc), True, DEV)
    o32 = torch.zeros_like(x)
    ops.groupnorm_apply(x, stats, w, b, B, T, Cc, True, out_f32=o32, out=dst, ld=Cc, rows_per_batch=T + 2, row_off=1)
    torch.cuda.synchronize()
    g = F.group_norm(x.double().transpose(1, 2), 32, w.double(), b.double(), 1e-6).transpose(1, 2)
    g = g * torch.sigmoid(g)
    assert relerr(o32, g) < 1e-5 and relerr(planes_ref(dst)[:, 1:-1], g) < 1e-5


def test_attention_hd(lib):
    """fp32 SIMT attention (attention_kernel<64, 32>) against fp64 softmax attention with RoPE"""
    from unified_audio_b200 import ops
    B, T, H, D = 2, 150, 4, 64
    qkv = _mk((B, T, 3 * H * D), 31)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    fr = torch.arange(T).float()[:, None] * inv[None]
    emb = torch.cat([fr, fr], -1)
    cos, sin = emb.cos().to(DEV).contiguous(), emb.sin().to(DEV).contiguous()
    out = ops.Planes.zeros((B, T, H * D), True, DEV)
    ops.attention_hd(qkv, B, T, H, D, cos, sin, out)
    torch.cuda.synchronize()
    q, k, v = [t.reshape(B, T, H, D).transpose(1, 2).double() for t in qkv.chunk(3, -1)]
    rot = lambda x: torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1)
    c, s = cos.double(), sin.double()
    q, k = q * c + rot(q) * s, k * c + rot(k) * s
    att = torch.softmax(q @ k.transpose(2, 3) * D ** -0.5, -1)
    ref = (att @ v).transpose(1, 2).reshape(B, T, H * D)
    e = relerr(planes_ref(out), ref)
    print("attention relerr", e)
    assert e < 1e-5


def test_attention_tc_alias(lib):
    """ops.attention_tc (a name bench.py's FLOP counter wraps) is the single-pass wgmma attention at head_dim 64, bit for bit"""
    from unified_audio_b200 import ops
    B, T, H, D = 2, 150, 4, 64
    qkv = _mk((B, T, 3 * H * D), 32)
    cos, sin = ops.rope_tables(T, D, DEV)
    n = ops.attention_tc_workspace_bytes(B, T, H)
    assert n == ops.attention_umma_workspace_bytes(B, T, H, D, False)
    tc, umma = ops.Planes.zeros((B, T, H * D), False, DEV), ops.Planes.zeros((B, T, H * D), False, DEV)
    ops.attention_tc(qkv, B, T, H, cos, sin, tc, torch.zeros(n, dtype=torch.uint8, device=DEV))
    ops.attention_umma(qkv, B, T, H, D, cos, sin, umma, torch.zeros(n, dtype=torch.uint8, device=DEV), split=False)
    torch.cuda.synchronize()
    assert bool(umma.hi.abs().max() > 0) and torch.equal(tc.hi, umma.hi)


@pytest.mark.parametrize("D,split", [(64, True), (64, False), (128, True), (128, False)])
@pytest.mark.parametrize("B,T,H", [(2, 37, 3), (1, 64, 2), (3, 250, 8), (2, 382, 4), (1, 515, 2)])
def test_attention_umma(lib, D, split, B, T, H):
    """wgmma attention (csrc/attention_umma.cu) against fp64 softmax attention; ragged lengths exercise the TMA zero fill of the
    last query / key tiles, 515 the 9-tile K/V ring; and against the fp32 SIMT kernel it replaces"""
    from unified_audio_b200 import ops
    qkv = _mk((B, T, 3 * H * D), 31 + T)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2).float() / D))
    fr = torch.arange(T).float()[:, None] * inv[None]
    emb = torch.cat([fr, fr], -1)
    cos, sin = emb.cos().to(DEV).contiguous(), emb.sin().to(DEV).contiguous()
    out = ops.Planes.zeros((B, T, H * D), split, DEV)
    ws = torch.zeros(ops.attention_umma_workspace_bytes(B, T, H, D, split), dtype=torch.uint8, device=DEV)
    ops.attention_umma(qkv, B, T, H, D, cos, sin, out, ws)
    torch.cuda.synchronize()
    q, k, v = [t.reshape(B, T, H, D).transpose(1, 2).double() for t in qkv.chunk(3, -1)]
    rot = lambda x: torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1)
    c, s = cos.double(), sin.double()
    q, k = q * c + rot(q) * s, k * c + rot(k) * s
    att = torch.softmax(q @ k.transpose(2, 3) * D ** -0.5, -1)
    ref = (att @ v).transpose(1, 2).reshape(B, T, H * D)
    got = planes_ref(out) if split else out.hi.double()
    e = relerr(got, ref)
    print(f"attention_umma D={D} split={split} B={B} T={T} H={H}: relerr {e:.2e}")
    assert e < (2e-5 if split else 3e-3)
    simt = ops.Planes.zeros((B, T, H * D), True, DEV)
    ops.attention_hd(qkv, B, T, H, D, cos, sin, simt)
    torch.cuda.synchronize()
    assert relerr(got, planes_ref(simt)) < (2e-5 if split else 3e-3)
    # causal mode (the AR-LM's prefill / teacher-forced attention): key tiles past the diagonal are skipped, the diagonal tiles masked
    ops.attention_umma(qkv, B, T, H, D, cos, sin, out, ws, causal=True)
    torch.cuda.synchronize()
    mask = torch.ones(T, T, dtype=torch.bool, device=DEV).tril()
    attc = torch.softmax((q @ k.transpose(2, 3) * D ** -0.5).masked_fill(~mask, float("-inf")), -1)
    refc = (attc @ v).transpose(1, 2).reshape(B, T, H * D)
    ec = relerr(planes_ref(out) if split else out.hi.double(), refc)
    print(f"   causal: relerr {ec:.2e}")
    assert ec < (2e-5 if split else 3e-3)


@pytest.mark.parametrize("B,T,H", [(2, 9, 256), (3, 20, 512), (5, 12, 1536), (70, 6, 512), (130, 5, 256)])
def test_lstm_tc(lib, B, T, H):
    from unified_audio_b200 import ops
    k = 1.0 / math.sqrt(H)
    g = torch.Generator().manual_seed(41)
    whh = ((torch.rand(4 * H, H, generator=g) * 2 - 1) * k).to(DEV)
    xp = _mk((B, T, 4 * H), 42)
    U = ops.lstm_tc_units(H)
    out = ops.Planes.zeros((B, T, H), True, DEV)
    ws = torch.zeros(ops.lstm_tc_workspace_bytes(B, H), dtype=torch.uint8, device=DEV)
    ops.lstm_tc(xp, ops.lstm_tc_permute(whh, U), U, B, T, H, out, ws)
    torch.cuda.synchronize()
    # reference recurrence in fp64 with the same fp16-rounded operands (W_hh and h_{t-1})
    W = whh.half().double()
    h = torch.zeros(B, H, dtype=torch.float64, device=DEV)
    c = torch.zeros_like(h)
    outs = []
    for t in range(T):
        gts = xp[:, t].double() + h.half().double() @ W.t()
        i, f, gg, o = gts.chunk(4, -1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        outs.append(h)
    ref = torch.stack(outs, 1)
    e = relerr(planes_ref(out), ref)
    print(f"lstm_tc B{B} T{T} H{H} U{U} relerr {e:.3e}")
    # fp16 re-rounding of h can flip one ulp on a knife edge; exact-model error is ~1e-6
    assert e < 2e-3 and relerr(planes_ref(out)[:, 0], ref[:, 0]) < 1e-5


def test_spectral(lib):
    from unified_audio_b200 import ops
    B, F_, n_fft = 2, 7, 1920
    hop, nf = n_fft // 2, n_fft // 2 + 1
    P, Q = 64, 30                                  # two-stage STFT factors of n_fft (include/quark_b200.h)
    T, M = F_ * hop, B * F_
    # gather: row (clip, f, b), col a = pad(wav)[hop f + Q a + b] * window[Q a + b]
    wav = _mk((B, T), 51, 0.1)
    win = _mk((n_fft,), 55).abs()
    ga = ops.Planes.zeros((M * Q, 64), True, DEV)
    ops.stft_gather(wav, hop, n_fft, P, Q, win, ga)
    torch.cuda.synchronize()
    pad = (n_fft - hop) // 2
    xw = torch.nn.functional.pad(wav.double(), (pad, pad)).unfold(1, n_fft, hop) * win.double()       # [B, F, n_fft]
    assert xw.shape[1] == F_
    assert relerr(planes_ref(ga), xw.reshape(B, F_, P, Q).transpose(2, 3).reshape(M * Q, P)) < 1e-6
    # twiddle: row (clip-frame, k1), cols b / Q + b = re / im of Y[(clip-frame, b), k1] * (cos, -sin)(2 pi k1 b / n_fft)
    Y = _mk((M * Q, 2 * P), 52)
    ang = 2 * math.pi * torch.arange(Q, dtype=torch.float64)[:, None] * torch.arange(P, dtype=torch.float64)[None] / n_fft
    tw = torch.stack([torch.cos(ang), -torch.sin(ang)], -1).reshape(Q * P, 2).float().to(DEV)
    Z = ops.Planes.zeros((M * P, 128), True, DEV)
    ops.stft_twiddle(Y, 2 * P, M, P, Q, tw, Z)
    torch.cuda.synchronize()
    yc = torch.view_as_complex(Y.double().reshape(M, Q, P, 2).contiguous())
    z = (yc * torch.view_as_complex(tw.double().reshape(Q, P, 2).contiguous())).transpose(1, 2)            # [M, P, Q]
    got = planes_ref(Z).reshape(M, P, 128)
    assert relerr(got[..., :Q], z.real) < 1e-6 and relerr(got[..., Q:2 * Q], z.imag) < 1e-6
    # post2: X[k] at row (clip, f, k % P), cols 2 (k / P), 2 (k / P) + 1 -> log(clip(|X|, 1e-5)), angle / pi, zero pad columns
    K2 = (nf - 1) // P + 1
    ldX = (2 * K2 + 3) // 4 * 4
    X = _mk((M * P, ldX), 56)
    dst = ops.Planes.zeros((B, F_ + 2, 1984), True, DEV)
    dst.hi.fill_(1.0)
    dst.lo.fill_(1.0)                              # the padding columns must be written, not left as they were
    ops.stft_post2(X, ldX, B, F_, nf, P, dst, 1984, F_ + 2, 1)
    torch.cuda.synchronize()
    k = torch.arange(nf)
    Xr = X.double().reshape(M, P, ldX)
    re, im = Xr[:, k % P, 2 * (k // P)], Xr[:, k % P, 2 * (k // P) + 1].clone()
    im[:, 0] = 0; im[:, -1] = 0
    mag = torch.log(torch.clip(torch.sqrt(re * re + im * im), min=1e-5))
    ph = torch.atan2(im, re) / math.pi
    got = planes_ref(dst)[:, 1:-1].reshape(M, 1984)
    assert relerr(got[:, :nf], mag) < 1e-5 and relerr(got[:, nf:2 * nf], ph) < 1e-5
    assert float(got[:, 2 * nf:].abs().max()) == 0
    head = _mk((B * F_, 2 * nf), 53)
    sp = ops.Planes.zeros((B * F_, 1984), True, DEV)
    ops.istft_pre(head, 2 * nf, B * F_, nf, sp, 1984)
    torch.cuda.synchronize()
    m = torch.clip(torch.exp(head[:, :nf].double()), max=100.0)
    assert relerr(planes_ref(sp)[:, :nf], m * torch.cos(head[:, nf:].double())) < 1e-5
    assert relerr(planes_ref(sp)[:, nf:2 * nf], m * torch.sin(head[:, nf:].double())) < 1e-5
    frames = _mk((B, F_, n_fft), 54)
    win = torch.hann_window(n_fft).to(DEV)
    y = torch.zeros(B, T, device=DEV)
    ops.istft_ola(frames, win, B, F_, n_fft, y)
    torch.cuda.synchronize()
    out_size = (F_ - 1) * hop + n_fft
    fold = lambda z: torch.nn.functional.fold(z, (1, out_size), (1, n_fft), stride=(1, hop))[:, 0, 0, hop // 2:-(hop // 2)]
    ref = fold(frames.transpose(1, 2)) / fold(win.square().expand(1, F_, -1).transpose(1, 2))
    assert relerr(y, ref) < 1e-6


def test_rvq(lib):
    import sys
    from unified_audio_b200 import ops
    from unified_audio_b200.rvq import ResidualVQ
    from oracle import rvq as orvq
    torch.manual_seed(0)
    M, D, K, nq = 1000, 128, 256, 4
    cb = torch.stack([torch.randn(K, D) * 0.35 * 0.85 ** q for q in range(nq)], 0)
    x = torch.randn(M, D)
    vq = ResidualVQ(dim=D, codebook_size=K, num_quantizers=nq).to(DEV)
    vq.set_codebooks(cb.to(DEV))
    quant, idx, _ = vq(x.to(DEV).reshape(1, M, D))
    oidx, oquant = orvq.rvq_encode(x, cb)
    tidx, margin = orvq.rvq_margin_audit(x, cb, oidx)
    idx = idx.reshape(M, nq).cpu()
    safe = margin > 1e-5
    print("rvq mismatches vs fp32 oracle:", int((idx != oidx).sum()), " min margin", float(margin.min()))
    assert bool((idx[safe.all(-1)] == oidx[safe.all(-1)]).all())
    assert bool((idx == tidx).all()) or int((idx != tidx).sum()) <= 0
    assert relerr(quant.reshape(M, D).cpu(), oquant) < 1e-6
    dec = vq.get_output_from_indices(idx.reshape(1, M, nq).to(DEV))
    assert torch.equal(dec.reshape(M, D).cpu(), orvq.rvq_decode(idx, cb))
