"""The BiCodec global-token kernels of csrc/speaker.cu (mel framing, spectrum magnitude, Res2Net sums, squeeze-excitation and
FSQ) one by one against plain fp64 / exactly rounded references, at the shapes and edges where each can go wrong: reflect padding
at both ends of a frame, factorisations other than the shipped one, grid-stride trips, channel counts above the block size, every
FSQ code of several level sets.  Outputs start as sentinels, so each test also checks what must stay untouched."""
import itertools
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF_SENTINEL = -1234.0          # exact in fp16, produced by none of these kernels
F32_SENTINEL = -4321.0
U32 = 2.0 ** -24                 # unit roundoff of fp32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _split(v32: torch.Tensor):
    """torch's hi / lo split of fp32 values, the planes every kernel here writes: hi = rn_fp16(v), lo = rn_fp16(v - hi)"""
    from unified_audio_b200.ops import Planes
    p = Planes.from_f32(v32.float(), True)
    return p.hi, p.lo


def _sentinel_planes(shape):
    from unified_audio_b200.ops import Planes
    return Planes(torch.full(shape, HALF_SENTINEL, dtype=torch.float16, device=DEV),
                  torch.full(shape, HALF_SENTINEL, dtype=torch.float16, device=DEV))


# ----------------------------------------------------------------------------------------------------------------- mel_gather
def _mel_gather_ref(wav, hop, n_fft, P, Q, win):
    """reflect-pad by n_fft / 2 + unfold x window in fp64, each product rounded once to fp32 (the kernel's one multiply), in the
    kernel's layout: row (clip, f, b), column a = sample Q a + b of the frame; columns P..63 zero"""
    B, L = wav.shape
    xpad = F.pad(wav.double().cpu()[:, None], (n_fft // 2, n_fft // 2), mode="reflect")[:, 0]
    fr = (xpad.unfold(-1, n_fft, hop) * win.double().cpu()).float()                  # [B, F, n_fft]
    Fn = fr.shape[1]
    assert Fn == 1 + L // hop
    v = torch.zeros(B * Fn * Q, 64)
    v[:, :P] = fr.reshape(B, Fn, P, Q).transpose(2, 3).reshape(B * Fn * Q, P)
    return v


@pytest.mark.parametrize("B,L,hop,n_fft,P,Q,win_length", [
    (2, 16000, 320, 1024, 64, 16, 640),      # the shipped mel: hann(640) zero-padded to n_fft 1024
    (2, 16000 + 123, 320, 1024, 64, 16, 640),  # L not a multiple of hop
    (3, 513, 320, 1024, 64, 16, 1024),       # L = n_fft / 2 + 1: frames reflect at both ends
    (2, 7919, 160, 640, 40, 16, 640),        # P < 64: columns 40..63 zero
    (1, 321, 160, 640, 40, 16, 400),         # shortest clip of that factorisation
    (4, 96000, 320, 1024, 64, 16, 640),      # 1.2 M elements: the capped grid takes a second grid-stride trip
])
def test_mel_gather_matches_reflect_unfold(lib, B, L, hop, n_fft, P, Q, win_length):
    from unified_audio_b200 import ops
    from unified_audio_b200.bicodec import hann_window
    wav = torch.randn(B, L, generator=_gen(L + B)) * 0.3
    win = hann_window(dict(n_fft=n_fft, win_length=win_length)).float()
    if win_length == n_fft:
        win = win + torch.rand(n_fft, generator=_gen(5)) * 0.1     # no zero taps: every sample of both reflected ends is read
    want = _mel_gather_ref(wav, hop, n_fft, P, Q, win)
    out = _sentinel_planes(tuple(want.shape))
    ops.mel_gather(wav.to(DEV), hop, n_fft, P, Q, win.to(DEV), out)
    torch.cuda.synchronize()
    hi, lo = _split(want)
    assert torch.equal(out.hi.cpu(), hi) and torch.equal(out.lo.cpu(), lo), \
        f"mel_gather: {int((out.hi.cpu() != hi).sum())} hi values differ from the rounded fp64 frames (columns P..63 zero)"


def test_mel_gather_refuses_before_launch(lib):
    from unified_audio_b200 import ops
    win = torch.ones(1024, device=DEV)
    out = _sentinel_planes((2 * 16, 64))
    with pytest.raises(RuntimeError, match="reflect padding"):
        ops.mel_gather(torch.randn(1, 512, device=DEV), 320, 1024, 64, 16, win, out)      # L = n_fft / 2
    with pytest.raises(RuntimeError, match="n_fft == P"):
        ops.mel_gather(torch.randn(1, 4000, device=DEV), 320, 1024, 64, 15, win, out)     # P * Q != n_fft
    torch.cuda.synchronize()
    assert bool((out.hi == HALF_SENTINEL).all()) and bool((out.lo == HALF_SENTINEL).all())


# ------------------------------------------------------------------------------------------------------------- spec_magnitude
@pytest.mark.parametrize("n_fft,P,M", [(1024, 64, 7), (640, 40, 5)])
def test_spec_magnitude(lib, n_fft, P, M):
    """|X[k]| from the second DFT stage's layout (row k % P, column pair k / P) with the minimal legal ldX; DC and Nyquist carry
    nonzero imaginary parts, which the kernel drops (|re| there, exactly), hypot elsewhere; columns nf..ld zero"""
    from unified_audio_b200 import ops
    nf = n_fft // 2 + 1
    ldX = 2 * ((nf - 1) // P + 1)
    ld = (nf + 63) // 64 * 64
    X = torch.randn(M * P, ldX, generator=_gen(n_fft))
    k = torch.arange(nf)
    Xr = X.reshape(M, P, ldX)
    re, im = Xr[:, k % P, 2 * (k // P)].double(), Xr[:, k % P, 2 * (k // P) + 1].double()        # [M, nf]
    assert bool((im[:, 0] != 0).all()) and bool((im[:, -1] != 0).all())
    want = torch.hypot(re, im)
    want[:, 0], want[:, -1] = re[:, 0].abs(), re[:, -1].abs()
    out = _sentinel_planes((M, ld))
    ops.spec_magnitude(X.to(DEV), ldX, M, nf, P, out, ld)
    torch.cuda.synchronize()
    hi, lo = out.hi.cpu(), out.lo.cpu()
    got = hi.double() + lo.double()
    ends = [0, nf - 1]
    for e in ends:                                                   # |re| is exact: bit-identical planes
        h, l_ = _split(want[:, e].float())
        assert torch.equal(hi[:, e], h) and torch.equal(lo[:, e], l_), f"spec_magnitude: bin {e} is not |re|"
    bound = 2.0 ** -20 * want + 2.0 ** -25                           # hypotf (3 ulp) + the planes' representation (2^-22)
    ratio = float(((got[:, :nf] - want).abs() / bound).max())
    print(f"[spec_magnitude n_fft {n_fft} P {P}] worst error / bound {ratio:.3f}")
    assert ratio <= 1.0
    assert float(hi[:, nf:].abs().max()) == 0.0 and float(lo[:, nf:].abs().max()) == 0.0, "columns nf..ld not zeroed"


# ----------------------------------------------------------------------------------------------------------------- add_planes
@pytest.mark.parametrize("B,T,w,ld,d", [(2, 37, 64, 64, 2), (3, 20, 40, 64, 3), (1, 5, 16, 48, 5)])
def test_add_planes_res2net_pattern(lib, B, T, w, ld, d):
    """Res2Conv1dReluBn's sums as bicodec.py issues them: chunk i of y (row pitch C = 8 w) plus chunk i - 1, chunk 0 alone, into
    a [B, T + 2 d, ld] buffer at row offset d.  hi / lo are the split of torch's fp32 sum; pad rows untouched; columns w..ld
    zeroed."""
    from unified_audio_b200 import ops
    C = 8 * w
    y = torch.randn(B * T, C, generator=_gen(w * 100 + T))
    yd = y.to(DEV)
    for i in range(8):
        sp = _sentinel_planes((B, T + 2 * d, ld))
        ops.add_planes(yd.view(-1)[w * i:], C, yd.view(-1)[w * (i - 1):] if i else None, C, B, T, w, sp, ld, T + 2 * d, d)
        torch.cuda.synchronize()
        v = y[:, w * i:w * (i + 1)] + (y[:, w * (i - 1):w * i] if i else 0.0)
        h, l_ = _split(v)
        hi, lo = sp.hi.cpu(), sp.lo.cpu()
        assert torch.equal(hi[:, d:d + T, :w].reshape(B * T, w), h) and torch.equal(lo[:, d:d + T, :w].reshape(B * T, w), l_), \
            f"add_planes chunk {i}: planes differ from the split of the fp32 sum"
        for p in (hi, lo):
            assert bool((p[:, d:d + T, w:] == 0).all()), f"add_planes chunk {i}: columns {w}..{ld} not zeroed"
            assert bool((p[:, :d] == HALF_SENTINEL).all()) and bool((p[:, d + T:] == HALF_SENTINEL).all()), \
                f"add_planes chunk {i}: pad rows written"


# -------------------------------------------------------------------------------------------------------------------- se_gate
def _se_gate_bound(z, w1, b1, w2, b2):
    """fp64 s and a per-element bound on |s_kernel - s|: the fp32 mean (one rounding of an fp64 sum), the two fp32 dot products
    (ceil(n / 32) fma steps per lane + a 5-level warp tree + the bias: gamma_k over the sum of |terms|), the sigmoid's few ulp"""
    B, T, C = z.shape
    R = w1.shape[0]
    m = z.double().mean(1)                                                       # [B, C]
    a1 = m @ w1.double().t() + b1.double()
    h = a1.clamp_min(0)
    a2 = h @ w2.double().t() + b2.double()
    s = torch.sigmoid(a2)
    g = lambda n: (math.ceil(n / 32) + 6) * U32 / (1 - (math.ceil(n / 32) + 6) * U32)
    s1 = m.abs() @ w1.double().abs().t()
    e1 = g(C) * (s1 + b1.double().abs()) + U32 * s1 * (1 + g(C))                  # error of a1 (and so of h: relu is 1-Lipschitz)
    s2 = h @ w2.double().abs().t()
    e2 = e1 @ w2.double().abs().t() * (1 + g(R)) + g(R) * (s2 + b2.double().abs())
    return s, 0.25 * e2 + 8 * U32 * s + 1e-30                                    # sigmoid' <= 1/4; expf + 1/x few ulp


@pytest.mark.parametrize("B,T,C,R", [
    (2, 200, 512, 128),     # the shipped SE_Connect
    (1, 50, 100, 25),       # fewer channels than threads
    (2, 77, 1000, 128),     # more channels than the 512 threads
    (1, 40, 512, 1),        # bottleneck of one
    (2, 64, 256, 37),       # bottleneck not a multiple of the 32 lanes
    (2, 1, 512, 128),       # T = 1
    (3, 150, 512, 128),     # three clips, different data
])
def test_se_gate_fp64(lib, B, T, C, R):
    from unified_audio_b200 import ops
    g = _gen(C * 7 + R + T)
    z = torch.randn(B, T, C, generator=g) * 2 + torch.randn(B, 1, C, generator=g)
    w1 = torch.randn(R, C, generator=g) / math.sqrt(C)
    b1 = torch.randn(R, generator=g) * 0.1
    w2 = torch.randn(C, R, generator=g) / math.sqrt(R)
    b2 = torch.randn(C, generator=g) * 0.1
    want, bound = _se_gate_bound(z, w1, b1, w2, b2)
    s = torch.full((B + 1, C), F32_SENTINEL, device=DEV)
    ops.se_gate(z.to(DEV), B, T, C, w1.to(DEV), b1.to(DEV), w2.to(DEV), b2.to(DEV), s)
    torch.cuda.synchronize()
    got = s[:B].double().cpu()
    ratio = float(((got - want).abs() / bound).max())
    print(f"[se_gate B{B} T{T} C{C} R{R}] worst error / bound {ratio:.3f}")
    assert ratio <= 1.0
    assert bool((s[B] == F32_SENTINEL).all()), "se_gate wrote past its clips"


def test_se_gate_mean_is_exact_over_a_large_offset(lib):
    """Channels at 1e3 +- 1e-2 over T = 3000: an fp32 running sum drifts by many ulp of the mean there.  With w1 = I, b1 = 0,
    w2 = I and b2 = -fp32(mean) every dot product is exact, so s = sigmoid(mean_kernel - fp32(mean)) shows the mean's error to
    1/4 ulp: it must be the fp64 mean rounded once (one ulp allowed for a mean within 1e-9 of a rounding tie)."""
    from unified_audio_b200 import ops
    B, T, C = 2, 3000, 256
    g = _gen(1000)
    z = 1e3 + (torch.rand(B, T, C, generator=g) - 0.5) * 2e-2 + torch.arange(C) * 1e-1
    m32 = z.double().mean(1).float()                                             # the fp64 mean rounded once
    s = torch.empty(B, C, device=DEV)
    eye = torch.eye(C, device=DEV)
    for b in range(B):     # b2 depends on the clip: one call per clip
        ops.se_gate(z[b:b + 1].contiguous().to(DEV), 1, T, C, eye, torch.zeros(C, device=DEV), eye, (-m32[b]).to(DEV), s[b:b + 1])
    torch.cuda.synchronize()
    a2 = torch.logit(s.double().cpu())          # mean_kernel - fp32(mean), exactly an fp32 difference of neighbours or zero
    ulp = (torch.nextafter(m32, torch.tensor(float("inf"))) - m32).double()
    worst = float((a2.abs() / ulp).max())
    print(f"[se_gate 1e3 offset, T {T}] worst mean error {worst:.2f} ulp; means exact on {int((a2 == 0).sum())}/{B * C}")
    assert worst <= 1.01


def test_se_gate_refuses_shared_memory_overflow(lib):
    from unified_audio_b200 import ops
    C, R = 12000, 289                                # (C + R) * 4 bytes > 48 KB
    z = torch.zeros(1, 1, C, device=DEV)
    with pytest.raises(RuntimeError, match="se_gate"):
        ops.se_gate(z, 1, 1, C, torch.zeros(R, C, device=DEV), torch.zeros(R, device=DEV), torch.zeros(C, R, device=DEV),
                    torch.zeros(C, device=DEV), torch.zeros(1, C, device=DEV))


# ------------------------------------------------------------------------------------------------------------------- se_apply
@pytest.mark.parametrize("B,T,C", [(3, 37, 512), (2, 19, 300)])
def test_se_apply_bit_identical(lib, B, T, C):
    """out = x + z * s[b] rounded as torch rounds it on the GPU (product, then sum); the planes at col_off of a 3C-wide buffer are
    its hi / lo split, the other columns untouched; planes alone (out None) and out alone give the same values"""
    from unified_audio_b200 import ops
    g = _gen(C + T)
    z, x = (torch.randn(B * T, C, generator=g).to(DEV) for _ in range(2))
    s = torch.rand(B, C, generator=g).to(DEV)
    want = x + z * s.repeat_interleave(T, 0)
    h, l_ = _split(want)
    for col_off, with_out, with_planes in ((C, True, True), (2 * C, False, True), (0, True, False)):
        out = torch.full((B * T + 1, C), F32_SENTINEL, device=DEV)
        cat = _sentinel_planes((B * T, 3 * C))
        ops.se_apply(z, s, x, B, T, C, out=out[:B * T] if with_out else None, planes=cat if with_planes else None, ld=3 * C,
                     col_off=col_off)
        torch.cuda.synchronize()
        if with_out:
            assert torch.equal(out[:B * T], want), f"se_apply out: {int((out[:B * T] != want).sum())} values differ from x + z * s"
        assert bool((out[B * T:] == F32_SENTINEL).all()) and (with_out or bool((out == F32_SENTINEL).all()))
        if with_planes:
            assert torch.equal(cat.hi[:, col_off:col_off + C], h) and torch.equal(cat.lo[:, col_off:col_off + C], l_), \
                f"se_apply planes at col_off {col_off} differ from the split of x + z * s"
        keep = torch.ones(3 * C, dtype=torch.bool, device=DEV)
        if with_planes:
            keep[col_off:col_off + C] = False
        assert bool((cat.hi[:, keep] == HALF_SENTINEL).all()) and bool((cat.lo[:, keep] == HALF_SENTINEL).all()), \
            "se_apply wrote planes outside its columns"


# --------------------------------------------------------------------------------------------------------------- fsq_tokenize
def _half_l(L):
    return (L - 1) * (1 + 1e-3) / 2


def _offset(L):
    return 0.5 if L % 2 == 0 else 0.0


def _planted_rows(codes, levels, dim, r):
    """rows x whose normalisation (gamma = 1) times w_in = (r / sqrt(dim)) I gives z_j at the centre of code cell q_j:
    bound(z_j) = q_j exactly, so every decision is 0.5 from a rounding boundary.  x = (z, 0, ..., s) with |x| = r."""
    z = np.empty(codes.shape, np.float64)
    for j, L in enumerate(levels):
        hl, off = _half_l(L), _offset(L)
        z[:, j] = np.arctanh((codes[:, j] + off) / hl) - np.arctanh(off / hl)
    n2 = (z * z).sum(1)
    assert n2.max() < r * r / 2
    x = np.zeros((codes.shape[0], dim), np.float64)
    x[:, :len(levels)] = z
    x[:, -1] = np.sqrt(r * r - n2)
    return x


def _fsq_run(x, levels, gamma, w_in, b_in, with_taps=False):
    from unified_audio_b200 import ops
    rows, dim = x.shape
    idx = torch.full((rows + 1,), -7, dtype=torch.int32, device=DEV)
    zt = torch.full((rows, len(levels)), F32_SENTINEL, device=DEV) if with_taps else None
    xn = torch.full((rows, dim), F32_SENTINEL, device=DEV) if with_taps else None
    ops.fsq_tokenize(x.float().to(DEV), rows, dim, gamma.float().to(DEV), w_in.float().to(DEV), b_in.float().to(DEV), levels, 1,
                     idx[:rows], zt, xn)
    torch.cuda.synchronize()
    assert int(idx[rows]) == -7, "fsq_tokenize wrote past its rows"
    return idx[:rows].cpu().long(), zt, xn


def _index(q, levels):
    """the exact integer index sum_j (q_j + L_j // 2) * prod_{i<j} L_i (oracle/bicodec_global.fsq_tokenize, in int64)"""
    basis = np.cumprod([1] + list(levels[:-1])).astype(np.int64)
    return ((q + np.array(levels, np.int64) // 2) * basis).sum(-1)


FSQ_ENUMERATED = [[4] * 6, [8, 6, 5], [8, 5, 5, 5], [7, 5, 5, 5, 5], [8, 8, 8, 6, 5], [6, 6, 6], [7, 7, 7], [5, 5, 5], [2] * 8]


@pytest.mark.parametrize("levels", FSQ_ENUMERATED, ids=lambda lv: "x".join(map(str, lv)))
def test_fsq_index_exact_on_every_code(lib, levels):
    """Every code of the level set, planted at the centre of its cell: the index must be the exact integer (levels 6 and 7 need
    hw = 3, where fp32 steps contracted into FMAs truncate (fl(-2/3) * 3 + 3) * basis to one below)"""
    n, dim, r = len(levels), 45, 32.0
    digits = np.array(list(itertools.product(*[range(L) for L in reversed(levels)])), np.int64)[:, ::-1]   # index order
    q = digits - np.array(levels, np.int64) // 2
    want = _index(q, levels)
    assert np.array_equal(want, np.arange(len(want)))
    x = torch.from_numpy(_planted_rows(q, levels, dim, r))
    w_in = torch.zeros(n, dim, dtype=torch.float64)
    w_in[:, :n] = torch.eye(n) * (r / math.sqrt(dim))
    got, _, _ = _fsq_run(x, levels, torch.ones(dim), w_in, torch.zeros(n))
    bad = np.nonzero(got.numpy() != want)[0]
    print(f"[fsq {levels}] {len(want)} codes, {len(bad)} wrong")
    assert len(bad) == 0, (f"fsq {levels}: {len(bad)} of {len(want)} indices wrong, e.g. " +
                           ", ".join(f"code {tuple(int(v) for v in q[i])} -> {int(got[i])} (want {int(want[i])})" for i in bad[:6]))


def test_fsq_largest_codebook_sampled(lib):
    """[8] * 8 is exactly 2^24 entries, the largest accepted: 4096 random codes plus both corners, exact"""
    levels, dim, r = [8] * 8, 45, 32.0
    rng = np.random.default_rng(24)
    q = rng.integers(-4, 4, size=(4096, 8))
    q[0], q[1] = -4, 3
    want = _index(q, levels)
    assert want[0] == 0 and want[1] == 2 ** 24 - 1
    x = torch.from_numpy(_planted_rows(q, levels, dim, r))
    w_in = torch.zeros(8, dim, dtype=torch.float64)
    w_in[:, :8] = torch.eye(8) * (r / math.sqrt(dim))
    got, _, _ = _fsq_run(x, levels, torch.ones(dim), w_in, torch.zeros(8))
    assert np.array_equal(got.numpy(), want), f"fsq [8]*8: {int((got.numpy() != want).sum())} of 4096 indices wrong"


@pytest.mark.parametrize("levels", [[4] * 6, [8, 6, 5], [7, 5, 5, 5, 5]], ids=lambda lv: "x".join(map(str, lv)))
def test_fsq_random_rows_fp64(lib, levels):
    """Random rows (rows not a multiple of the 8 warps of a block, dim not a multiple of 32): RMSNorm output and project_in
    against fp64 within an fp32 dot-product bound; tokens exact wherever every decision is at least tau from a boundary"""
    from oracle import bicodec_global as og
    rows, dim, n = 203, 77, len(levels)
    g = _gen(rows + n)
    x = torch.randn(rows, dim, generator=g) * 3
    gamma = 1 + 0.2 * torch.randn(dim, generator=g)
    w_in = torch.randn(n, dim, generator=g) / math.sqrt(dim)
    b_in = 0.1 * torch.randn(n, generator=g)
    got, zt, xn = _fsq_run(x, levels, gamma, w_in, b_in, with_taps=True)
    x64 = x.double()
    xn64 = x64 / x64.norm(dim=1, keepdim=True) * math.sqrt(dim) * gamma.double()
    z64 = xn64 @ w_in.double().t() + b_in.double()
    e_xn = float(((xn.double().cpu() - xn64).abs() / (xn64.abs() + 1e-30)).max())
    k = math.ceil(dim / 32) + 6
    zb = (k + 18) * U32 * (xn64.abs() @ w_in.double().abs().t() + b_in.double().abs())
    r_z = float(((zt.double().cpu() - z64).abs() / zb).max())
    print(f"[fsq random {levels}] xn max rel {e_xn:.2e} ({e_xn / U32:.1f} u); z error / bound {r_z:.3f}")
    assert e_xn <= 8 * U32 + (math.ceil(dim / 32) + 5) * U32 and r_z <= 1.0
    tau = max(10 * float((zt.double().cpu() - z64).abs().max()), 1e-4)
    safe = (og.fsq_margins(z64, levels) >= tau).all(-1)
    q = torch.round(og.fsq_bound(z64, levels)).long().numpy()
    want = _index(q, levels)
    assert int(safe.sum()) > rows // 2
    assert np.array_equal(got.numpy()[safe.numpy()], want[safe.numpy()]), "fsq random rows: token differs at a safe margin"


def test_fsq_refusals(lib):
    from unified_audio_b200 import ops
    x, g, w, b = (torch.zeros(s, device=DEV) for s in ((4, 32), (32,), (9, 32), (9,)))
    idx = torch.zeros(4, dtype=torch.int32, device=DEV)
    for levels, nq, what in (([4] * 6, 2, "quantizers"), ([2] * 9, 1, "at most 8"), ([4, 1, 4], 1, ">= 2"),
                             ([9] + [8] * 7, 1, "2\\^24")):
        with pytest.raises(RuntimeError, match=what):
            ops.fsq_tokenize(x, 4, 32, g, w, b, levels, nq, idx)
