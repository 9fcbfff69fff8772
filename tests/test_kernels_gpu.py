"""Every variant of the elementwise, normalisation, SSL, attention, loss and RVQ launchers against plain fp64 torch on the same
device, at the shapes and layouts where each launcher switches kernels (csrc/elementwise.cu, ssl.cu, attention.cu, llm.cu,
rvq.cu).  Outputs start as sentinels; each test also checks that nothing outside the intended window was written."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF_SENTINEL = -1234.0          # exact in fp16, produced by none of these kernels
F32_TOL = 1e-6                   # fp32-output kernels, relative to the largest reference value
PLANES_REP = 2.0 ** -21          # hi + lo planes represent an fp32 value to ~2^-22


def _rnd(shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + offset).to(DEV)


def planes_ref(hi, lo=None):
    return hi.double() + (lo.double() if lo is not None else 0.0)


def relerr(got, ref):
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _planes_buf(B, rows, ld, split=True):
    """(Planes, backing [2, B, rows, ld] buffer): both planes pre-filled with the sentinel; the lo half stays the sentinel
    when split is False (the kernel is handed hi only)."""
    from unified_audio_b200 import ops
    buf = torch.full((2, B, rows, ld), HALF_SENTINEL, dtype=torch.float16, device=DEV)
    return ops.Planes(buf[0], buf[1] if split else None), buf


def _window(B, rows, ld, off, T, C):
    m = torch.zeros(B, rows, ld, dtype=torch.bool, device=DEV)
    m[:, off:off + T, :C] = True
    return m


def _check_planes(name, buf, off, T, C, ref, split=True, tol=F32_TOL, zero_cols_to=None):
    """planes interior [off, off+T) x [0, C) against ref, the rest of the rows' columns up to zero_cols_to zero, all else
    the sentinel."""
    hi, lo = buf[0], buf[1]
    got = planes_ref(hi[:, off:off + T, :C], lo[:, off:off + T, :C] if split else None)
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite output"
    e = relerr(got, ref)
    print(f"{name}: error {e:.2e} of the largest value")
    rep = PLANES_REP if split else 2.0 ** -11
    bound = tol * float(ref.abs().max()) + rep * ref.abs() + 2.0 ** -25
    assert bool(((got - ref).abs() <= bound).all()), f"{name}: error {e:.2e} beyond the bound"
    B, rows, ld = hi.shape
    written = _window(B, rows, ld, off, T, C)
    if zero_cols_to:
        written[:, off:off + T, C:zero_cols_to] = True
        assert bool((hi[:, off:off + T, C:zero_cols_to] == 0).all()), f"{name}: pad columns not zeroed"
    assert bool((hi[~written] == HALF_SENTINEL).all()), f"{name}: hi written outside its window"
    if split:
        assert bool((lo[~written] == HALF_SENTINEL).all()), f"{name}: lo written outside its window"
    else:
        assert bool((lo == HALF_SENTINEL).all()), f"{name}: lo written although only hi was requested"


def _dwconv_ref(x, w, b):
    """depthwise conv over time, zero 'same' padding: x [B, T, C], w [C, k]"""
    C, k = w.shape
    return F.conv1d(x.double().transpose(1, 2), w.double()[:, None, :], b.double() if b is not None else None, padding=k // 2,
                    groups=C).transpose(1, 2)


def _ln(h, eps):
    return F.layer_norm(h, (h.shape[-1],), eps=eps)


# ---------------------------------------------------------------------------------------------- dwconv7 + (Ada)LayerNorm
# dwconv7_ln_launch: v2 <8,384,2> for C % 128 == 0 and C / 4 <= 384; v2 <8,512,1> for C / 4 in (384, 512]; the warp kernel
# otherwise (C % 128 != 0, or a per-clip AdaLN stride that is not a multiple of 4)
@pytest.mark.parametrize("C,T,B,ada", [
    (256, 5, 2, None),        # v2 <8,384,2>: T < 7 (every tap of the window falls off an edge) and T not a multiple of 8
    (256, 13, 3, 4),          # v2 <8,384,2>, per-clip AdaLN rows
    (1536, 20, 2, 4),         # v2 <8,384,2> at C / 4 = 384
    (2048, 11, 2, None),      # v2 <8,512,1>
    (1664, 9, 2, 4),          # v2 <8,512,1>, AdaLN
    (96, 20, 3, None),        # warp kernel: C % 128 != 0
    (96, 6, 2, 4),            # warp kernel, AdaLN
    (256, 10, 3, 1),          # warp kernel: AdaLN stride not a multiple of 4
])
def test_dwconv7_ln(lib, C, T, B, ada):
    from unified_audio_b200 import ops
    x = _rnd((B, T, C), 1, 2.0, 0.3)
    dw_w, dw_b = _rnd((C, 7), 2, 0.3), _rnd((C,), 3, 0.1)
    h = _ln(_dwconv_ref(x, dw_w, dw_b), 1e-6)
    out, buf = _planes_buf(1, B * T, C)
    if ada is None:
        ln_w, ln_b = _rnd((C,), 4, 0.1, 1.0), _rnd((C,), 5, 0.1)
        ops.dwconv7_ln(x, dw_w, dw_b, ln_w, ln_b, B, T, C, ops.Planes(out.hi.view(B, T, C), out.lo.view(B, T, C)))
        ref = h * ln_w.double() + ln_b.double()
    else:
        # per-clip rows of a conditioning matrix [B, 2C + pad] (scale at +0, shift at +C), `stride` floats apart, as the
        # backbone's AdaLayerNorm rows (bicodec.py cond_rows); ada = 4 keeps the rows 16-byte aligned for v2
        stride = 2 * C + ada
        cond = _rnd((B * stride + C,), 6, 0.5)
        scale, shift = cond[:B * stride].view(B, stride)[:, :C], cond[C:C + B * stride].view(B, stride)[:, :C]
        ops.dwconv7_adaln(x, dw_w, dw_b, cond, cond[C:], stride, B, T, C, ops.Planes(out.hi.view(B, T, C), out.lo.view(B, T, C)))
        ref = h * scale.double()[:, None] + shift.double()[:, None]
    torch.cuda.synchronize()
    _check_planes(f"dwconv7 C={C} T={T} ada={ada}", buf, 0, B * T, C, ref.reshape(1, B * T, C), tol=2e-6)


# ---------------------------------------------------------------------------------------------- Snake -> planes
@pytest.mark.parametrize("C,ld,x_off,strided", [
    (256, 320, 64, True),     # snake_planes_v8 on a strided batch view (bicodec.py: rows pad_t.. of the up-sampled buffer)
    (256, 256, 0, False),     # v8, contiguous
    (100, 128, 0, False),     # scalar: C % 8 != 0
    (256, 256, 1, True),      # scalar: x not 16-byte aligned
    (96, 100, 0, False),      # scalar: ld % 8 != 0
])
def test_snake_planes(lib, C, ld, x_off, strided):
    from unified_audio_b200 import ops
    B, T, rows, off = 3, 37, 43, 3
    bstride = (T + 5) * C + 8 if strided else T * C
    flat = _rnd((x_off + B * bstride,), 7, 2.0)
    x = flat[x_off:]
    g = torch.Generator(device="cpu").manual_seed(8)
    alpha = torch.logspace(-3, math.log10(5.0), C, dtype=torch.float64).float()[torch.randperm(C, generator=g)].to(DEV)
    out, buf = _planes_buf(B, rows, ld)
    ops.snake_planes(x, bstride, alpha, B, T, C, out, ld, rows, off)
    torch.cuda.synchronize()
    xv = torch.stack([x[b * bstride:b * bstride + T * C].view(T, C) for b in range(B)])
    t = (alpha * xv).double()                       # the kernel's fp32 argument
    ref = xv.double() + torch.sin(t) ** 2 / (alpha.double() + 1e-9)
    _check_planes(f"snake C={C} ld={ld} x_off={x_off}", buf, off, T, C, ref, zero_cols_to=ld)


# ---------------------------------------------------------------------------------------------- GroupNorm
@pytest.mark.parametrize("C,G,ld,swish", [
    (256, 32, 256, True),     # float4 stats, float4 apply
    (256, 32, 258, False),    # float4 stats, scalar apply (ld % 4 != 0)
    (96, 32, 96, True),       # scalar stats and apply: C / G = 3
    (100, 25, 104, True),     # float4 (C / G = 4)
    (90, 30, 96, False),      # scalar stats and apply: C % 4 != 0
])
def test_groupnorm(lib, C, G, ld, swish):
    from unified_audio_b200 import ops
    B, T, rows, off = 2, 29, 33, 2
    x = _rnd((B, T, C), 9, 1.5, 0.7)
    w, b = _rnd((C,), 10, 0.2, 1.0), _rnd((C,), 11, 0.2)
    stats = torch.full((B, G, 2), float("nan"), device=DEV)
    ops.groupnorm_stats(x, B, T, C, stats, groups=G)
    o32 = torch.full((B, T, C), float("nan"), device=DEV)
    out, buf = _planes_buf(B, rows, ld)
    ops.groupnorm_apply(x, stats, w, b, B, T, C, swish, out_f32=o32, out=out, ld=ld, rows_per_batch=rows, row_off=off, groups=G)
    torch.cuda.synchronize()
    ref = F.group_norm(x.double().transpose(1, 2), G, w.double(), b.double(), 1e-6).transpose(1, 2)
    if swish:
        ref = ref * torch.sigmoid(ref)
    e = relerr(o32, ref)
    print(f"groupnorm C={C} G={G} ld={ld}: fp32 error {e:.2e}")
    assert e < F32_TOL
    _check_planes(f"groupnorm C={C} G={G} ld={ld}", buf, off, T, C, ref)


# ---------------------------------------------------------------------------------------------- LayerNorm + GELU, AdaLayerNorm
@pytest.mark.parametrize("act", [0, 1])
def test_layernorm_act(lib, act):
    from unified_audio_b200 import ops
    B, T, C, rows, off, ld = 2, 45, 512, 50, 3, 576
    x = _rnd((B, T, C), 12, 3.0, 1.0)
    w, b = _rnd((C,), 13, 0.2, 1.0), _rnd((C,), 14, 0.5)
    o32 = torch.full((B, T, C), float("nan"), device=DEV)
    out, buf = _planes_buf(B, rows, ld)
    ops.layernorm_act(x, w, b, B, T, C, act, eps=1e-5, out_f32=o32, out=out, ld=ld, rows_per_batch=rows, row_off=off)
    torch.cuda.synchronize()
    ref = _ln(x.double(), 1e-5) * w.double() + b.double()
    if act:
        ref = F.gelu(ref)                        # exact erf GELU
    e = relerr(o32, ref)
    print(f"layernorm_act act={act}: fp32 error {e:.2e}")
    assert e < 2e-6
    _check_planes(f"layernorm_act act={act}", buf, off, T, C, ref, tol=2e-6)


def test_adalayernorm(lib):
    from unified_audio_b200 import ops
    B, T, C, rows, off = 3, 21, 384, 24, 1
    stride = 2 * C * 3                           # 3 norms' rows per clip, as bicodec.py's cond matrix
    x = _rnd((B, T, C), 15, 2.0, -0.5)
    cond = _rnd((B, stride), 16, 0.5)
    j = 1                                        # the second norm's scale / shift
    scale, shift = cond[:, 2 * C * j:2 * C * j + C], cond[:, 2 * C * j + C:2 * C * (j + 1)]
    o32 = torch.full((B, T, C), float("nan"), device=DEV)
    out, buf = _planes_buf(B, rows, C)
    base = cond.view(-1)
    ops.adalayernorm(x, base[2 * C * j:], base[2 * C * j + C:], stride, B, T, C, eps=1e-6, out_f32=o32, out=out, ld=C,
                     rows_per_batch=rows, row_off=off)
    torch.cuda.synchronize()
    ref = _ln(x.double(), 1e-6) * scale.double()[:, None] + shift.double()[:, None]
    e = relerr(o32, ref)
    print(f"adalayernorm: fp32 error {e:.2e}")
    assert e < 2e-6
    _check_planes("adalayernorm", buf, off, T, C, ref, tol=2e-6)


# ---------------------------------------------------------------------------------------------- plane conversions
def _split_exact(x):
    hi = x.float().clamp(-65504.0, 65504.0).half()
    return hi, (x.float() - hi.float()).half()


def test_split_f16(lib):
    from unified_audio_b200 import ops
    x = _rnd((3000,), 17, 10.0)
    x[:6] = torch.tensor([1e5, -1e5, 65519.0, 3e-6, -0.0, 0.0], device=DEV)
    buf = torch.full((2, 3001), HALF_SENTINEL, dtype=torch.float16, device=DEV)
    ops.split_f16(x, ops.Planes(buf[0, :3000], buf[1, :3000]))
    torch.cuda.synchronize()
    hi, lo = _split_exact(x)
    assert torch.equal(buf[0, :3000].view(torch.int16), hi.view(torch.int16))
    assert torch.equal(buf[1, :3000].view(torch.int16), lo.view(torch.int16))
    assert float(buf[0, 3000]) == HALF_SENTINEL and float(buf[1, 3000]) == HALF_SENTINEL


@pytest.mark.parametrize("repeat,act", [(1, 0), (2, 3), (3, 0)])
def test_rows_to_planes(lib, repeat, act):
    from unified_audio_b200 import ops
    B, T, C, ld, off = 2, 17, 100, 128, 2
    rows = off + T * repeat + 3
    x = _rnd((B * T, C), 18, 2.0)
    out, buf = _planes_buf(B, rows, ld)
    ops.rows_to_planes(x, B, T, C, out, ld, rows, off, repeat=repeat, act=act)
    torch.cuda.synchronize()
    ref = x.view(B, T, C).double().repeat_interleave(repeat, dim=1)
    if act == 3:
        ref = F.elu(ref)
    _check_planes(f"rows_to_planes repeat={repeat} act={act}", buf, off, T * repeat, C, ref, zero_cols_to=ld)


def test_bct_to_planes(lib):
    from unified_audio_b200 import ops
    B, C, T, ld, rows, off = 2, 70, 45, 128, 48, 1
    x = _rnd((B, C, T), 19, 3.0)
    out, buf = _planes_buf(B, rows, ld)
    ops.bct_to_planes(x, out, ld, rows, off)
    torch.cuda.synchronize()
    hi, lo = _split_exact(x.transpose(1, 2))
    assert torch.equal(buf[0, :, off:off + T, :C], hi) and torch.equal(buf[1, :, off:off + T, :C], lo)
    _check_planes("bct_to_planes", buf, off, T, C, x.transpose(1, 2).double(), tol=0.0, zero_cols_to=ld)


def test_addvec_planes(lib):
    from unified_audio_b200 import ops
    B, T, C, ld, rows, off = 3, 19, 100, 128, 25, 3
    x, vec = _rnd((B, T, C), 20), _rnd((B, C), 21)
    out, buf = _planes_buf(B, rows, ld)
    ops.addvec_planes(x, vec, B, T, C, out, ld, rows, off)
    torch.cuda.synchronize()
    hi, lo = _split_exact(x + vec[:, None])          # one fp32 add, then the split: exact
    assert torch.equal(buf[0, :, off:off + T, :C], hi) and torch.equal(buf[1, :, off:off + T, :C], lo)
    _check_planes("addvec_planes", buf, off, T, C, (x.double() + vec.double()[:, None]), zero_cols_to=ld)


@pytest.mark.parametrize("pad_l,pad_r", [(3, 3), (1, 4), (0, 2)])
def test_reflect_pad_rows(lib, pad_l, pad_r):
    from unified_audio_b200 import ops
    B, T, ld, off = 2, 9, 136, 5
    rows = off + T + 6
    buf = torch.full((2, B, rows, ld), HALF_SENTINEL, dtype=torch.float16, device=DEV)
    interior = _rnd((2, B, T, ld), 22).half()
    buf[:, :, off:off + T] = interior
    ops.reflect_pad_rows(ops.Planes(buf[0], buf[1]), B, rows, ld, T, off, pad_l, pad_r)
    torch.cuda.synchronize()
    # F.pad(mode="reflect") over time, both planes
    ref = F.pad(interior.float().permute(0, 1, 3, 2).reshape(2 * B, ld, T), (pad_l, pad_r), mode="reflect")
    ref = ref.reshape(2, B, ld, T + pad_l + pad_r).permute(0, 1, 3, 2).half()
    assert torch.equal(buf[:, :, off - pad_l:off + T + pad_r], ref)
    assert bool((buf[:, :, :off - pad_l] == HALF_SENTINEL).all()) and bool((buf[:, :, off + T + pad_r:] == HALF_SENTINEL).all())


@pytest.mark.parametrize("k,bias", [(3, True), (7, False)])
def test_dwconv(lib, k, bias):
    from unified_audio_b200 import ops
    B, T, C = 2, 33, 300
    x, w = _rnd((B, T, C), 23), _rnd((C, k), 24, 0.4)
    b = _rnd((C,), 25) if bias else None
    out = torch.full((B, T, C), float("nan"), device=DEV)
    ops.dwconv(x, w, b, B, T, C, k, out)
    torch.cuda.synchronize()
    e = relerr(out, _dwconv_ref(x, w, b))
    print(f"dwconv k={k}: error {e:.2e}")
    assert e < F32_TOL


# ---------------------------------------------------------------------------------------------- SSL front end
@pytest.mark.parametrize("T_in,k,s", [(1000, 10, 5), (333, 3, 2)])
def test_ssl_conv0(lib, T_in, k, s):
    """conv layer 0 with T0 not a multiple of the 64-frame block: GroupNorm(C groups) + GELU -> planes, and + bias -> fp32"""
    from unified_audio_b200 import ops
    B, C = 2, 192
    T0 = (T_in - k) // s + 1
    assert T0 % 64
    x = _rnd((B, T_in), 26, 0.3)
    w, gw, gb, bias = _rnd((C, k), 27, 0.5), _rnd((C,), 28, 0.2, 1.0), _rnd((C,), 29, 0.2), _rnd((C,), 30)
    conv = F.conv1d(x.double()[:, None], w.double()[:, None], stride=s).transpose(1, 2)       # [B, T0, C]
    rows, off, ld = T0 + 4, 2, 256
    out, buf = _planes_buf(B, rows, ld)
    ys = torch.empty(B, T0, C, device=DEV)
    ws = torch.empty(ops.ssl_conv0_workspace_bytes(B, T0, C), dtype=torch.uint8, device=DEV)
    ops.ssl_conv0_gn_gelu(x, w, gw, gb, 1e-5, k, s, out, ld, rows, off, ys, ws)
    y = torch.full((B, T0, C), float("nan"), device=DEV)
    ops.ssl_conv0_bias(x, w, bias, k, s, y)
    torch.cuda.synchronize()
    e = relerr(y, conv + bias.double())
    print(f"ssl_conv0_bias: error {e:.2e}")
    assert e < F32_TOL
    ref = F.gelu(F.group_norm(conv.transpose(1, 2), C, gw.double(), gb.double(), 1e-5).transpose(1, 2))
    _check_planes(f"ssl_conv0_gn_gelu T0={T0}", buf, off, T0, C, ref, tol=2e-6)


@pytest.mark.parametrize("kind", ["random", "constant", "dc_offset"])
def test_wav_normalize(lib, kind):
    from unified_audio_b200 import ops
    B, T = 3, 16001
    if kind == "random":
        x = _rnd((B, T), 31, 0.2)
    elif kind == "constant":                      # variance 0: the result is 0 / sqrt(eps), not NaN
        x = torch.full((B, T), 0.37, device=DEV)
    else:                                         # large DC offset: E[x^2] - mean^2 would cancel
        x = _rnd((B, T), 32, 1e-3, 1000.0)
    out = torch.full((B, T), float("nan"), device=DEV)
    ops.wav_normalize(x, 1e-7, out)
    torch.cuda.synchronize()
    xd = x.double()
    ref = (xd - xd.mean(1, keepdim=True)) / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-7)
    assert bool(torch.isfinite(out).all())
    if kind == "constant":
        assert bool((out == 0).all())
    else:
        e = relerr(out, ref)
        print(f"wav_normalize {kind}: error {e:.2e}")
        assert e < F32_TOL


@pytest.mark.parametrize("accumulate", [0, 1])
def test_axpy(lib, accumulate):
    from unified_audio_b200 import ops
    n = 100003
    x, o0 = _rnd((n,), 33), _rnd((n,), 34)
    out = o0.clone()
    ops.axpy(x, 1.0 / 13, out, accumulate=bool(accumulate))
    torch.cuda.synchronize()
    # one fp32 rounding of the exact value (fma); 1/13 itself is rounded to fp32 first, as the kernel's argument
    ref = torch.tensor(1.0 / 13, dtype=torch.float32).double().item() * x.double() + (o0.double() if accumulate else 0.0)
    assert bool(((out.double() - ref).abs() <= 2.0 ** -24 * ref.abs() + 1e-45).all())


@pytest.mark.parametrize("power,channel_first", [(0.3, 1), (0.3, 0), (0.0, 1)])
def test_ssl_compress(lib, power, channel_first):
    from unified_audio_b200 import ops
    B, T, C = 2, 37, 70
    x = _rnd((B, T, C), 35)
    x[0, :3] = 0.0                                # exact zeros: the reference's sign(x) is -1 there -> -0.0
    x[1, 5, :4] = -0.0
    out = torch.full((B * T * C,), float("nan"), device=DEV)
    ops.ssl_compress(x, B, T, C, power, channel_first, out)
    torch.cuda.synchronize()
    xd = x.double()
    if power > 0:
        ref = ((xd > 0).double() * 2 - 1) * xd.abs() ** power
    else:
        ref = xd
    if channel_first:
        ref = ref.transpose(1, 2)
    got = out.view(ref.shape)
    assert bool(((got.double() - ref).abs() <= 1e-6 * ref.abs()).all())
    assert torch.equal(torch.signbit(got), torch.signbit(ref.float())), "sign of zero"


@pytest.mark.parametrize("left,T_out,wrap", [(160, 1320, False), (5, 3107, True), (0, 700, False), (3, 700, True),
                                             (-4, 500, True)])
def test_pad_wav(lib, left, T_out, wrap):
    from unified_audio_b200 import ops
    B, T_in = 2, 1000
    x = _rnd((B, T_in), 36)
    out = ops.pad_wav(x, left, T_out, wrap=wrap)
    torch.cuda.synchronize()
    j = torch.arange(T_out, device=DEV) - left
    inside = (j >= 0) & (j < T_in)
    src = j % T_in if wrap else j.clamp(0, T_in - 1)
    ref = torch.where(inside | wrap, x[:, src], torch.zeros((), device=DEV))
    assert torch.equal(out, ref)


# ---------------------------------------------------------------------------------------------- WavLM gate + relative-bias attention
def test_wavlm_gate(lib):
    from unified_audio_b200 import ops
    B, T, H, D = 2, 37, 12, 64
    x = _rnd((B, T, H * D), 37)
    w, bias, cst = _rnd((8, D), 38, 0.2), _rnd((8,), 39, 0.2), _rnd((H,), 40, 0.5, 1.0)
    gate = torch.full((B, H, T), float("nan"), device=DEV)
    ops.wavlm_gate(x, B, T, H, D, w, bias, cst, gate)
    torch.cuda.synchronize()
    p = x.double().view(B, T, H, D) @ w.double().t() + bias.double()                            # [B, T, H, 8]
    ga, gb = torch.sigmoid(p[..., :4].sum(-1)), torch.sigmoid(p[..., 4:].sum(-1))
    ref = (ga * (gb * cst.double() - 1) + 2).permute(0, 2, 1)
    e = relerr(gate, ref)
    print(f"wavlm_gate: error {e:.2e}")
    assert e < F32_TOL


@pytest.mark.parametrize("T", [1, 33, 129, 300])
def test_attention_relbias(lib, T):
    from unified_audio_b200 import ops
    B, H, D = 2, 3, 64
    qkv = _rnd((B, T, 3 * H * D), 41 + T)
    rel = _rnd((H, 2 * T - 1), 42, 2.0)
    gate = _rnd((B, H, T), 43, 0.3, 1.5)
    out, buf = _planes_buf(1, B * T, H * D)
    ops.attention_relbias(qkv, B, T, H, D, rel, gate, ops.Planes(out.hi.view(B, T, H * D), out.lo.view(B, T, H * D)))
    torch.cuda.synchronize()
    q, k, v = [t.reshape(B, T, H, D).transpose(1, 2).double() for t in qkv.chunk(3, -1)]
    i = torch.arange(T, device=DEV)
    bias = rel.double()[:, (i[None, :] - i[:, None]) + T - 1]                                   # [H, T(i), T(j)]
    att = torch.softmax(q @ k.transpose(2, 3) * D ** -0.5 + gate.double()[..., None] * bias[None], -1)
    ref = (att @ v).transpose(1, 2).reshape(1, B * T, H * D)
    _check_planes(f"attention_relbias T={T}", buf, 0, B * T, H * D, ref, tol=5e-6)


# ---------------------------------------------------------------------------------------------- teacher-forced loss
@pytest.mark.parametrize("ls", [0.0, 0.1])
def test_lm_loss(lib, ls):
    from unified_audio_b200 import ops
    M, V, ld = 6, 12291, 12300
    logits = _rnd((M, ld), 44, 3.0)
    logits[:, V:] = 1e4                            # columns past V must not be read
    targets = torch.tensor([5, 12290, 77, 300, 4000, 9000], device=DEV)
    # tied maxima: row 0's maximum at 5 and 6000 (target 5, the lower index: a hit), row 3's at 100 and 300 (target 300: a miss)
    logits[0, 5] = logits[0, 6000] = 40.0
    logits[3, 100] = logits[3, 300] = 40.0
    logits[2, 77] = 50.0                           # a plain hit
    logits[[1, 4, 5], targets[[1, 4, 5]]] = -20.0  # plain misses
    out = ops.lm_loss(logits, ld, M, V, targets, ls)
    torch.cuda.synchronize()
    lp = torch.log_softmax(logits[:, :V].double(), -1)
    q = torch.full((M, V), ls / (V - 1), dtype=torch.float64, device=DEV)
    q[torch.arange(M), targets] = 1 - ls
    kl = torch.where(q > 0, q * (torch.log(q.clamp_min(1e-300)) - lp), torch.zeros((), dtype=torch.float64, device=DEV))
    ref_loss = float(kl.sum() / M)
    e = abs(float(out[0]) - ref_loss) / abs(ref_loss)
    print(f"lm_loss ls={ls}: loss {float(out[0]):.6f} vs {ref_loss:.6f}, error {e:.2e}")
    assert e < 2e-6
    assert float(out[1]) == float(torch.tensor(2.0 / M, dtype=torch.float32))   # rows 0 and 2: the lowest index of a tie wins


# ---------------------------------------------------------------------------------------------- RVQ
def _rvq_ref(x, cb):
    """residual in fp32 (r = r - e), squared distances of the fp32 values in fp64, arg-min with the lowest index on ties"""
    r = x.cpu().float()
    cbc = cb.cpu().float()
    out = torch.zeros_like(r)
    idx = []
    for q in range(cbc.shape[0]):
        e64 = cbc[q].double()
        best = torch.cat([((r[i:i + 16].double()[:, None] - e64[None]) ** 2).sum(-1).argmin(-1)
                          for i in range(0, r.shape[0], 16)])
        e = cbc[q][best]
        r = r - e
        out = out + e
        idx.append(best)
    return torch.stack(idx, -1), out


def _rvq_books(kind, K, D, nq, g):
    cb = torch.stack([torch.randn(K, D, generator=g) * 0.5 * 0.7 ** q for q in range(nq)])
    M = 203
    x = torch.randn(M, D, generator=g) * 0.5
    if kind == "duplicates":                      # codewords j and j + K/2 equal: the lower index must win
        h = K // 2
        cb[0, h:2 * h] = cb[0, :h]
        pick = torch.randint(0, h, (M,), generator=g) + h
        x = cb[0, pick] + torch.randn(M, D, generator=g) * 1e-3
        cb[1, h:2 * h] = cb[1, :h]
    elif kind == "exact":                          # inputs equal to a codeword (then a zero residual)
        x = cb[0, torch.randint(0, K, (M,), generator=g)].clone()
        x[::3] = cb[0, 7]
    elif kind == "near_ties":                      # two codewords whose distances to the input differ by ~1e-7 relative
        pick = torch.randint(0, K // 2, (M,), generator=g)
        u = torch.randn(K // 2, D, generator=g)
        u = u / u.norm(dim=-1, keepdim=True)
        v = torch.randn(K // 2, D, generator=g)
        v = v / v.norm(dim=-1, keepdim=True)
        c = torch.randn(K // 2, D, generator=g) * 0.5
        cb[0, :K // 2] = c + 0.1 * u
        cb[0, K // 2:2 * (K // 2)] = c + 0.1 * (1 + 5e-8) * v
        x = c[pick].clone()
    elif kind == "offset":                         # a large common offset: |e|^2 - 2 r.e cancels
        cb[0] = cb[0] * 0.1 + 30.0
        x = x * 0.1 + 30.0
    return x, cb


@pytest.mark.parametrize("kind", ["duplicates", "exact", "near_ties", "offset"])
@pytest.mark.parametrize("K,D", [(100, 64), (1024, 256), (100, 256), (1024, 64)])
def test_rvq_adversarial(lib, kind, K, D):
    """rvq.cu's guarantee: the index is the exact arg-min of the fp32 residual path, lowest index on exact ties."""
    from unified_audio_b200 import ops
    from unified_audio_b200.rvq import ResidualVQ
    nq = 3
    g = torch.Generator().manual_seed(K + D)
    x, cb = _rvq_books(kind, K, D, nq, g)
    M = x.shape[0]
    vq = ResidualVQ(dim=D, codebook_size=K, num_quantizers=nq).to(DEV)
    vq.set_codebooks(cb.to(DEV))
    p = vq._prepare()
    idx = torch.full((M, nq), -7, dtype=torch.int64, device=DEV)
    quant = torch.full((M, D), float("nan"), device=DEV)
    ws = torch.empty(ops.rvq_workspace_bytes(M, D, K), dtype=torch.uint8, device=DEV)
    ops.rvq_encode(x.to(DEV), p["cb"], p["planes"], p["consts"], p["e2max"], M, D, K, nq, idx, quant, ws)
    torch.cuda.synchronize()
    ridx, rquant = _rvq_ref(x, cb)
    bad = (idx.cpu() != ridx).any(-1)
    assert not bool(bad.any()), f"{kind}: {int(bad.sum())} rows differ, first {idx.cpu()[bad][:3].tolist()} vs {ridx[bad][:3].tolist()}"
    assert torch.equal(quant.cpu(), rquant)
    if kind == "duplicates":
        assert bool((ridx[:, 0] < K // 2).all())   # the construction did exercise the tie rule


def test_rvq_decode(lib):
    """-1 entries (dropped layers) contribute nothing; the rows land at col_off of a wider output"""
    from unified_audio_b200 import ops
    M, D, K, nq, ld, col_off = 37, 64, 100, 4, 200, 72
    g = torch.Generator().manual_seed(3)
    cb = torch.randn(nq, K, D, generator=g)
    idx = torch.randint(0, K, (M, nq), generator=g)
    idx[::3, 1] = -1
    idx[5] = -1
    out = torch.full((M, ld), float("nan"), device=DEV)
    ops.rvq_decode(idx.to(DEV), cb.to(DEV), M, D, K, nq, out, ld, col_off)
    torch.cuda.synchronize()
    from oracle import rvq as orvq
    assert torch.equal(out[:, col_off:col_off + D].cpu(), orvq.rvq_decode(idx, cb))
    assert bool(out[:, :col_off].isnan().all()) and bool(out[:, col_off + D:].isnan().all())
    assert bool((out[5, col_off:col_off + D] == 0).all())
