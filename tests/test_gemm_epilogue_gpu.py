"""qb_gemm's epilogues on each of its three kernel instantiations (<3,128,3> split, <1,128,6> single pass n <= 128,
<1,256,4> single pass n > 128) against an fp64 reference of the same contraction over the fp16 planes the kernel reads.

Every output buffer starts as a sentinel (NaN for fp32, a fixed half for planes) and every case checks that nothing outside
the window the descriptor names was written: pad rows, columns n..ld, and the lo plane when only hi is requested.
Every case is also run through the SIMT evaluation of the same descriptor, and the two fast epilogue kinds (EPI_HI,
EPI_F32) are checked bit for bit against epilogue_pair, which a 4-byte aligned bias selects instead."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF_SENTINEL = -1234.0          # exact in fp16; no epilogue below produces it
GEMM_TOL = 2e-5                  # relative to the largest pre-activation, as tests/test_gemm_wide_gpu.py
SIN_ERR = 3e-7                   # |sine error| of snake_f for |alpha x| < 64, as stated above it in csrc/gemm.cu

NONE, GELU, SWIGLU, ELU, TANH, SNAKE = 0, 1, 2, 3, 4, 5
ACT_NAMES = {NONE: "none", GELU: "gelu", SWIGLU: "swiglu", ELU: "elu", TANH: "tanh", SNAKE: "snake"}

# kernel instantiation -> (split operands, n values it is chosen for)
INSTS = {"split": (True, (1, 2, 127, 128, 129, 255, 256, 257, 520)),
         "n128": (False, (1, 2, 127, 128)),
         "n256": (False, (129, 255, 256, 257, 520))}

# (act, act2, outputs, bias, gamma, residual): f = fp32, h = fp16 hi plane, l = lo plane; residual None / "sep" / "inplace".
# Covers every pair of act x act2, act x outputs, act2 x outputs, and the combinations the callers use (noted).
EPILOGUES = [
    (NONE, NONE, "f", True, False, None),          # linear layers, transposed convs, RVQ scores (bias * gamma)
    (GELU, NONE, "h", True, False, None),          # ConvNeXt pwconv1 -> EPI_HI
    (NONE, NONE, "f", True, True, "inplace"),      # ConvNeXt pwconv2 -> EPI_F32
    (NONE, NONE, "h", False, False, None),         # EPI_HI without bias
    (NONE, NONE, "f", False, True, "sep"),         # EPI_F32 without bias
    (NONE, NONE, "fh", True, True, "inplace"),
    (SWIGLU, NONE, "h", False, False, None),       # transformer / LM feed-forward
    (SWIGLU, NONE, "f", True, True, "sep"),
    (SWIGLU, ELU, "fhl", False, False, None),
    (SWIGLU, SNAKE, "fh", True, False, "inplace"),
    (ELU, NONE, "hl", True, False, None),          # semantic residual unit conv 1
    (ELU, ELU, "h", False, True, None),
    (ELU, SNAKE, "fhl", True, True, "inplace"),
    (TANH, NONE, "f", True, False, None),          # BiCodec conv_f
    (TANH, ELU, "fhl", True, False, "sep"),
    (TANH, SNAKE, "h", False, True, "sep"),
    (SNAKE, NONE, "hl", True, False, None),        # BiCodec dilated conv
    (SNAKE, NONE, "f", False, True, "sep"),
    (SNAKE, ELU, "fh", False, False, "inplace"),
    (SNAKE, SNAKE, "fh", True, True, "sep"),
    (NONE, ELU, "fhl", True, False, None),         # semantic encoder convs
    (NONE, ELU, "fhl", False, False, "inplace"),   # semantic residual unit conv 2
    (NONE, SNAKE, "hl", True, False, "sep"),       # BiCodec 1x1 conv + residual, no fp32 trunk
    (NONE, SNAKE, "fhl", True, False, "sep"),      # ... with the trunk
    (GELU, NONE, "f", True, False, "sep"),         # SSL positional conv
    (GELU, ELU, "fh", False, True, None),
    (GELU, SNAKE, "hl", False, False, "sep"),
]


def _fast_kind(n, act, act2, outs, gamma, res, ld):
    """Mirror of classify_epilogue (csrc/gemm.cu) for an 8-byte aligned bias: 'hi', 'f32' or None."""
    if n % 2 or act2 != NONE or ld % 2:
        return None
    if outs == "h" and not gamma and res is None and act in (NONE, GELU):
        return "hi"
    if outs == "f" and act == NONE:
        return "f32"
    return None


def _kernel_name(split, n):
    return "gemm_tc_kernel<3,128,3>" if split else "gemm_tc_kernel<1,256,4>" if n > 128 else "gemm_tc_kernel<1,128,6>"


def _alphas(k, g):
    """Snake alpha per column: 1e-3 .. 60 log-spaced, shuffled, so that |alpha x| crosses snake_f's branch point at 64."""
    a = torch.logspace(-3, math.log10(60.0), k, dtype=torch.float64).float()
    return a[torch.randperm(k, generator=g)].to(DEV)


def _snake(v, a):
    return v + torch.sin(a * v) ** 2 / (a + 1e-9)


def _act(code, v, alpha=None):
    if code == GELU:
        return F.gelu(v)
    if code == ELU:
        return F.elu(v)
    if code == TANH:
        return torch.tanh(v)
    if code == SNAKE:
        return _snake(v, alpha.double())
    return v


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _within(name, got, ref, bound):
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite values inside the output window"
    err = (got.double() - ref).abs()
    bad = err > bound
    assert not bool(bad.any()), (f"{name}: {int(bad.sum())} of {bad.numel()} elements beyond the bound; worst excess "
                                 f"{float((err - bound).max()):.3e}, max error {float(err.max()):.3e}")


def run_gemm_case(split, n, K, act, act2, outs, bias, gamma, res, *, batched, pitch, taps=1, stride=1, dil=1,
                  grouped=False, seed=0):
    from unified_audio_b200 import ops
    B, m = (3, 70) if batched else (1, 200)
    rpb, off = (m + 5, 2) if batched else (m, 0)          # padded output rowmaps: pad rows before and after every batch
    C = 64 if grouped else K                              # channels contracted per tap
    a_ld, col_off = (3 * 64, 64) if grouped else (K, 0)
    rows = m * stride + (taps - 1) * dil
    rows += (-rows) % stride
    n_out = n // 2 if act == SWIGLU else n
    ld, ld_r = n_out + pitch, n_out + pitch + 2
    g = torch.Generator(device="cpu").manual_seed(seed)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(DEV)
    x = rnd(B, rows, a_ld)
    w = rnd(n, taps * C, scale=1.5 * (taps * C) ** -0.5)
    a, wp = ops.Planes.from_f32(x, split), ops.Planes.from_f32(w, split)
    bvec = rnd(n, scale=0.5) if bias else None
    gvec = rnd(n_out) if gamma else None
    alpha = _alphas(n, g) if act == SNAKE else None
    alpha2 = _alphas(n_out, g) if act2 == SNAKE else None
    rint = rnd(B, m, n_out) if res is not None else None

    def launch(bias_t, simt=False):
        o32 = torch.full((B, rpb, ld), float("nan"), device=DEV) if "f" in outs else None
        pl = torch.full((2, B, rpb, ld), HALF_SENTINEL, dtype=torch.float16, device=DEV) if "h" in outs else None
        resmap = None
        if res == "sep":
            r = torch.full((B, rpb, ld_r), float("nan"), device=DEV)
            r[:, off:off + m, :n_out] = rint
            resmap = ops.rowmap(r, ld_r, rpb, off)
        elif res == "inplace":
            o32[:, off:off + m, :n_out] = rint
            resmap = ops.rowmap(o32, ld, rpb, off)
        ops.gemm(a, wp, n, a_batch=B, a_rows_per_batch=rows, a_ld=a_ld, m_per_batch=m, taps=taps, stride=stride, dilation=dil,
                 bias=bias_t, gamma=gvec, residual=resmap, act=act, act2=act2, act_param=alpha, act2_param=alpha2,
                 out_f32=ops.rowmap(o32, ld, rpb, off) if o32 is not None else None,
                 out_planes=ops.Planes(pl[0], pl[1] if "l" in outs else None) if pl is not None else None,
                 out_planes_map=(ld, rpb, off), a_cols=64 if grouped else 0, a_col_off=col_off, simt=simt)
        return o32, pl

    o32, pl = launch(bvec)
    torch.cuda.synchronize()
    assert ops.gemm_kernel_name(m, n, split) == _kernel_name(split, n)

    # fp64 reference over the planes the kernel reads (split: hi*hi + lo*hi + hi*lo, the lo*lo term omitted)
    ah, wh = a.hi.double()[..., col_off:col_off + C], wp.hi.double()
    al = a.lo.double()[..., col_off:col_off + C] if split else None
    wl = wp.lo.double() if split else None
    base = torch.arange(m, device=DEV) * stride
    acc = torch.zeros(B, m, n, dtype=torch.float64, device=DEV)
    for t in range(taps):
        r_idx, ws = base + t * dil, slice(t * C, (t + 1) * C)
        acc += ah[:, r_idx] @ wh[:, ws].t()
        if split:
            acc += al[:, r_idx] @ wh[:, ws].t() + ah[:, r_idx] @ wl[:, ws].t()
    v = acc + (bvec.double() if bias else 0.0)
    scale = float(v.abs().max())
    if act == SWIGLU:
        v = F.silu(v[..., 0::2]) * v[..., 1::2]
    else:
        v = _act(act, v, alpha)
    if gamma:
        v = v * gvec.double()
    if res is not None:
        v = v + rint.double()
    # how far the epilogue can stretch an accumulator error: Snake's slope is 1 + sin(2 alpha x) <= 2, SwiGLU's about
    # 1.1 |up| + |silu(gate)|, gamma multiplies it
    lip = 2.0 ** ((act == SNAKE) + (act2 == SNAKE)) * (2.2 * scale if act == SWIGLU else 1.0)
    lip *= max(1.0, float(gvec.abs().max())) if gamma else 1.0
    tol = GEMM_TOL * scale * lip

    inside = torch.zeros(B, rpb, ld, dtype=torch.bool, device=DEV)
    inside[:, off:off + m, :n_out] = True
    tag = f"{_kernel_name(split, n)} n={n} act={ACT_NAMES[act]} act2={ACT_NAMES[act2]} outs={outs}"
    if o32 is not None:
        got = o32[:, off:off + m, :n_out]
        e = float((got.double() - v).abs().max()) / scale
        print(f"{tag}: fp32 error {e:.2e} of the largest pre-activation")
        _within(f"{tag} fp32", got, v, tol + 2.0 ** -22 * v.abs())
        assert bool(o32[~inside].isnan().all()), f"{tag}: fp32 written outside its window"
    if pl is not None:
        u = _act(act2, v, alpha2)
        hi, lo = pl[0][:, off:off + m, :n_out], pl[1][:, off:off + m, :n_out]
        got = hi.double() + (lo.double() if "l" in outs else 0.0)
        rep = 2.0 ** -21 if "l" in outs else 2.0 ** -11      # the planes' own rounding: hi + lo ~ 2^-22, hi alone 2^-11
        _within(f"{tag} planes", got, u, tol + rep * u.abs())
        assert bool((pl[0][~inside] == HALF_SENTINEL).all()), f"{tag}: hi plane written outside its window"
        if "l" in outs:
            assert bool((pl[1][~inside] == HALF_SENTINEL).all()), f"{tag}: lo plane written outside its window"
        else:
            assert bool((pl[1] == HALF_SENTINEL).all()), f"{tag}: lo plane written although only hi was requested"
        if act2 != NONE and o32 is not None:
            # act2 against the kernel's own fp32 output: the bound of the activation alone
            vk = o32[:, off:off + m, :n_out].double()
            uk = _act(act2, vk, alpha2)
            bound = rep * uk.abs() + 2.0 ** -25          # + half the fp16 subnormal spacing
            if act2 == SNAKE:                            # sin error 2 SIN_ERR |sin| / alpha, fp32 rounding of alpha x and the fma
                a2 = alpha2.double()
                bound = bound + 2 * SIN_ERR * torch.sin(a2 * vk).abs() / (a2 + 1e-9) + 1e-12 / a2 + 2e-7 * vk.abs()
            _within(f"{tag} act2 on the kernel's fp32 output", got, uk, bound)

    # the SIMT evaluation of the same descriptor
    s32, spl = launch(bvec, simt=True)
    torch.cuda.synchronize()
    if o32 is not None:
        _within(f"{tag} vs SIMT fp32", o32[:, off:off + m, :n_out], s32[:, off:off + m, :n_out].double(),
                tol + 2.0 ** -22 * v.abs())
        assert bool(s32[~inside].isnan().all())
    if pl is not None:
        both = lambda p: p[0][:, off:off + m, :n_out].double() + (p[1][:, off:off + m, :n_out].double() if "l" in outs else 0.0)
        rep2 = 2.0 ** -20 if "l" in outs else 2.0 ** -10
        _within(f"{tag} vs SIMT planes", both(pl), both(spl), 2 * tol + rep2 * both(spl).abs() + 2.0 ** -24)

    # the fast kinds do the same arithmetic in the same order as epilogue_pair: a bias at a 4-byte offset makes
    # classify_epilogue fall back to the generic epilogue, whose vector branch must give the same bits
    if bias and _fast_kind(n, act, act2, outs, gamma, res, ld):
        buf = torch.empty(n + 1, device=DEV)
        buf[1:] = bvec
        g32, gpl = launch(buf[1:])
        torch.cuda.synchronize()
        if o32 is not None:
            assert torch.equal(_bits(o32), _bits(g32)), f"{tag}: EPI_F32 and epilogue_pair differ"
        if pl is not None:
            assert torch.equal(_bits(pl), _bits(gpl)), f"{tag}: EPI_HI and epilogue_pair differ"


def _cases():
    out = []
    for inst, (split, ns) in INSTS.items():
        for i, (act, act2, outs, bias, gamma, res) in enumerate(EPILOGUES):
            n = ns[i % len(ns)]
            fast = _fast_kind(n + n % 2, act, act2, outs, gamma, res, 0) is not None
            if n % 2 and (act == SWIGLU or fast):   # keep the fast kinds reachable: an even n of the same instantiation
                n += 1
            pitch = (0, 8)[i % 2] if fast else (0, 8, 3)[i % 3]
            K = (64, 448)[i % 2]                     # one K-block; 7 K-blocks, more than any instantiation has stages
            batched = (i // 2) % 2 == 1              # 3 batches of 70 rows through padded rowmaps
            out.append(pytest.param(split, n, K, act, act2, outs, bias, gamma, res, batched, pitch,
                                    id=f"{inst}-n{n}-K{K}-{ACT_NAMES[act]}-{ACT_NAMES[act2]}-{outs}"
                                       f"{'-b' if bias else ''}{'-g' if gamma else ''}{'-r' + res if res else ''}"
                                       f"{'-batched' if batched else ''}-pitch{pitch}"))
    return out


@pytest.mark.parametrize("split,n,K,act,act2,outs,bias,gamma,res,batched,pitch", _cases())
def test_gemm_epilogue(lib, split, n, K, act, act2, outs, bias, gamma, res, batched, pitch):
    run_gemm_case(split, n, K, act, act2, outs, bias, gamma, res, batched=batched, pitch=pitch, seed=n * 31 + act * 7 + act2)


# convolutions: (taps, stride, dilation, grouped) with the epilogue their callers use
CONV_CASES = [
    # semantic encoder conv k3 -> fp32 trunk + ELU planes into the next padded buffer
    ("split", 256, 3, 1, 1, False, (NONE, ELU, "fhl", True, False, None)),
    ("n256", 520, 3, 1, 1, False, (NONE, ELU, "fhl", True, False, None)),
    # strided down-sampling conv on the 256-wide tile (and on the others)
    ("n256", 260, 4, 2, 1, False, (NONE, ELU, "fh", True, False, None)),
    ("n256", 257, 3, 2, 1, False, (NONE, NONE, "f", True, False, None)),
    ("split", 260, 4, 2, 1, False, (NONE, NONE, "f", True, True, "sep")),
    ("n128", 128, 4, 2, 1, False, (GELU, NONE, "h", True, False, None)),
    # BiCodec dilated residual unit: Snake (act) -> planes
    ("n256", 130, 7, 1, 3, False, (SNAKE, NONE, "hl", True, False, None)),
    ("n128", 96, 7, 1, 9, False, (SNAKE, NONE, "h", True, False, None)),
    # BiCodec conv_f: one output channel, tanh
    ("n128", 1, 7, 1, 1, False, (TANH, NONE, "f", True, False, None)),
    ("split", 1, 7, 1, 1, False, (TANH, NONE, "f", True, False, None)),
    # SSL grouped positional conv: channels [64, 128) of a 192-channel buffer, GELU, + residual, pitch > n
    ("n128", 48, 5, 1, 1, True, (GELU, NONE, "f", True, False, "sep")),
    ("split", 48, 5, 1, 1, True, (GELU, NONE, "f", True, False, "sep")),
    ("n256", 130, 5, 1, 1, True, (GELU, NONE, "f", True, False, "sep")),
]


@pytest.mark.parametrize("inst,n,taps,stride,dil,grouped,epi", CONV_CASES,
                         ids=[f"{c[0]}-n{c[1]}-k{c[2]}s{c[3]}d{c[4]}{'-grouped' if c[5] else ''}" for c in CONV_CASES])
def test_gemm_epilogue_conv(lib, inst, n, taps, stride, dil, grouped, epi):
    split = INSTS[inst][0]
    run_gemm_case(split, n, 128, *epi, batched=True, pitch=16 if grouped else 0, taps=taps, stride=stride, dil=dil,
                  grouped=grouped, seed=taps * 100 + n)


@pytest.mark.parametrize("inst,n", [("split", 260), ("n128", 128), ("n256", 260)])
@pytest.mark.parametrize("kind", ["f32", "hi_fast", "hi_pair", "hi_scalar", "hi_lo", "f32_hi"])
def test_gemm_nan_and_saturation(lib, inst, n, kind):
    """A NaN operand row gives NaN in every output kind, and a row beyond the fp16 range saturates the hi plane to
    +-65504 with the right sign, on the vector stores (EPI_HI, epilogue_pair's half2 branch) and the scalar one alike."""
    from unified_audio_b200 import ops
    split = INSTS[inst][0]
    M, K = 130, 128
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(M, K, generator=g)
    x[3] = float("nan")
    x[3, 1:] = 0.0                              # one NaN element is enough to poison the whole row
    x[100] = 60000.0                            # |acc| well beyond 65504 in most columns
    x = x.to(DEV)
    w = (torch.randn(n, K, generator=g) * K ** -0.5).to(DEV)
    bias = (torch.randn(n, generator=g) * 0.1).to(DEV)
    a, wp = ops.Planes.from_f32(x, split), ops.Planes.from_f32(w, split)
    ld = n + 1 if kind == "hi_scalar" else n     # an odd pitch forces the scalar store
    bias_t = bias
    if kind == "hi_pair":                       # a 4-byte aligned bias: generic epilogue, half2 branch of epilogue_pair
        buf = torch.empty(n + 1, device=DEV)
        buf[1:] = bias
        bias_t = buf[1:]
    o32 = torch.full((M, ld), 7.0, device=DEV) if kind in ("f32", "f32_hi") else None
    pl = ops.Planes(torch.zeros(M, ld, dtype=torch.float16, device=DEV),
                    torch.zeros(M, ld, dtype=torch.float16, device=DEV) if kind in ("hi_lo", "f32_hi") else None) \
        if kind != "f32" else None
    ops.gemm(a, wp, n, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias_t,
             out_f32=ops.rowmap(o32, ld, M, 0) if o32 is not None else None, out_planes=pl, out_planes_map=(ld, M, 0))
    torch.cuda.synchronize()
    ref = planes_ref64(a) @ planes_ref64(wp).t() + bias.double()
    if o32 is not None:
        assert bool(o32[3, :n].isnan().all()), "fp32: a NaN row must stay NaN"
        assert bool(torch.isfinite(o32[torch.arange(M, device=DEV) != 3, :n]).all())
    if pl is not None:
        hi = pl.hi[:, :n]
        assert bool(hi[3].isnan().all()), f"{kind}: the hi plane of a NaN row must be NaN, got {hi[3, :4].tolist()}"
        if pl.lo is not None:
            assert bool(pl.lo[3, :n].isnan().all()), "the lo plane of a NaN row must be NaN"
        big = ref[100].abs() > 65600
        assert int(big.sum()) >= 10
        assert bool((hi[100][big].double() == 65504.0 * ref[100][big].sign()).all()), "saturation to +-65504"
        others = torch.arange(M, device=DEV) != 3
        assert bool(torch.isfinite(hi[others]).all())


def planes_ref64(p):
    return p.hi.double() + (p.lo.double() if p.lo is not None else 0.0)
