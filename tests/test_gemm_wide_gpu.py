"""qb_gemm across its tile widths (128 x 256 tiles for single-pass n > 128, 128 x 128 otherwise) and epilogue kinds
(GELU -> fp16 hi, bias * gamma + residual -> fp32, the element-by-element generic path), against the fp64 product of
the fp16 planes."""
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


def _ref(a, wp, split):
    ref = planes_ref(a) @ planes_ref(wp).t()
    if split:  # the kernel omits the lo*lo term
        ref = ref - a.lo.double() @ wp.lo.double().t()
    return ref


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("N", [128, 129, 257])
def test_gemm_tile_width_boundary(lib, split, N):
    from unified_audio_b200 import ops
    M, K = 300, 192
    x, w, bias = _mk((M, K), 1), _mk((N, K), 2, K ** -0.5), _mk((N,), 3)
    a, wp = ops.Planes.from_f32(x, split), ops.Planes.from_f32(w, split)
    out = torch.full((M, N), float("nan"), device=DEV)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias, out_f32=ops.rowmap(out, N, M, 0))
    torch.cuda.synchronize()
    assert ops.gemm_kernel_name(M, N, split) == ("gemm_tc_kernel<3,128,3>" if split else
                                                 "gemm_tc_kernel<1,256,4>" if N > 128 else "gemm_tc_kernel<1,128,6>")
    assert relerr(out, _ref(a, wp, split) + bias.double()) < 2e-5


def test_gemm_single_pass_gelu_hi(lib):
    """pwconv1's epilogue: bias + GELU -> fp16 hi plane only, on a 256-wide tile with a partial last tile."""
    import torch.nn.functional as F
    from unified_audio_b200 import ops
    M, N, K = 260, 640, 256
    x, w, bias = _mk((M, K), 4), _mk((N, K), 5, K ** -0.5), _mk((N,), 6)
    a, wp = ops.Planes.from_f32(x, False), ops.Planes.from_f32(w, False)
    out = ops.Planes(torch.full((M, N), float("nan"), device=DEV, dtype=torch.float16), None)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias, act=ops.ACT_GELU,
             out_planes=out, out_planes_map=(N, M, 0))
    torch.cuda.synchronize()
    ref = F.gelu(_ref(a, wp, False) + bias.double())
    # the output is one fp16 plane: its own rounding (half an ulp, 2^-11 relative) on top of the GEMM's 2e-5
    assert bool(((out.hi.double() - ref).abs() <= ref.abs() * 2.0 ** -11 + 2e-5 * ref.abs().max()).all())


def test_gemm_single_pass_gamma_residual_f32(lib):
    """pwconv2's epilogue: (acc + bias) * gamma + residual -> fp32, in place, on 256-wide tiles."""
    from unified_audio_b200 import ops
    M, N, K = 300, 768, 320
    x, w, bias, gamma, res = _mk((M, K), 7), _mk((N, K), 8, K ** -0.5), _mk((N,), 9), _mk((N,), 10), _mk((M, N), 11)
    a, wp = ops.Planes.from_f32(x, False), ops.Planes.from_f32(w, False)
    r2 = res.clone()
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias, gamma=gamma,
             residual=ops.rowmap(r2, N, M, 0), out_f32=ops.rowmap(r2, N, M, 0))
    torch.cuda.synchronize()
    assert relerr(r2, (_ref(a, wp, False) + bias.double()) * gamma.double() + res.double()) < 2e-5


@pytest.mark.parametrize("split", [False, True])
def test_gemm_odd_pitch_scalar_store(lib, split):
    """An odd output pitch rules out the vector stores: every element goes through the scalar path."""
    from unified_audio_b200 import ops
    M, N, K, ld = 200, 384, 128, 385
    x, w, bias, gamma = _mk((M, K), 12), _mk((N, K), 13, K ** -0.5), _mk((N,), 14), _mk((N,), 15)
    a, wp = ops.Planes.from_f32(x, split), ops.Planes.from_f32(w, split)
    out = torch.full((M, ld), float("nan"), device=DEV)
    ops.gemm(a, wp, N, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bias, gamma=gamma,
             out_f32=ops.rowmap(out, ld, M, 0))
    torch.cuda.synchronize()
    assert relerr(out[:, :N], (_ref(a, wp, split) + bias.double()) * gamma.double()) < 2e-5
    assert bool(out[:, N:].isnan().all())


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("k,dil,Cin,Cout,T,B", [(3, 3, 128, 384, 90, 2), (3, 1, 128, 512, 500, 8)])
def test_gemm_conv_wide(lib, split, k, dil, Cin, Cout, T, B):
    """Dilated conv on a 256-wide tile, and 8 batches of 500 rows (a partial M-tile at the end of every batch)."""
    import torch.nn.functional as F
    from unified_audio_b200 import ops
    pad = dil * (k - 1) // 2
    Tp = T + 2 * pad
    x = _mk((B, T, Cin), 16)
    w = _mk((Cout, Cin, k), 17, (Cin * k) ** -0.5)
    bias = _mk((Cout,), 18)
    buf = ops.Planes.zeros((B, Tp, Cin), split, DEV)
    ops.rows_to_planes(x.reshape(B * T, Cin), B, T, Cin, buf, Cin, Tp, pad)
    wp = ops.Planes.from_f32(w.permute(0, 2, 1).reshape(Cout, k * Cin), split)
    out = torch.full((B, T, Cout), float("nan"), device=DEV)
    ops.gemm(buf, wp, Cout, a_batch=B, a_rows_per_batch=Tp, a_ld=Cin, m_per_batch=T, taps=k, dilation=dil, bias=bias,
             out_f32=ops.rowmap(out, Cout, T, 0))
    torch.cuda.synchronize()
    xq = planes_ref(ops.Planes(buf.hi[:, pad:pad + T], buf.lo[:, pad:pad + T] if split else None))
    ref = F.conv1d(xq.transpose(1, 2), planes_ref(wp).reshape(Cout, k, Cin).permute(0, 2, 1), bias.double(),
                   padding=pad, dilation=dil).transpose(1, 2)
    if split:
        xl = buf.lo[:, pad:pad + T].double()
        ref = ref - F.conv1d(xl.transpose(1, 2), wp.lo.double().reshape(Cout, k, Cin).permute(0, 2, 1),
                             padding=pad, dilation=dil).transpose(1, 2)
    assert relerr(out, ref) < 3e-5
