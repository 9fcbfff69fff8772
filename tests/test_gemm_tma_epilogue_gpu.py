"""The TMA epilogues of qb_gemm (EPI_HI: bias, GELU -> fp16 hi plane; EPI_F32: bias, gamma, residual -> fp32) on each kernel
instantiation, against an fp64 reference of the same contraction over the fp16 planes the kernel reads.

Output rows run through padded row maps (rows_per_batch > m_per_batch, a nonzero row offset) whose guard rows and pad columns
start as a sentinel and must stay untouched; m_per_batch = 500 leaves a partial last tile in every batch, and n is not a
multiple of the tile width.  The in-place residual must give the bits of the out-of-place one, and a row pitch TMA cannot
address (not a multiple of 16 bytes) takes the generic epilogue, which must give the same bits as the TMA one.  So does an
fp16 row of n elements that is not a multiple of 16 bytes: a TMA store would write its last chunk past n, into the pad."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF_SENTINEL = -1234.0
GEMM_TOL = 2e-5                  # relative to the largest pre-activation, as tests/test_gemm_epilogue_gpu.py
NONE, GELU = 0, 1

# instantiation -> (split operands, n): n > 128 picks the 256-wide tile unless split; none of them a multiple of the tile width,
# all of them rows of whole 16-byte chunks in fp16 and fp32
INSTS = {"split": (True, 200), "n128": (False, 104), "n256": (False, 312)}
B, M, K = 3, 500, 448
RPB, OFF = M + 7, 3


def _planes_ref(p):
    return p.hi.double() + (p.lo.double() if p.lo is not None else 0.0)


def _setup(split, n, seed):
    from unified_audio_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(seed)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(DEV)   # noqa: E731
    a = ops.Planes.from_f32(rnd(B, M, K), split)
    w = ops.Planes.from_f32(rnd(n, K, scale=1.5 * K ** -0.5), split)
    acc = torch.einsum("bmk,nk->bmn", _planes_ref(a), _planes_ref(w))
    if split:                                      # the kernel omits the lo * lo term
        acc -= torch.einsum("bmk,nk->bmn", a.lo.double(), w.lo.double())
    return a, w, acc, rnd


def _gemm(a, w, n, **kw):
    from unified_audio_b200 import ops
    ops.gemm(a, w, n, a_batch=B, a_rows_per_batch=M, a_ld=K, m_per_batch=M, **kw)


def _check(tag, got, ref, scale, rep):
    """|got - ref| within the accumulation bound plus the output's own rounding (rep relative)."""
    assert bool(torch.isfinite(got).all()), f"{tag}: non-finite values in the output window"
    excess = (got.double() - ref).abs() - (GEMM_TOL * scale + rep * ref.abs())
    assert float(excess.max()) <= 0.0, f"{tag}: {int((excess > 0).sum())} elements beyond the bound (scale {scale:.3e})"


@pytest.mark.parametrize("inst", list(INSTS))
@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("row", ["whole", "partial"])
def test_epi_hi(lib, inst, gelu, bias, row):
    from unified_audio_b200 import ops
    split, n = INSTS[inst]
    n -= 4 if row == "partial" else 0              # 8 bytes short of a 16-byte multiple: the generic epilogue
    a, w, acc, rnd = _setup(split, n, 11 + 2 * gelu + bias)
    bvec = rnd(n, scale=0.5) if bias else None

    def run(ld):
        hi = torch.full((B, RPB, ld), HALF_SENTINEL, dtype=torch.float16, device=DEV)
        _gemm(a, w, n, bias=bvec, act=GELU if gelu else NONE, out_planes=ops.Planes(hi, None), out_planes_map=(ld, RPB, OFF))
        return hi

    ld = n + (-n) % 8 + 8                          # 16-byte row pitch: the TMA epilogue
    hi = run(ld)
    torch.cuda.synchronize()
    v = acc + (bvec.double() if bias else 0.0)
    scale = float(v.abs().max())
    ref = F.gelu(v) if gelu else v
    _check(f"{inst} hi", hi[:, OFF:OFF + M, :n], ref, scale, 2.0 ** -11)
    inside = torch.zeros_like(hi, dtype=torch.bool)
    inside[:, OFF:OFF + M, :n] = True
    assert bool((hi[~inside] == HALF_SENTINEL).all()), f"{inst}: guard rows or pad columns written"
    # a pitch of ld + 2 halves (4 bytes off 16): the generic epilogue, same bits
    hg = run(ld + 2)
    torch.cuda.synchronize()
    assert torch.equal(hg[:, OFF:OFF + M, :n].view(torch.int16), hi[:, OFF:OFF + M, :n].view(torch.int16)), \
        f"{inst}: generic and TMA epilogues differ"


F32_CASES = [  # (bias, gamma, residual)
    (True, False, False),
    (False, True, False),
    (False, False, True),
    (True, True, True),                            # ConvNeXt pwconv2
]


@pytest.mark.parametrize("inst", list(INSTS))
@pytest.mark.parametrize("bias,gamma,res", F32_CASES, ids=["bias", "gamma", "residual", "bias-gamma-residual"])
def test_epi_f32(lib, inst, bias, gamma, res):
    from unified_audio_b200 import ops
    split, n = INSTS[inst]
    a, w, acc, rnd = _setup(split, n, 31 + 4 * bias + 2 * gamma + res)
    bvec = rnd(n, scale=0.5) if bias else None
    gvec = rnd(n) if gamma else None
    rint = rnd(B, M, n) if res else None

    def run(ld, inplace):
        out = torch.full((B, RPB, ld), float("nan"), device=DEV)
        resmap = None
        if res and inplace:
            out[:, OFF:OFF + M, :n] = rint
            resmap = ops.rowmap(out, ld, RPB, OFF)
        elif res:
            r = torch.full((B, RPB + 2, ld + 4), float("nan"), device=DEV)
            r[:, OFF + 1:OFF + 1 + M, :n] = rint
            resmap = ops.rowmap(r, ld + 4, RPB + 2, OFF + 1)
        _gemm(a, w, n, bias=bvec, gamma=gvec, residual=resmap, out_f32=ops.rowmap(out, ld, RPB, OFF))
        return out

    ld = n + (-n) % 4 + 4                          # 16-byte row pitch: the TMA epilogue
    out = run(ld, inplace=False)
    torch.cuda.synchronize()
    v = acc + (bvec.double() if bias else 0.0)
    scale = float(v.abs().max()) * (max(1.0, float(gvec.abs().max())) if gamma else 1.0)
    if gamma:
        v = v * gvec.double()
    if res:
        v = v + rint.double()
    _check(f"{inst} f32", out[:, OFF:OFF + M, :n], v, scale, 2.0 ** -22)
    inside = torch.zeros_like(out, dtype=torch.bool)
    inside[:, OFF:OFF + M, :n] = True
    assert bool(out[~inside].isnan().all()), f"{inst}: guard rows or pad columns written"
    bits = lambda t: t[:, OFF:OFF + M, :n].contiguous().view(torch.int32)   # noqa: E731
    if res:
        same = run(ld, inplace=True)
        torch.cuda.synchronize()
        assert torch.equal(bits(same), bits(out)), f"{inst}: in-place residual differs from out-of-place"
        assert bool(same[~inside].isnan().all()), f"{inst}: in-place: guard rows or pad columns written"
    # a pitch of ld + 2 floats (8 bytes off 16): the generic epilogue, same bits
    gen = run(ld + 2, inplace=False)
    torch.cuda.synchronize()
    assert torch.equal(bits(gen), bits(out)), f"{inst}: generic and TMA epilogues differ"


@pytest.mark.parametrize("inst", list(INSTS))
def test_epi_hi_nan_and_saturation(lib, inst):
    """A NaN row stays NaN and a row beyond the fp16 range saturates to +-65504 through the TMA store."""
    from unified_audio_b200 import ops
    split, n = INSTS[inst]
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(B, M, K, generator=g)
    x[1, 3] = 0.0
    x[1, 3, 0] = float("nan")
    x[2, 499] = 60000.0
    x = x.to(DEV)
    w = (torch.randn(n, K, generator=g) * K ** -0.5).to(DEV)
    a, wp = ops.Planes.from_f32(x, split), ops.Planes.from_f32(w, split)
    ld = n + (-n) % 8
    hi = torch.zeros(B, M, ld, dtype=torch.float16, device=DEV)
    _gemm(a, wp, n, out_planes=ops.Planes(hi, None), out_planes_map=(ld, M, 0))
    torch.cuda.synchronize()
    ref = _planes_ref(a)[2, 499] @ _planes_ref(wp).t()
    assert bool(hi[1, 3, :n].isnan().all())
    big = ref.abs() > 65600
    assert int(big.sum()) >= 10
    assert bool((hi[2, 499, :n][big].double() == 65504.0 * ref[big].sign()).all())


@pytest.mark.parametrize("inst", list(INSTS))
@pytest.mark.parametrize("out", ["f32", "hi"])
def test_many_tiles_per_block(lib, inst, out):
    """K = 64 (one K-block) over 600 row tiles: every block runs many tiles back to back, so each epilogue starts while the
    previous tile's stores may still be reading the subtile buffers.  Same bits as the generic epilogue."""
    from unified_audio_b200 import ops
    split, n = INSTS[inst]
    m, k = 128 * 600, 64
    g = torch.Generator(device="cpu").manual_seed(7)
    a = ops.Planes.from_f32(torch.randn(m, k, generator=g).to(DEV), split)
    w = ops.Planes.from_f32((torch.randn(n, k, generator=g) * k ** -0.5).to(DEV), split)

    def run(ld):
        if out == "f32":
            o = torch.full((m, ld), float("nan"), device=DEV)
            ops.gemm(a, w, n, a_batch=1, a_rows_per_batch=m, a_ld=k, m_per_batch=m, out_f32=ops.rowmap(o, ld, m, 0))
        else:
            o = torch.full((m, ld), HALF_SENTINEL, dtype=torch.float16, device=DEV)
            ops.gemm(a, w, n, a_batch=1, a_rows_per_batch=m, a_ld=k, m_per_batch=m, out_planes=ops.Planes(o, None),
                     out_planes_map=(ld, m, 0))
        torch.cuda.synchronize()
        return o[:, :n].contiguous().view(torch.int32 if out == "f32" else torch.int16)

    step = 4 if out == "f32" else 8
    assert torch.equal(run(n + step), run(n + step + 2)), f"{inst} {out}: TMA and generic epilogues differ"
