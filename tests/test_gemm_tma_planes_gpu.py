"""The fp16 planes written by qb_gemm's TMA epilogues: EPI_HI with a lo plane and GELU / ELU / SwiGLU, and EPI_F32 with
(ELU ->) hi + lo planes beside its fp32 output, against an fp64 reference of the same contraction over the fp16 planes the
kernel reads.

As in tests/test_gemm_tma_epilogue_gpu.py, m_per_batch = 500 leaves a partial last tile in every batch, n is not a multiple of
the tile width, and outputs run through padded row maps whose guard rows and pad columns start as a sentinel and must stay
untouched.  The planes of EPI_F32 go through their own row map, rows_per_batch = m + 2 at offset 1, the zero-padded input of
the next k = 3 conv.  Every case is also run with a planes pitch 4 bytes off a multiple of 16, which TMA cannot address: the
generic epilogue, which must give the same bits."""
import pytest
import torch
import torch.nn.functional as F

from test_gemm_tma_epilogue_gpu import B, GEMM_TOL, HALF_SENTINEL, INSTS, K, M, OFF, RPB, _gemm, _planes_ref, _setup

pytestmark = pytest.mark.gpu
DEV = "cuda"
NONE, GELU, SWIGLU, ELU = 0, 1, 2, 3
ACTS = {"none": NONE, "gelu": GELU, "elu": ELU, "swiglu": SWIGLU}


def _act(act, v):
    if act == SWIGLU:
        return F.silu(v[..., 0::2]) * v[..., 1::2]
    return F.gelu(v) if act == GELU else F.elu(v) if act == ELU else v


def _within(tag, got, ref, bound):
    assert bool(torch.isfinite(got).all()), f"{tag}: non-finite values in the output window"
    excess = (got.double() - ref).abs() - bound
    assert float(excess.max()) <= 0.0, f"{tag}: {int((excess > 0).sum())} elements beyond the bound"


def _planes(rows, ld, lo):
    from unified_audio_b200 import ops
    hi = torch.full((B, rows, ld), HALF_SENTINEL, dtype=torch.float16, device=DEV)
    return ops.Planes(hi, torch.full_like(hi, HALF_SENTINEL) if lo else None)


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _check_planes(tag, pl, rows, off, n_out, ref, tol):
    """hi (+ lo) within tol + their own rounding of ref; nothing outside rows [off, off + M) x columns [0, n_out) written."""
    lo = pl.lo is not None
    got = pl.hi[:, off:off + M, :n_out].double() + (pl.lo[:, off:off + M, :n_out].double() if lo else 0.0)
    _within(f"{tag} planes", got, ref, tol + (2.0 ** -21 if lo else 2.0 ** -11) * ref.abs())
    inside = torch.zeros(B, rows, pl.hi.shape[-1], dtype=torch.bool, device=DEV)
    inside[:, off:off + M, :n_out] = True
    for t in (pl.hi, pl.lo) if lo else (pl.hi,):
        assert bool((t[~inside] == HALF_SENTINEL).all()), f"{tag}: guard rows or pad columns of the planes written"


# the 128 x 256 tile (<1,256,4>) keeps SwiGLU and the lo plane on the generic epilogue (csrc/gemm.cu, classify_epilogue): its
# cases check that path against fp64 and the pad columns, at both pitches
SWIGLU_N = {"split": 208, "n256": 304}           # 104 / 152 output columns: rows of whole 16-byte chunks
PLANES_CASES = [pytest.param("split", a, lo, id=f"split-{a}-{'hl' if lo else 'h'}") for a in ACTS for lo in (True, False)]
PLANES_CASES += [pytest.param("n256", "swiglu", lo, id=f"n256-swiglu-{'hl' if lo else 'h'}") for lo in (True, False)]


@pytest.mark.parametrize("inst,act,lo", PLANES_CASES)
@pytest.mark.parametrize("bias", [False, True])
def test_epi_planes(lib, inst, act, lo, bias):
    split, n = INSTS[inst]
    code = ACTS[act]
    n = SWIGLU_N[inst] if code == SWIGLU else n
    a, w, acc, rnd = _setup(split, n, 41 + 4 * code + 2 * lo + bias)
    bvec = rnd(n, scale=0.5) if bias else None
    n_out = n // 2 if code == SWIGLU else n

    def run(ld):
        pl = _planes(RPB, ld, lo)
        _gemm(a, w, n, bias=bvec, act=code, out_planes=pl, out_planes_map=(ld, RPB, OFF))
        torch.cuda.synchronize()
        return pl

    ld = n_out + (-n_out) % 8 + 8                  # 16-byte row pitch: the TMA epilogue
    pl = run(ld)
    v = acc + (bvec.double() if bias else 0.0)
    scale = float(v.abs().max())
    lip = 2.2 * scale if code == SWIGLU else 1.0   # SwiGLU's slope, about 1.1 |up| + |silu(gate)|
    _check_planes(f"{inst} {act}", pl, RPB, OFF, n_out, _act(code, v), GEMM_TOL * scale * lip)
    gen = run(ld + 2)                              # 4 bytes off 16: the generic epilogue, same bits
    for t, g in ((pl.hi, gen.hi), (pl.lo, gen.lo)) if lo else ((pl.hi, gen.hi),):
        assert torch.equal(_bits(t[:, OFF:OFF + M, :n_out]), _bits(g[:, OFF:OFF + M, :n_out])), \
            f"{inst} {act}: generic and TMA epilogues differ"


@pytest.mark.parametrize("inst", list(INSTS))
@pytest.mark.parametrize("act2", ["none", "elu"])
@pytest.mark.parametrize("res", [None, "sep", "inplace"])
def test_epi_f32_planes(lib, inst, act2, res):
    """(bias) (+ residual) -> fp32 and (ELU) -> hi + lo planes: the semantic encoder's convs.  The strided conv has a bias and
    no residual, the residual unit's 1x1 conv a residual that is its own output."""
    from unified_audio_b200 import ops
    split, n = INSTS[inst]
    code2, bias = ACTS[act2], res is None
    a, w, acc, rnd = _setup(split, n, 61 + 4 * code2 + (res is not None) + (res == "inplace"))
    bvec = rnd(n, scale=0.5) if bias else None
    rint = rnd(B, M, n) if res else None
    prows = M + 2                                  # planes: rows_per_batch m + 2 at offset 1

    def run(ld, ldp):
        out = torch.full((B, RPB, ld), float("nan"), device=DEV)
        resmap = None
        if res == "inplace":
            out[:, OFF:OFF + M, :n] = rint
            resmap = ops.rowmap(out, ld, RPB, OFF)
        elif res == "sep":
            r = torch.full((B, RPB + 2, ld + 4), float("nan"), device=DEV)
            r[:, OFF + 1:OFF + 1 + M, :n] = rint
            resmap = ops.rowmap(r, ld + 4, RPB + 2, OFF + 1)
        pl = _planes(prows, ldp, True)
        _gemm(a, w, n, bias=bvec, residual=resmap, act2=code2, out_f32=ops.rowmap(out, ld, RPB, OFF), out_planes=pl,
              out_planes_map=(ldp, prows, 1))
        torch.cuda.synchronize()
        return out, pl

    ld, ldp = n + (-n) % 4 + 4, n + (-n) % 8 + 8   # 16-byte row pitches: the TMA epilogue
    out, pl = run(ld, ldp)
    v = acc + (bvec.double() if bias else 0.0)
    scale = float(v.abs().max())
    if res:
        v = v + rint.double()
    tol = GEMM_TOL * scale
    _within(f"{inst} f32", out[:, OFF:OFF + M, :n], v, tol + 2.0 ** -22 * v.abs())
    inside = torch.zeros_like(out, dtype=torch.bool)
    inside[:, OFF:OFF + M, :n] = True
    assert bool(out[~inside].isnan().all()), f"{inst}: guard rows or pad columns of the fp32 output written"
    _check_planes(f"{inst} act2={act2}", pl, prows, 1, n, _act(code2, v), tol)
    # the planes are act2 of the kernel's own fp32 output, rounded by split_f16: hi + lo within 2^-21 of it
    u = _act(code2, out[:, OFF:OFF + M, :n].double())
    got = pl.hi[:, 1:1 + M, :n].double() + pl.lo[:, 1:1 + M, :n].double()
    _within(f"{inst} act2 on the kernel's fp32 output", got, u, 2.0 ** -21 * u.abs() + 2.0 ** -25)
    win = lambda t, o: _bits(t[:, o:o + M, :n])    # noqa: E731
    gen_out, gen_pl = run(ld, ldp + 2)             # planes 4 bytes off 16: the generic epilogue, same bits
    assert torch.equal(win(gen_out, OFF), win(out, OFF)), f"{inst}: generic and TMA epilogues differ in fp32"
    assert torch.equal(win(gen_pl.hi, 1), win(pl.hi, 1)) and torch.equal(win(gen_pl.lo, 1), win(pl.lo, 1)), \
        f"{inst}: generic and TMA epilogues differ in the planes"


@pytest.mark.parametrize("kind", ["hi-lo", "swiglu", "f32-elu"])
def test_planes_nan_and_saturation(lib, kind):
    """A NaN input row stays NaN in both planes, and a row beyond the fp16 range saturates hi to +-65504 through split_f16;
    the same bits as the generic epilogue."""
    from unified_audio_b200 import ops
    split, n = INSTS["split"]
    act = SWIGLU if kind == "swiglu" else NONE
    n = SWIGLU_N["split"] if act == SWIGLU else n
    n_out = n // 2 if act == SWIGLU else n
    g = torch.Generator(device="cpu").manual_seed(9)
    x = torch.randn(B, M, K, generator=g)
    x[1, 3] = 0.0
    x[1, 3, 0] = float("nan")
    x[2, 499] = 60000.0
    a = ops.Planes.from_f32(x.to(DEV), split)
    wp = ops.Planes.from_f32((torch.randn(n, K, generator=g) * K ** -0.5).to(DEV), split)

    def run(ldp):
        pl = _planes(M, ldp, True)
        kw = dict(act=act, out_planes=pl, out_planes_map=(ldp, M, 0))
        if kind == "f32-elu":
            o = torch.empty(B, M, n + (-n) % 4, device=DEV)
            kw.update(act2=ELU, out_f32=ops.rowmap(o, o.shape[-1], M, 0))
        _gemm(a, wp, n, **kw)
        torch.cuda.synchronize()
        return pl

    ldp = n_out + (-n_out) % 8
    pl = run(ldp)
    v = _planes_ref(a)[2, 499] @ _planes_ref(wp).t()
    ref = F.elu(v) if kind == "f32-elu" else _act(act, v)
    assert bool(pl.hi[1, 3, :n_out].isnan().all()) and bool(pl.lo[1, 3, :n_out].isnan().all())
    big = ref.abs() > 65600
    assert int(big.sum()) >= 10
    assert bool((pl.hi[2, 499, :n_out][big].double() == 65504.0 * ref[big].sign()).all())
    gen = run(ldp + 2)
    for t, u in ((pl.hi, gen.hi), (pl.lo, gen.lo)):
        assert torch.equal(_bits(t[..., :n_out]), _bits(u[..., :n_out])), f"{kind}: generic and TMA epilogues differ"


def test_f32_rows_not_whole_chunks(lib):
    """The decoder head's shape: n = 1922 fp32 columns (7688 bytes, half a 16-byte chunk past a multiple) under a 16-byte
    pitch of 1984.  A TMA store would write the whole last chunk, so this row map takes the generic epilogue: the pad columns
    stay untouched, at either pitch."""
    from unified_audio_b200 import ops
    n, ld = 1922, 1984
    g = torch.Generator(device="cpu").manual_seed(13)
    a = ops.Planes.from_f32(torch.randn(1, M, K, generator=g).to(DEV), True)
    w = ops.Planes.from_f32((torch.randn(n, K, generator=g) * K ** -0.5).to(DEV), True)
    bvec = torch.randn(n, generator=g).to(DEV)

    def run(pitch):
        o = torch.full((M, pitch), float("nan"), device=DEV)
        ops.gemm(a, w, n, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, bias=bvec, out_f32=ops.rowmap(o, pitch, M, 0))
        torch.cuda.synchronize()
        return o

    o = run(ld)
    assert bool(o[:, n:].isnan().all()), "pad columns written"
    o2 = run(ld + 2)
    assert bool(o2[:, n:].isnan().all()), "pad columns written"
    ref = (_planes_ref(a)[0] @ _planes_ref(w).t() - a.lo[0].double() @ w.lo.double().t()) + bvec.double()
    _within("dec.head f32", o[:, :n], ref, GEMM_TOL * float(ref.abs().max()) + 2.0 ** -22 * ref.abs())
    assert torch.equal(_bits(o2[:, :n]), _bits(o[:, :n])), "the two pitches differ"
