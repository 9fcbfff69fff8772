"""Every softmax-attention kernel at the score ranges trained weights produce, against fp64 softmax(S) V on the same device.

The scores are planted, not random: q_i = (a_i, 1, r_i, 0 ...), k_j = (b_j, c_j, 1, 0 ...) give S[i, j] = a_i b_j + c_j + r_i with values
of few mantissa bits, RoPE tables cos = 1 / sin = 0, so the prep kernels do one fp32 multiply per element (q * head_dim^-0.5) that
torch reproduces and the reference is taken from the operands a kernel really contracts (rounded to fp16 for the single-pass
kernels).  Each planted case replays the wgmma kernel's reference-maximum rule (csrc/attention_umma.cu: m from key tile 0, moved
when a later tile exceeds it by more than 2^8) on the fp64 scores and asserts that the rescale branch is reached, or not reached, as
the case claims, so a retuned constant cannot silently empty a case.  Tolerances are per-element bounds derived from the operand
and weight roundings of each kernel; every case prints its score span, the moves of the reference maximum and error / bound."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
# key-tile width and rescale distance (log2 units) of fa5_kernel: F5_BK and F5_RESCALE_LOG2, csrc/attention_umma.cu:30-31
F5_BK = 64
F5_RESCALE_LOG2 = 8.0
LOG2E = 1.4426950408889634
SENT = -1234.0                   # exact in fp16, far from any output here
LENGTHS = [1, 63, 64, 65, 127, 128, 129, 193, 257]
B, H = 2, 2                      # every (batch, head) gets its own parameters: a head / batch mix-up cannot hide
# a later tile's maximum just under / just over the rescale distance, as fp16-exact nats: 701/128 = 7.901 and 719/128 = 8.104 log2 units
UNDER, OVER = 701.0 / 128.0, 719.0 / 128.0
assert UNDER * LOG2E < F5_RESCALE_LOG2 - 0.05 and OVER * LOG2E > F5_RESCALE_LOG2 + 0.05
PLANTED = ["ramp", "ramp_noise", "half_a", "half_b", "spike", "sink", "under", "over", "uniform"]
MOVES = {"ramp", "ramp_noise", "spike", "over", "causal"}      # cases that claim a moving reference maximum (as do half_a / half_b)
STAYS = {"sink", "under", "uniform"}                           # and one that stays


# ---------------------------------------------------------------------------------------------- planted operands
def _scale(D):
    """head_dim^-0.5 as the kernels compute it (1.0f / sqrtf(D)), as a Python float holding the fp32 value"""
    return float(1.0 / torch.sqrt(torch.tensor(float(D), dtype=torch.float32)))


def _plant(pattern, Lq, T, D, seed, row0=0):
    """q target (after the 1/sqrt(D) scale), k, v [B, H, *, D] fp32 on the device: queries row0 .. row0 + Lq, keys 0 .. T"""
    g = (torch.arange(B)[:, None] * H + torch.arange(H)[None, :])[..., None].float()          # [B, H, 1]: head index
    i = (torch.arange(Lq) + row0)[None, None, :].float().expand(B, H, Lq)
    j = torch.arange(T)[None, None, :].float().expand(B, H, T)
    tile = torch.floor(j / F5_BK)
    zq, zk = torch.zeros(B, H, Lq), torch.zeros(B, H, T)
    a, r, b, c = zq, zq, zk, zk
    if pattern in ("ramp", "ramp_noise"):        # >= 6 nats per key tile, steeper for later heads and for some rows
        a, b, c = 1.0 + 0.25 * (i % 4), 2.0 * tile, (6.0 + g) * tile + 0.25 * (j % 4)
    elif pattern in ("half_a", "half_b"):        # one half of every 16-row fragment ramps, the other is flat
        first = ((i - row0) % 16) < 8          # by the row's place in its 16-row fragment, which a continuation counts from row0
        a = (first if pattern == "half_a" else ~first).float()
        b, c = (6.0 + g) * tile, 0.25 * (j % 4)
    elif pattern in ("spike", "sink"):           # one key beats the rest by ~80 nats: late in the last tile, or key 0
        js = torch.clamp(T - 1 - g, min=0) if pattern == "spike" else torch.zeros_like(g)
        a, b = 0.5 * (i % 3), 0.25 * ((j % 5) - 2.0)
        c = 0.25 * (((j * 7) % 9) - 4.0) + (j == js).float() * (80.0 + 4.0 * g)
    elif pattern in ("under", "over"):           # tile 0 peaks at 0, every later tile at 7.9 / 8.1 log2 units above it
        c = torch.where(tile == 0, zk, zk + (UNDER if pattern == "under" else OVER)) - 0.25 * ((j % F5_BK) % 3)
        r = 3.0 * g + (i % 2)
    elif pattern == "uniform":                   # all scores of a row equal, +-200 nats
        r = 200.0 * (1.0 - 2.0 * ((i + g) % 2))
    elif pattern == "causal":                    # S = slope (j - i): every masked key outranks every visible one; the last key
        slope = 2.0 ** -g                        # spikes: the diagonal element of the last row, masked for all others
        c, r = slope * j + (j == T - 1).float() * 40.0, -slope * i
    else:
        raise ValueError(pattern)
    gen = torch.Generator().manual_seed(seed)
    q, k = torch.zeros(B, H, Lq, D), torch.zeros(B, H, T, D)
    if pattern == "ramp_noise":                  # the other head dims live: fp16-exact noise, |score change| ~ 0.01 nat
        q = (torch.randn(B, H, Lq, D, generator=gen) / 32).half().float()
        k = (torch.randn(B, H, T, D, generator=gen) / 32).half().float()
    q[..., 0], q[..., 1], q[..., 2] = a, 1.0, r
    k[..., 0], k[..., 1], k[..., 2] = b, c, 1.0
    v = torch.randn(B, H, T, D, generator=gen)   # distinct per key and per dim: a wrong accumulator register shows
    return q.to(DEV), k.to(DEV), v.to(DEV)


def _pack(q, k, v):
    """[B, H, L, D] x 3 -> the in_proj layout [B, L, 3 * H * D]"""
    f = lambda t: t.transpose(1, 2).reshape(t.shape[0], t.shape[2], -1)
    return torch.cat([f(q), f(k), f(v)], -1).contiguous()


def _identity_rope(rows, D):
    return torch.ones(rows, D, device=DEV), torch.zeros(rows, D, device=DEV)


def _rot(t):
    h = t.shape[-1] // 2
    return torch.cat([-t[..., h:], t[..., :h]], -1)


def _wide(L, D, seed):
    """randn q x 8 against unit k under real RoPE tables (scores of about +-40): the fp32 inputs, the tables, and the fp64
    operands after RoPE and scale with the magnitude bound A >= sum_d |q_d k_d| of their fp32 evaluation"""
    from unified_audio_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    q, k, v = [torch.randn(B, H, L, D, generator=gen).to(DEV) for _ in range(3)]
    q = q * 8.0
    cos, sin = ops.rope_tables(L, D, DEV)
    c, s = cos.double(), sin.double()
    rope = lambda t: t.double() * c + _rot(t.double()) * s
    mag = lambda t: t.double().abs() + _rot(t.double()).abs()
    A = (mag(q) * _scale(D)) @ mag(k).transpose(2, 3)
    return q, k, v, cos, sin, rope(q) * _scale(D), rope(k).double(), A


# ---------------------------------------------------------------------------------------------- reference, bound, premise
def _moves(S, mask):
    """fa5_kernel's update rule replayed on fp64 scores [.., Lq, T] (nats): how often each row's reference maximum moves"""
    Sm = S.masked_fill(~mask, float("-inf")) * LOG2E
    moves = torch.zeros(S.shape[:-1], dtype=torch.int64, device=S.device)
    m = Sm[..., :F5_BK].amax(-1)
    for t0 in range(F5_BK, S.shape[-1], F5_BK):
        mx = Sm[..., t0:t0 + F5_BK].amax(-1)
        mv = mx > m + F5_RESCALE_LOG2
        m = torch.where(mv, mx, m)
        moves += mv
    return moves


def _reference(qs, k, v, mask, kind, bias=None, A=None, ds=2.0 ** -22, hi_only=False):
    """fp64 softmax(S) V over the visible keys for operands qs (scaled q), k, v [B, H, *, D], with the per-element bound.

    A score error d_ij changes weight p_ij by the factor e^d, so the output moves by at most sum_j p_ij |d_ij| |v_j - out_i|
    <= 2 max_j |v_j| sum_j p_ij |d_ij|.  d_ij = ds * (sum_d |q_d k_d| + |bias| + 8 + (max_i - S_ij)): the fp32 accumulation of the
    score (2^-22 covers the 3-term split's dropped lo.lo as well), and the rounding of the exponent's argument, whose magnitude
    is the distance to the reference maximum (at most 2^8 below the row maximum in fa5_kernel), with ex2.approx / expf's 2 ulp.
    On top: fp32 kernels 1e-6 of the largest value and 2^-23 |v| for the T-term fp32 sums; tensor-core kernels the fp32
    accumulation of P.V in T/16 steps per plane product; split kernels 2^-22 each for P, V and the output as fp16 hi + lo;
    single-pass kernels 2^-11 on each weight P (operands and V are handed over already rounded) and 2^-11 on an output that has
    no lo plane.  A lo plane is fp16 too: below 2^-14 it is subnormal and rounds to 2^-25 absolute, once for the output's and
    once for V's (a single key returns v itself: measured 7e-8 absolute on elements of 1e-2)."""
    qd, kd, vd = qs.double(), k.double(), v.double()
    S = qd @ kd.transpose(2, 3)
    A = (qd.abs() @ kd.abs().transpose(2, 3)) if A is None else A
    if bias is not None:
        S, A = S + bias, A + bias.abs()
    Sm = S.masked_fill(~mask, float("-inf"))
    P = torch.softmax(Sm, -1)
    ref = P @ vd
    dist = torch.where(mask, Sm.amax(-1, keepdim=True) - Sm, torch.zeros_like(S))
    d = (P * ds * (A + F5_RESCALE_LOG2 + dist)).sum(-1, keepdim=True)          # [B, H, Lq, 1]
    vmax = vd.abs().amax(2, keepdim=True)                                        # [B, H, 1, D]
    T = k.shape[2]
    if kind == "f32":
        eps = 1e-6 * ref.abs().max() + 2.0 ** -23 * vmax + 2.0 ** -25
    elif kind == "split":
        eps = (2.0 ** -20 + 2.0 ** -24 * (3 * T // 16 + 16)) * vmax + 2.0 ** -24
    else:
        eps = (2.0 ** -10 + 2.0 ** -24 * (T // 16 + 16)) * vmax + (2.0 ** -11 if hi_only else 2.0 ** -22) * ref.abs()
    rows = lambda t: t.transpose(1, 2).reshape(t.shape[0] * t.shape[2], -1)
    return rows(ref), rows(eps + 2.0 * d * vmax + 1e-30), S


def _report(tag, pattern, got, ref, bound, S, mask, T):
    """print span / moves / error over bound; assert finiteness, the bound, and the premise of a planted self-attention case
    (pattern None: the fa5 rule is only reported)"""
    assert bool(torch.isfinite(got).all()), f"{tag}: non-finite output"
    vis = S[..., mask]
    mv = _moves(S, mask)
    first = (torch.arange(mv.shape[-1], device=mv.device) % 16) < 8               # rows ra of a fragment; the others are ra + 8
    n_a, n_b = int(mv[..., first].sum()), int(mv[..., ~first].sum())
    err = (got - ref).abs()
    ratio = float((err / bound).max())
    print(f"{tag}: scores [{float(vis.min()):.1f}, {float(vis.max()):.1f}] nats, reference maximum moves {n_a} (rows r) + {n_b} "
          f"(rows r + 8), error {float(err.max() / ref.abs().max()):.2e} of the largest value, {ratio:.3f} of the bound")
    sees = mask[:, F5_BK:].any(-1) if T > F5_BK else torch.zeros_like(first)      # rows with a visible key past tile 0
    if pattern in ("half_a", "half_b"):
        ramp, flat = (n_a, n_b) if pattern == "half_a" else (n_b, n_a)
        if bool((sees & (first if pattern == "half_a" else ~first)).any()):
            assert ramp > 0 and flat == 0, f"{tag}: the two halves of a fragment must differ ({n_a} / {n_b})"
    elif pattern in MOVES and bool(sees.any()):
        assert n_a + n_b > 0, f"{tag}: the case no longer moves the reference maximum"
        if pattern == "over":
            assert int(mv.max()) == 1, f"{tag}: one move, at the first tile past the threshold"
    elif pattern in STAYS:
        assert n_a + n_b == 0, f"{tag}: the case claims a reference maximum that stays ({n_a} + {n_b} moves)"
    assert ratio <= 1.0, f"{tag}: error beyond the bound ({ratio:.2f} x)"


def _out_buf(rows, cols):
    """hi / lo planes with one spare sentinel row each"""
    return torch.full((2, rows + 1, cols), SENT, dtype=torch.float16, device=DEV)


def _planes(buf, rows, lo=True):
    from unified_audio_b200 import ops
    return ops.Planes(buf[0, :rows], buf[1, :rows] if lo else None)


def _collect(tag, buf, rows, lo=True):
    torch.cuda.synchronize()
    assert bool((buf[:, rows] == SENT).all()), f"{tag}: output written past row B * L"
    if not lo:
        assert bool((buf[1] == SENT).all()), f"{tag}: lo plane written in single-pass mode"
        return buf[0, :rows].double()
    return buf[0, :rows].double() + buf[1, :rows].double()


def _mask(Lq, T, causal, row0=0):
    m = torch.ones(Lq, T, dtype=torch.bool, device=DEV)
    return m.tril(diagonal=row0) if causal else m


def _fp16(t):
    return t.half().float()


def _self_attention_cases(pattern, D, kind, causal, run, tag):
    """all LENGTHS of one pattern through run(qkv, L, cos, sin) -> (summed output planes, hi_only)"""
    scale = _scale(D)
    for L in LENGTHS:
        mask = _mask(L, L, causal)
        if pattern == "wide":
            q, k_in, v, cos, sin, qs, kk, A = _wide(L, D, 100 + L)
            ref_args = dict(A=A, ds=2.0 ** -20)      # RoPE's three fp32 roundings on each operand on top of the split's
        else:
            qt, kk, v = _plant(pattern, L, L, D, 100 + L)
            q, k_in = qt / scale, kk
            cos, sin = _identity_rope(L, D)
            qs = q * scale                           # the one fp32 multiply of the prep kernels
            ref_args = {}
        got, hi_only = run(_pack(q, k_in, v), L, cos, sin)
        if kind == "single":
            qs, kk, v = _fp16(qs), _fp16(kk), _fp16(v)
        ref, bound, S = _reference(qs, kk, v, mask, kind, hi_only=hi_only, **ref_args)
        _report(f"{tag} {pattern} L={L}", pattern, got, ref, bound, S, mask, L)


# ---------------------------------------------------------------------------------------------- wgmma attention
# the masked-keys case is a causal one; scores of +-40 from unrounded operands are for the split kernels only
UMMA_CASES = [(D, split, causal, pattern) for D in (64, 128) for split in (True, False) for causal in (False, True)
              for pattern in PLANTED + ["causal", "wide"] if (causal or pattern != "causal") and (split or pattern != "wide")]


@pytest.mark.parametrize("D,split,causal,pattern", UMMA_CASES)
def test_attention_umma_range(lib, D, split, causal, pattern):
    """fa5_kernel<64 / 128, split / single>, causal and not: the reference maximum moving at every tile, in one half of a fragment
    only, at a late spike and just past the threshold; staying just under it and under a sink; masked keys above visible ones"""
    from unified_audio_b200 import ops

    def run(qkv, L, cos, sin):
        ws = torch.zeros(ops.attention_umma_workspace_bytes(B, L, H, D, split), dtype=torch.uint8, device=DEV)
        buf = _out_buf(B * L, H * D)
        ops.attention_umma(qkv, B, L, H, D, cos, sin, _planes(buf, B * L, split), ws, split=split, causal=causal)
        return _collect("attention_umma", buf, B * L, split), not split

    _self_attention_cases(pattern, D, "split" if split else "single", causal, run,
                          f"attention_umma D={D} {'split' if split else 'single'}{' causal' if causal else ''}")


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("L", [37, 131, 257])
def test_attention_umma_dirty_workspace(lib, D, split, L):
    """The workspace is a reused arena in the engine: 0xFF bytes (fp16 NaN) wherever the prep launch does not write, among them the
    V^T pad columns [L, Lp).  Same bits as with a zeroed workspace, and nothing written past the advertised size"""
    from unified_audio_b200 import ops
    qt, k, v = _plant("ramp_noise", L, L, D, 7 + L)
    qkv = _pack(qt / _scale(D), k, v)
    cos, sin = ops.rope_tables(L, D, DEV)
    n = ops.attention_umma_workspace_bytes(B, L, H, D, split)
    outs = []
    for fill in (0xFF, 0):
        for causal in (False, True):
            ws = torch.full((n + 256,), fill, dtype=torch.uint8, device=DEV)
            buf = _out_buf(B * L, H * D)
            ops.attention_umma(qkv, B, L, H, D, cos, sin, _planes(buf, B * L, split), ws[:n], split=split, causal=causal)
            got = _collect("attention_umma", buf, B * L, split)
            assert bool(torch.isfinite(got).all()), f"fill {fill:#x} causal {causal}: non-finite output"
            assert bool((ws[n:] == fill).all()), "workspace written past qb_attention_umma_workspace_bytes"
            outs.append(buf.clone())
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3]), "the output depends on stale workspace bytes"


# ---------------------------------------------------------------------------------------------- fp32 SIMT attention
@pytest.mark.parametrize("pattern", PLANTED + ["wide"])
@pytest.mark.parametrize("D", [64, 96, 128])
def test_attention_hd_range(lib, D, pattern):
    """attention_kernel<64, 32>, <96, 16> (the H-Codec-1.0 head) and <128, 16, 2> (two lanes per row) on the same cases"""
    from unified_audio_b200 import ops

    def run(qkv, L, cos, sin):
        buf = _out_buf(B * L, H * D)
        ops.attention_hd(qkv, B, L, H, D, cos, sin, _planes(buf, B * L))
        return _collect("attention_hd", buf, B * L), False

    _self_attention_cases(pattern, D, "f32", False, run, f"attention_hd D={D}")


@pytest.mark.parametrize("pattern", ["ramp", "spike"])
def test_attention_relbias_range(lib, pattern):
    """The WavLM gated relative bias carrying the spread (gate * table of +-40), q.k only noise: a bias rising with the offset,
    and +-40 planted on a few offsets"""
    from unified_audio_b200 import ops
    D = 64
    for L in LENGTHS:
        gen = torch.Generator().manual_seed(300 + L)
        q, k, v = [torch.randn(B, H, L, D, generator=gen).to(DEV) for _ in range(3)]
        off = torch.arange(-(L - 1), L).float()                                  # table column o holds offset j - i = o - (L - 1)
        if pattern == "ramp":
            rel = torch.stack([0.125 * (h + 1) * off for h in range(H)])
        else:
            rel = torch.randn(H, 2 * L - 1, generator=gen)
            for h in range(H):
                rel[h, off == 3 + h] = 40.0
                rel[h, off == -2 - h] = 36.0
                rel[h, off == 0] = -40.0
        rel = rel.to(DEV).contiguous()
        gate = (0.5 + 0.25 * torch.randint(0, 4, (B, H, L), generator=gen).float()).to(DEV)
        buf = _out_buf(B * L, H * D)
        ops.attention_relbias(_pack(q, k, v), B, L, H, D, rel, gate, _planes(buf, B * L))
        got = _collect("attention_relbias", buf, B * L)
        i = torch.arange(L, device=DEV)
        bias = gate.double()[..., None] * rel.double()[:, (i[None, :] - i[:, None]) + L - 1][None]
        mask = _mask(L, L, False)
        ref, bound, S = _reference(q * 0.125, k, v, mask, "f32", bias=bias)
        _report(f"attention_relbias {pattern} L={L}", None, got, ref, bound, S, mask, L)


# ---------------------------------------------------------------------------------------------- LM continuation prefill
@pytest.mark.parametrize("pattern", PLANTED + ["causal", "wide"])
@pytest.mark.parametrize("pos0", [0, 37, 64])
def test_lm_flash_attn_range(lib, pos0, pattern):
    """lm_qkv_prep + lm_flash_attn continuing a planted cache of pos0 keys (rows >= pos0 + L NaN): causal, masked keys scoring
    above the visible ones, rows whose visible keys end inside tile 0"""
    from unified_audio_b200 import ops
    D = 64
    for L in LENGTHS:
        T = pos0 + L
        Lmax = T + 5
        if pattern == "wide":
            qa, ka, v, cos, sin, qs, kk, A = _wide(T, D, 200 + T)
            q, qs, A = qa[:, :, pos0:], qs[:, :, pos0:], A[:, :, pos0:]
            ref_args = dict(A=A, ds=2.0 ** -20)
            k_cache = kk.float()                     # the cache rows an earlier prefill would have left: RoPE already applied
        else:
            qt, ka, v = _plant(pattern, L, T, D, 200 + T, row0=pos0)
            q = qt * 8.0
            cos, sin = _identity_rope(T, D)
            qs, kk, k_cache = q * 0.125, ka, ka
            ref_args = {}
        kc = torch.full((B, H, Lmax, D), float("nan"), device=DEV)
        vc = torch.full((B, H, Lmax, D), float("nan"), device=DEV)
        kc[:, :, :pos0], vc[:, :, :pos0] = k_cache[:, :, :pos0], v[:, :, :pos0]
        q32 = torch.empty(B, H, L, D, device=DEV)
        buf = _out_buf(B * L, H * D)
        ops.lm_qkv_prep(_pack(q, ka[:, :, pos0:], v[:, :, pos0:]), B, L, H, pos0, cos, sin, q32, kc, vc, Lmax)
        ops.lm_flash_attn(q32, kc, vc, B, L, H, pos0, Lmax, _planes(buf, B * L))
        got = _collect("lm_flash_attn", buf, B * L)
        assert bool(torch.isnan(kc[:, :, T:]).all()) and bool(torch.isnan(vc[:, :, T:]).all()), "cache rows past pos0 + L written"
        mask = _mask(L, T, True, row0=pos0)
        ref, bound, S = _reference(qs, kk, v, mask, "split", **ref_args)
        _report(f"lm_flash_attn pos0={pos0} {pattern} L={L}", pattern, got, ref, bound, S, mask, T)


# ---------------------------------------------------------------------------------------------- perceiver cross attention
XATT_MAX_KEYS = 48 * 1024 // (4 * 4)         # one fp32 score per key for each of a block's 4 warps in 48 KB of shared memory


@pytest.mark.parametrize("pattern", ["ramp", "spike", "sink", "uniform", "wide"])
@pytest.mark.parametrize("Nk", [1, 31, 32, 33, XATT_MAX_KEYS])
def test_cross_attention_range(lib, Nk, pattern):
    """cross_attention_kernel (one warp per query, 4 per block) with query counts that leave warps of the last block idle, key
    counts around the 32-lane stride of its softmax pass and at the largest its shared memory admits"""
    from unified_audio_b200 import ops
    D = 64
    for Nq in (1, 6, 9):
        if pattern == "wide":
            gen = torch.Generator().manual_seed(Nk + Nq)
            q = (torch.randn(B, H, Nq, D, generator=gen) * 8.0).to(DEV)
            k, v = [torch.randn(B, H, Nk, D, generator=gen).to(DEV) for _ in range(2)]
        else:
            qt, k, v = _plant(pattern, Nq, Nk, D, Nk + Nq)
            q = qt * 8.0
        f = lambda t: t.transpose(1, 2).reshape(B, t.shape[2], H * D)
        kv = torch.cat([f(k), f(v)], -1).contiguous()                            # [B, Nk, 2 * H * D]: keys, then values
        buf = _out_buf(B * Nq, H * D)
        ops.cross_attention(f(q).contiguous(), kv, B, Nq, Nk, H, _planes(buf, B * Nq))
        got = _collect("cross_attention", buf, B * Nq)
        mask = _mask(Nq, Nk, False)
        ref, bound, S = _reference(q * 0.125, k, v, mask, "f32")
        _report(f"cross_attention {pattern} Nq={Nq} Nk={Nk}", None, got, ref, bound, S, mask, Nk)


def test_cross_attention_too_many_keys(lib):
    """one key more than the shared memory holds is refused before any launch"""
    from unified_audio_b200 import ops
    Nk, Nq, D = XATT_MAX_KEYS + 1, 3, 64
    q = torch.zeros(B, Nq, H * D, device=DEV)
    kv = torch.zeros(B, Nk, 2 * H * D, device=DEV)
    buf = _out_buf(B * Nq, H * D)
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match="cross_attention"):
        ops.cross_attention(q, kv, B, Nq, Nk, H, _planes(buf, B * Nq))
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 and bool((buf == SENT).all()), "a kernel ran"
