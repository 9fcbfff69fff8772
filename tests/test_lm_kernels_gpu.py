"""The UniSE LM kernels of csrc/llm.cu against plain fp64 torch on the same device, through their public launchers: the weight
packer, the fused decode projections (lm_skinny QKV / RESID / GATEUP / HEAD at all three K tilings), the decode attention at both
keys-in-flight settings, the continuation prefill (lm_qkv_prep + lm_flash_attn), and the greedy and sampled heads.  The operands
are the ones the kernels read (the fp32 weights that were packed, RMSNorm weight folded in as LLM_SFT._prepare does).  Output
buffers start as sentinels and cache rows the kernel must not touch as NaN or random bits; each test checks that nothing outside
the intended window changed."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = -1234.5                   # exact in fp32, produced by none of these kernels
F32_TOL = 1e-6                   # fp32 kernels, relative to the largest reference value
SPLIT_TOL = 2e-5                 # 3-term fp16 split attention (as attention_umma split)
# lm_skinny: x and W are each split into fp16 hi + lo (~2^-22 relative each) and the lo*lo product is dropped (~2^-22):
# per element about 2^-20 * (|W|.|x|) * rsqrt(mean x^2 + eps), plus one fp32 rounding per mma / cross-warp add
SKINNY = 2.0 ** -20
SHAPES = [(128, 2, 512), (256, 4, 1024), (512, 8, 2048)]     # down projection K = 512 / 1024 / 2048: <4,8>, <4,16>, <8,16>


def _rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _rot(t):
    return torch.cat([-t[..., 32:], t[..., :32]], -1)


def _check(name, got, ref, bound):
    got = got.double()
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite output"
    err = (got - ref).abs()
    ratio = float((err / bound).max())
    print(f"{name}: error {float(err.max() / ref.abs().max()):.2e} of the largest value, {ratio:.3f} of the bound")
    assert ratio <= 1.0, f"{name}: error beyond the bound ({ratio:.2f} x)"


def _skinny_ref(x, w, norm):
    """fp64 x . W^T (RMSNorm'd rows when `norm`) and its per-element bound"""
    xd, wd = x.double(), w.double()
    r = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6) if norm else torch.ones_like(xd[:, :1])
    val = (xd @ wd.T) * r
    S = (xd.abs() @ wd.abs().T) * r
    K = x.shape[1]
    return val, SKINNY * S + 2.0 ** -24 * (3 * K // 16 + 16) * val.abs() + 1e-30


def _attn_ref(q, K, V, n=None):
    """fp64 softmax(q K^T) V for q [B, h, 64], K / V [B, h, T, 64], and the bound of an fp32 kernel: 1e-6 of the largest value,
    plus the fp32 rounding of each 64-term score (2^-22 of sum |q_d k_d|) carried through the softmax weights onto V.
    n (int [B]): row b attends to its keys 0 .. n[b] - 1 only (the rest may hold anything); default all T"""
    q, K, V = q.double(), K.double(), V.double()
    if n is not None:
        keep = (torch.arange(K.shape[2], device=K.device)[None] < n.to(K.device)[:, None])[:, None, :, None]
        K, V = K.masked_fill(~keep, 0.0), V.masked_fill(~keep, 0.0)
    sc = torch.einsum("bhd,bhtd->bht", q, K)
    if n is not None:
        sc = sc.masked_fill(~keep[..., 0], float("-inf"))
    ref = torch.einsum("bht,bhtd->bhd", torch.softmax(sc, -1), V)
    ds = 2.0 ** -22 * torch.einsum("bhd,bhtd->bht", q.abs(), K.abs()).amax(-1)
    bound = F32_TOL * ref.abs().max() + 2.0 * ds[..., None] * V.abs().amax(2) + 1e-30
    return ref, bound, sc


def _rope_ref(t, bt, c, s):
    """rotate-half RoPE of t [..., 64] at one position (c, s [64]) and the propagated bound (+ the kernel's own fp32 rounding)"""
    y = t * c + _rot(t) * s
    swap = lambda u: torch.cat([u[..., 32:], u[..., :32]], -1)
    return y, c.abs() * bt + s.abs() * swap(bt) + 2.0 ** -23 * ((t * c).abs() + (_rot(t) * s).abs())


def _layer(hidden, inter, seed, q_gain=1.0):
    """seeded decoder-layer weights: the fp32 operands the decode kernels read, and their packed planes"""
    from unified_audio_b200 import ops
    H = hidden
    wqkv = _rnd((3 * H, H), seed, 2.0 / H ** 0.5)
    wqkv[:H] *= q_gain
    in_w, post_w = 1.0 + 0.1 * _rnd((H,), seed + 5), 1.0 + 0.1 * _rnd((H,), seed + 6)
    f = dict(wqkv=wqkv * in_w[None, :], wo=_rnd((H, H), seed + 1, 2.0 / H ** 0.5),
             wg=_rnd((inter, H), seed + 2, 2.0 / H ** 0.5) * post_w[None, :],
             wu=_rnd((inter, H), seed + 3, 2.0 / H ** 0.5) * post_w[None, :], wd=_rnd((H, inter), seed + 4, 2.0 / inter ** 0.5))
    packed = {k + "_p": ops.lm_pack_weight(v) for k, v in f.items()}
    return f, packed


# ---------------------------------------------------------------------------------------------- weight packing
def test_lm_pack_weight(lib):
    """{hi[4], lo[4]} per 4 consecutive k of a row, hi = fp16(w), lo = fp16(w - hi), bit for bit; values whose hi overflows to
    inf, whose lo underflows to zero or a subnormal, and subnormal weights included"""
    from unified_audio_b200 import _lib, ops
    n, k = 37, 96
    w = _rnd((n, k), 1, 3.0)
    w[0, :12] = torch.tensor([70000.0, -70000.0, 65504.0, 65519.0, 65520.0, 1.0 + 2.0 ** -30, -(1.0 + 2.0 ** -22), 3e-8,
                              -5.9e-8, 1e-5, 2.0 ** -25, 6.1e-5 + 1e-12])
    w[1] *= 1e-6
    w[2] *= 1e4
    out = torch.full((n + 1, 2 * k), -77.0, dtype=torch.float16, device=DEV)    # one spare row: must stay untouched
    _lib.check(_lib.load().qb_lm_pack_weight(ops._p(w), n, k, ops._p(out), ops._stream()))
    torch.cuda.synchronize()
    hi = w.half()
    lo = (w - hi.float()).half()
    g = out[:n].view(n, k // 4, 2, 4)
    assert torch.equal(g[:, :, 0].reshape(n, k).view(torch.int16), hi.view(torch.int16)), "hi plane"
    assert torch.equal(g[:, :, 1].reshape(n, k).view(torch.int16), lo.view(torch.int16)), "lo plane"
    assert bool((out[n] == -77.0).all()), "written past the packed rows"
    assert torch.equal(ops.lm_pack_weight(w), out[:n])


# ---------------------------------------------------------------------------------------------- one decode layer
@pytest.mark.parametrize("hidden,heads,inter", SHAPES)
@pytest.mark.parametrize("B", [1, 5, 8, 9, 31, 32])
def test_lm_decode_layer(lib, hidden, heads, inter, B):
    """One lm_decode_layer_tc (QKV + RoPE + cache append, decode attention, o_proj + residual, gate/up + SwiGLU, down + residual)
    against an fp64 HF Llama decoder layer, stage by stage from the kernel's own inputs to that stage; every row at one position,
    then the rows at different positions (prefixes of different lengths), each row against its own position's reference"""
    from unified_audio_b200 import ops
    H = hidden
    f, Lw = _layer(H, inter, 10 * hidden + B)
    Lmax = 48
    cos, sin = ops.rope_tables(Lmax + 16, 64, DEV)                # the table is longer than the cache
    cases = [[pos] * B for pos in (0, 37, Lmax - 1)] + [[(17 * b + Lmax - 1) % Lmax for b in range(B)]]
    for pos in cases:
        seed = 1000 * B + pos[0]
        x_all = torch.full((33, H), SENT, device=DEV)
        x_all[:B] = _rnd((B, H), seed, 1.5) + 0.2
        kc, vc = _rnd((B, heads, Lmax, 64), seed + 1), _rnd((B, heads, Lmax, 64), seed + 2)
        for b, p in enumerate(pos):                              # row p is the kernel's to write, rows above are never read
            kc[b, :, p:] = float("nan")
            vc[b, :, p:] = float("nan")
        kc0, vc0 = _bits(kc).clone(), _bits(vc).clone()
        q_all, a_all = torch.full((33, H), SENT, device=DEV), torch.full((33, H), SENT, device=DEV)
        m_all = torch.full((33, inter), SENT, device=DEV)
        pos_t = torch.tensor(pos, dtype=torch.int32, device=DEV)
        x0 = x_all[:B].clone()
        ops.lm_decode_layer_tc(x_all[:B], B, H, heads, inter, Lw, kc, vc, Lmax, pos_t, cos, sin, q_all[:B], a_all[:B], m_all[:B])
        torch.cuda.synchronize()
        tag = f"decode layer {H}/{heads}/{inter} B={B} pos={pos[0] if len(set(pos)) == 1 else 'per row'}"
        for nm, buf in (("x", x_all), ("q_buf", q_all), ("attn_buf", a_all), ("mlp_buf", m_all)):
            assert bool((buf[B:] == SENT).all()), f"{tag}: {nm} written past row B"
        assert pos_t.tolist() == pos, "the layer must not move the positions"
        # QKV + RoPE at each row's position (q pre-scaled by 1/sqrt(64)), K/V appended at that row of the cache
        val, bnd = _skinny_ref(x0, f["wqkv"], True)
        sh = lambda t: t.reshape(B, 3, heads, 64)
        val, bnd = sh(val), sh(bnd)
        pl, bi = pos_t.long(), torch.arange(B, device=DEV)
        c, s = cos[pl].double()[:, None], sin[pl].double()[:, None]
        q_ref, q_bnd = _rope_ref(val[:, 0], bnd[:, 0], c, s)
        k_ref, k_bnd = _rope_ref(val[:, 1], bnd[:, 1], c, s)
        _check(f"{tag} q_buf", q_all[:B].view(B, heads, 64), q_ref * 0.125, q_bnd * 0.125)
        _check(f"{tag} k row", kc[bi, :, pl], k_ref, k_bnd)
        _check(f"{tag} v row", vc[bi, :, pl], val[:, 2], bnd[:, 2])
        rows = torch.ones(B, Lmax, dtype=torch.bool, device=DEV)
        rows[bi, pl] = False
        other = lambda t: t.transpose(1, 2)[rows]
        assert torch.equal(other(_bits(kc)), other(kc0)) and torch.equal(other(_bits(vc)), other(vc0)), \
            f"{tag}: a cache row other than the row's position changed"
        # attention of each row over its rows 0..pos[b] of the kernel's cache with the kernel's q
        a_ref, a_bnd, _ = _attn_ref(q_all[:B].view(B, heads, 64), kc, vc, pos_t + 1)
        _check(f"{tag} attn_buf", a_all[:B].view(B, heads, 64), a_ref, a_bnd)
        a_ref = a_ref.reshape(B, H)
        # o_proj + residual (not observable on its own: its bound carries into the MLP and the final x)
        o_val, o_bnd = _skinny_ref(a_all[:B], f["wo"], False)
        x_mid = x0.double() + o_val
        e_mid = o_bnd + 2.0 ** -24 * x_mid.abs()
        r = torch.rsqrt(x_mid.pow(2).mean(-1, keepdim=True) + 1e-6)
        g_val, g_bnd = _skinny_ref(x_mid, f["wg"], True)
        u_val, u_bnd = _skinny_ref(x_mid, f["wu"], True)
        g_bnd = g_bnd + r * (e_mid @ f["wg"].double().abs().T)
        u_bnd = u_bnd + r * (e_mid @ f["wu"].double().abs().T)
        m_ref = torch.nn.functional.silu(g_val) * u_val
        m_bnd = 1.1 * g_bnd * (u_val.abs() + u_bnd) + torch.nn.functional.silu(g_val).abs() * u_bnd + 2.0 ** -20 * m_ref.abs()
        _check(f"{tag} mlp_buf", m_all[:B], m_ref, m_bnd)
        d_val, d_bnd = _skinny_ref(m_all[:B], f["wd"], False)
        x_ref = x_mid + d_val
        _check(f"{tag} x", x_all[:B], x_ref, e_mid + d_bnd + 2.0 ** -24 * x_ref.abs())


# ---------------------------------------------------------------------------------------------- decode attention
@pytest.mark.parametrize("unroll", [4, 8])
@pytest.mark.parametrize("n", [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 300])
def test_lm_decode_attention(lib, unroll, n):
    """lm_decode_attn2 at 4 and 8 keys in flight per lane (16U - 1, 16U, 16U + 1 keys end a trip early, exactly, late), scores
    spanning about +-60 (the online-softmax rescale), cache rows >= n NaN: finite, within 1e-6 of fp64 softmax(q K^T) V"""
    from unified_audio_b200 import ops
    Lmax, pos = 300, n - 1
    cos, sin = ops.rope_tables(Lmax + 4, 64, DEV)
    try:
        ops.lm_set_att_unroll(unroll)
        for B, heads in ((32, 1), (5, 8), (3, 3)):
            H = 64 * heads
            f, Lw = _layer(H, 64, 7 * heads + B, q_gain=10.0)      # |q| ~ 20, |k| ~ 1: scores of +-60
            x = _rnd((B, H), n + B)
            kc, vc = _rnd((B, heads, Lmax, 64), n + 1), _rnd((B, heads, Lmax, 64), n + 2)
            kc[:, :, n:] = float("nan")
            vc[:, :, n:] = float("nan")
            qb, ab, mb = torch.empty(B, H, device=DEV), torch.full((B, H), SENT, device=DEV), torch.empty(B, 64, device=DEV)
            ops.lm_decode_layer_tc(x, B, H, heads, 64, Lw, kc, vc, Lmax, torch.full((B,), pos, dtype=torch.int32, device=DEV),
                                   cos, sin, qb, ab, mb)
            torch.cuda.synchronize()
            ref, bound, sc = _attn_ref(qb.view(B, heads, 64), kc[:, :, :n], vc[:, :, :n])
            print(f"U={unroll} n={n} B={B} heads={heads}: scores span [{float(sc.min()):.1f}, {float(sc.max()):.1f}]")
            _check(f"decode attention U={unroll} n={n} B={B} heads={heads}", ab.view(B, heads, 64), ref, bound)
    finally:
        ops.lm_set_att_unroll(8)                                 # LM_ATT_U_DEFAULT (csrc/common.cuh)


# ---------------------------------------------------------------------------------------------- continuation prefill
@pytest.mark.parametrize("pos0,L,B,heads", [(0, 1, 1, 1), (0, 65, 2, 8), (37, 30, 3, 3), (64, 64, 1, 8), (100, 129, 2, 2),
                                            (5, 200, 3, 5)])
def test_lm_prefill_continuation(lib, pos0, L, B, heads):
    """lm_qkv_prep + lm_flash_attn continuing a cache filled up to pos0: q32 (RoPE at absolute positions, x 1/8), K/V rows
    [pos0, pos0 + L) and nothing else written, and the output planes against fp64 causal attention over keys 0 .. pos0 + t"""
    from unified_audio_b200 import ops
    H = heads * 64
    Lmax = pos0 + L + 7
    cos, sin = ops.rope_tables(Lmax + 16, 64, DEV)
    qkv = _rnd((B, L, 3 * H), 31 + L + pos0)
    kc, vc = _rnd((B, heads, Lmax, 64), 41 + pos0), _rnd((B, heads, Lmax, 64), 42 + pos0)
    kc[:, :, pos0:] = float("nan")
    vc[:, :, pos0:] = float("nan")
    kc0, vc0 = _bits(kc).clone(), _bits(vc).clone()
    nq = B * heads * L * 64
    q_all = torch.full((nq + 64,), SENT, device=DEV)
    q32 = q_all[:nq].view(B, heads, L, 64)
    out_buf = torch.full((2, B * L + 1, H), -1234.0, dtype=torch.float16, device=DEV)
    out = ops.Planes(out_buf[0, :B * L], out_buf[1, :B * L])
    ops.lm_qkv_prep(qkv, B, L, heads, pos0, cos, sin, q32, kc, vc, Lmax)
    ops.lm_flash_attn(q32, kc, vc, B, L, heads, pos0, Lmax, out)
    torch.cuda.synchronize()
    tag = f"continuation pos0={pos0} L={L} B={B} heads={heads}"
    assert bool((q_all[nq:] == SENT).all()), f"{tag}: q32 written past its end"
    assert bool((out_buf[:, B * L] == -1234.0).all()), f"{tag}: output planes written past row B*L"
    x = qkv.double().view(B, L, 3, heads, 64).permute(2, 0, 3, 1, 4)        # [3, B, heads, L, 64]
    c, s = cos[pos0:pos0 + L].double(), sin[pos0:pos0 + L].double()
    rnd = lambda t: 2.0 ** -22 * ((t * c).abs() + (_rot(t) * s).abs()) + 1e-30
    _check(f"{tag} q32", q32, (x[0] * c + _rot(x[0]) * s) * 0.125, rnd(x[0]) * 0.125)
    _check(f"{tag} k rows", kc[:, :, pos0:pos0 + L], x[1] * c + _rot(x[1]) * s, rnd(x[1]))
    assert torch.equal(vc[:, :, pos0:pos0 + L], qkv.view(B, L, 3, heads, 64)[:, :, 2].transpose(1, 2)), f"{tag}: v rows"
    rows = torch.ones(Lmax, dtype=torch.bool, device=DEV)
    rows[pos0:pos0 + L] = False
    assert torch.equal(_bits(kc)[:, :, rows], kc0[:, :, rows]) and torch.equal(_bits(vc)[:, :, rows], vc0[:, :, rows]), \
        f"{tag}: a cache row outside [pos0, pos0 + L) changed"
    T = pos0 + L
    K, V = kc[:, :, :T].double(), vc[:, :, :T].double()
    sc = q32.double() @ K.transpose(2, 3)
    mask = torch.ones(L, T, dtype=torch.bool, device=DEV).tril(diagonal=pos0)
    ref = (torch.softmax(sc.masked_fill(~mask, float("-inf")), -1) @ V).transpose(1, 2).reshape(B * L, H)
    got = out.hi.double() + out.lo.double()
    _check(f"{tag} output", got, ref, SPLIT_TOL * ref.abs().max() + 1e-30)
    if pos0 == 0:
        ws = torch.zeros(ops.attention_umma_workspace_bytes(B, L, heads, 64, True), dtype=torch.uint8, device=DEV)
        um = ops.Planes.zeros((B * L, H), True, DEV)
        ops.attention_umma(qkv, B, L, heads, 64, cos, sin, um, ws, split=True, causal=True)
        torch.cuda.synchronize()
        _check(f"{tag} attention_umma causal", um.hi.double() + um.lo.double(), ref, SPLIT_TOL * ref.abs().max() + 1e-30)


# ---------------------------------------------------------------------------------------------- heads
HK = 128          # hidden of the head tests


def _planted_head(V, pad_rows, vals):
    """packed head weight over V + pad_rows rows (rows >= V lie past the vocabulary but inside the allocation) whose row j
    has vals[j, d] in input column d: with x = e_d every logit is vals[:, d] times one common RMSNorm factor, exactly"""
    from unified_audio_b200 import ops
    w = torch.zeros(V + pad_rows, HK, device=DEV)
    w[:, :vals.shape[1]] = vals
    return ops.lm_pack_weight(w)


def _onehot_x(B, ds):
    """x_b = e_{ds[b]} + sqrt(HK - 1) e_{HK-1}: mean x^2 = 1, so the RMSNorm factor is ~1, and column HK - 1 of W is zero"""
    x = torch.zeros(B, HK, device=DEV)
    x[torch.arange(B), torch.tensor(ds)] = 1.0
    x[:, HK - 1] = (HK - 1) ** 0.5
    return x


@pytest.mark.parametrize("width", [16, 40, 4096, 4100])
def test_lm_head_argmax(lib, width):
    """Greedy head: the arg-max of the range over planted exact logits.  The row maximum just outside the range (lo - 1 and
    hi .. hi + 15, also past the end of the vocabulary) never wins; ties inside a CTA's two 8-column halves, across lanes and
    across CTAs resolve to the lowest id as torch.argmax does; x_next is emb[token] bit for bit; several back-to-back steps
    advance every row's position and slot once each and fill out_ids column by column"""
    from unified_audio_b200 import ops
    gs = ss = width
    V = 3 + gs + ss
    max_cols = -(-width // 16) * 16
    g = torch.Generator().manual_seed(width)
    pat = []                                    # in-range columns planted with the maximum, one pattern per batch row
    for cols in ([width // 2], [19, 27], [17, 21], [16 * 5 + 9, 16 * 2 + 12], [width - 1, 6], [3, 11, 8 + 3], list(range(width)),
                 [width - 1]):
        cols = sorted({c for c in cols if c < width})
        pat.append(cols or [width - 1])
    B, D = len(pat), len(pat)
    emb = torch.randn(V + 16, HK, generator=g).to(DEV)          # rows past V: what a token past the vocabulary would gather
    for lo in (3, 3 + gs):
        hi = lo + width
        vals = torch.randint(-20, 20, (V + 16, D), generator=g).float().to(DEV)
        vals[lo - 1] = 100.0
        vals[hi:hi + 16] = 100.0
        for d, cols in enumerate(pat):
            vals[lo + torch.tensor(cols), d] = 50.0
        wp = _planted_head(V, 16, vals)
        x = _onehot_x(B, list(range(B)))
        rng = torch.tensor([lo, hi], dtype=torch.int32, device=DEV)
        steps = 4
        out_ids = torch.full((B, steps + 2), -7, dtype=torch.int64, device=DEV)
        x_next = torch.full((B + 1, HK), SENT, device=DEV)
        pos_all = torch.arange(B + 1, dtype=torch.int32, device=DEV) + 5       # one position per row, and a sentinel after them
        pos = pos_all[:B]
        slot = torch.zeros(2, dtype=torch.int32, device=DEV)
        pv = torch.zeros(max_cols // 16 + 1, 32, device=DEV)
        pi = torch.zeros(max_cols // 16 + 1, 32, dtype=torch.int32, device=DEV)
        for _ in range(steps):                                     # no sync between steps
            ops.lm_head_argmax_tc(x, B, HK, wp, rng, max_cols, emb, x_next[:B], out_ids, steps + 2, pos, slot, pv, pi)
        torch.cuda.synchronize()
        want = lo + vals[lo:hi, :B].argmax(0)
        want_cols = torch.tensor([c[0] for c in pat], device=DEV) + lo
        assert torch.equal(want, want_cols)                        # the planted ties: torch.argmax takes the first
        got = out_ids[:, :steps]
        bad = (got != want[:, None]).any(1).nonzero().flatten().tolist()
        assert not bad, (f"width {width} lo {lo}: rows {bad} picked {got[bad, 0].tolist()} instead of {want[bad].tolist()} "
                         f"(range [{lo}, {hi}))")
        assert bool((out_ids[:, steps:] == -7).all()), "out_ids written past the steps taken"
        assert torch.equal(x_next[:B], emb[want]), "x_next must be emb[token]"
        assert bool((x_next[B] == SENT).all())
        want_pos = torch.arange(B + 1, dtype=torch.int32) + 5 + torch.tensor([steps] * B + [0], dtype=torch.int32)
        assert torch.equal(pos_all.cpu(), want_pos) and slot.tolist() == [steps, 0], f"pos {pos_all.tolist()} slot {slot.tolist()}"


@pytest.mark.parametrize("B", [1, 9, 32])
def test_lm_head_logits(lib, B):
    """lm_skinny<HEAD> at the shipped head (hidden 512, vocabulary 12291, final RMSNorm weight folded in): the logits the sampled
    head writes for the global range (4096 of max_cols 8192) and the semantic range (8192, ending at the vocabulary) against
    fp64 within the skinny bound; columns past the range untouched"""
    from unified_audio_b200 import ops
    Hd, V, max_cols = 512, 12291, 8192
    w = _rnd((V, Hd), 70, 2.0 / Hd ** 0.5) * (1.0 + 0.1 * _rnd((Hd,), 71))[None, :]
    wp = ops.lm_pack_weight(w)
    x = _rnd((B, Hd), 72 + B, 1.3) + 0.1
    emb = _rnd((V, Hd), 73)
    for lo, hi in ((3, 4099), (4099, V)):
        logits = torch.full((B, max_cols), SENT, device=DEV)
        seed = torch.tensor([1, 2, 0, 0], dtype=torch.int32, device=DEV)
        ops.lm_head_sample_tc(x, B, Hd, wp, torch.tensor([lo, hi], dtype=torch.int32, device=DEV), max_cols, emb,
                              torch.empty(B, Hd, device=DEV), torch.zeros(B, 1, dtype=torch.int64, device=DEV), 1,
                              torch.zeros(B, dtype=torch.int32, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV),
                              torch.zeros(max_cols // 16 + 1, 32, device=DEV),
                              torch.zeros(max_cols // 16 + 1, 32, dtype=torch.int32, device=DEV), logits, 0.8, 50, 0.95, seed)
        torch.cuda.synchronize()
        val, bnd = _skinny_ref(x, w[lo:hi], True)
        _check(f"head logits B={B} [{lo}, {hi})", logits[:, :hi - lo], val, bnd)
        assert bool((logits[:, hi - lo:] == SENT).all()), "logits written past the range"


def _run_sampler(lo, width, V, logits_vals, temperature, top_k, top_p, seed=987654321012345, call=3, slot0=7):
    """lm_head_sample_tc on planted exact logits: row b of the range is logits_vals[:, b]"""
    from unified_audio_b200 import ops
    B = logits_vals.shape[1]
    max_cols = -(-width // 16) * 16
    vals = torch.zeros(V + 16, B, device=DEV)
    vals[lo:lo + width] = logits_vals
    vals[lo + width:lo + width + 16] = 1e4                        # just past the range (past the vocabulary for the last one)
    vals[lo - 1] = 1e4
    wp = _planted_head(V, 16, vals)
    x = _onehot_x(B, list(range(B)))
    rng = torch.tensor([lo, lo + width], dtype=torch.int32, device=DEV)
    emb = _rnd((V + 16, HK), 5)
    x_next = torch.empty(B, HK, device=DEV)
    out_ids = torch.full((B, 16), -7, dtype=torch.int64, device=DEV)
    pos = torch.full((B,), 11, dtype=torch.int32, device=DEV)
    slot0_d = torch.tensor([slot0, 0], dtype=torch.int32, device=DEV)
    slot = slot0_d.clone()
    pv = torch.zeros(max_cols // 16 + 1, 32, device=DEV)
    pi = torch.zeros(max_cols // 16 + 1, 32, dtype=torch.int32, device=DEV)
    logits = torch.full((B, max_cols), SENT, device=DEV)
    dbg = torch.zeros(B, 4, device=DEV)
    to_i32 = lambda v: v - (1 << 32) if v >= (1 << 31) else v
    sd = torch.tensor([to_i32(seed & 0xFFFFFFFF), to_i32(seed >> 32), call, 0], dtype=torch.int32, device=DEV)

    def run():
        slot.copy_(slot0_d)
        ops.lm_head_sample_tc(x, B, HK, wp, rng, max_cols, emb, x_next, out_ids, 16, pos, slot, pv, pi, logits, temperature, top_k,
                              top_p, sd, dbg)

    return dict(run=run, logits=logits, dbg=dbg, out_ids=out_ids, x_next=x_next, emb=emb, slot=slot, pos=pos, seed=seed, call=call,
                slot0=slot0, lo=lo)


def _check_sampler(tag, st, width, temperature, top_k, top_p):
    """the kernel's draw against oracle.llama.sample_filter + inverse_cdf_pick on the kernel's own logits"""
    from oracle import llama
    lg = st["logits"][:, :width].cpu()
    dbg = st["dbg"].cpu()
    ids = st["out_ids"][:, st["slot0"]].cpu()
    B = lg.shape[0]
    assert bool((st["logits"][:, width:].cpu() == SENT).all()), f"{tag}: logits written past the range"
    assert torch.equal(st["out_ids"][:, :st["slot0"]].cpu(), torch.full((B, st["slot0"]), -7)), f"{tag}: out_ids column"
    assert torch.equal(st["out_ids"][:, st["slot0"] + 1:].cpu(), torch.full((B, 16 - st["slot0"] - 1), -7)), f"{tag}: out_ids column"
    n_near = 0
    for b in range(B):
        row = lg[b]
        u = llama.sample_uniform(st["seed"], st["call"], st["slot0"], b)
        assert float(dbg[b, 0]) == u, f"{tag} row {b}: uniform {float(dbg[b, 0])} vs {u}"
        kk = min(top_k, width)
        kth = torch.topk(row, kk)[0][-1]
        assert int(dbg[b, 1]) == int((row >= kth).sum()), f"{tag} row {b}: survivors {int(dbg[b, 1])} vs {int((row >= kth).sum())}"
        probs = llama.sample_filter(row[None], temperature, kk, top_p)[0]       # torch.topk needs k <= n; k = n keeps every token
        surv = torch.sort(row[row >= kth].double(), descending=True).values
        cum = torch.cumsum(torch.softmax(surv, 0), 0)
        near_p = top_p < 1.0 and float((cum - top_p).abs().min()) < 1e-6
        kept = 1 + int((cum[:-1] <= top_p).sum()) if top_p < 1.0 else len(surv)     # a token goes once the mass before it > top_p
        if not near_p:
            assert int(dbg[b, 2]) == kept, f"{tag} row {b}: top-p keeps {int(dbg[b, 2])} vs {kept}"
        want, near = llama.inverse_cdf_pick(probs, u)
        tok = int(ids[b]) - st["lo"]
        if tok != want:
            assert near < 1e-6 or near_p, f"{tag} row {b}: token {tok} vs {want} (boundary distance {near:.2e})"
            n_near += 1
        assert torch.equal(st["x_next"][b], st["emb"][int(ids[b])]), f"{tag} row {b}: x_next is not emb[token]"
    print(f"{tag}: {B - n_near}/{B} tokens equal to the oracle's pick, {n_near} on a boundary")
    return ids


def _fp16_exact(t):
    return t.half().float()


SAMPLE_CASES = {
    "defaults": (0.8, 50, 0.95),
    "greedy": (1.0, 1, 1.0),
    "wide": (0.05, 1024, 0.999),
}


@pytest.mark.parametrize("case", list(SAMPLE_CASES))
def test_lm_head_sample(lib, case):
    """Sampled head on planted exact logits: the uniform, the exact survivor count, the top-p count and the token against the
    oracle; rows with very negative entries (probability exactly 0); (1.0, 1, 1.0) is the arg-max"""
    temperature, top_k, top_p = SAMPLE_CASES[case]
    g = torch.Generator().manual_seed(len(case))
    width, gs = 4096, 4096
    V = 3 + gs + 8192
    B = 6
    vals = _fp16_exact(torch.randn(width, B, generator=g) * 3.0)
    vals[::7, 1] = -60000.0                                       # exp underflows to 0 after the max is subtracted
    vals[:, 2] = _fp16_exact(torch.randn(width, generator=g) * 0.05)  # flat row: many survivors carry mass
    vals[:, 3] = torch.randint(-4, 4, (width,), generator=g).float()  # many ties everywhere
    for lo in (3, 3 + gs):
        st = _run_sampler(lo, width, V if lo == 3 else lo + width, vals.to(DEV), temperature, top_k, top_p)
        st["run"]()
        torch.cuda.synchronize()
        ids = _check_sampler(f"sample {case} lo={lo}", st, width, temperature, top_k, top_p)
        if top_k == 1:                                             # rows whose maximum is unique: the arg-max
            lg = st["logits"][:, :width].cpu()
            uniq = (lg == lg.max(1, keepdim=True).values).sum(1) == 1
            assert int(uniq.sum()) >= 4 and torch.equal((ids - lo)[uniq], lg.argmax(1)[uniq]), "top_k = 1 must be the arg-max"


def test_lm_head_sample_small_range(lib):
    """top_k >= n (a 40-column range), and five ties straddling rank 50 of a 4096-column range: all five kept"""
    g = torch.Generator().manual_seed(3)
    vals = _fp16_exact(torch.randn(40, 3, generator=g) * 2.0)
    st = _run_sampler(3, 40, 3 + 40 + 100, vals.to(DEV), 0.8, 50, 0.95)
    st["run"]()
    torch.cuda.synchronize()
    _check_sampler("sample top_k >= n", st, 40, 0.8, 50, 0.95)
    assert st["dbg"][:, 1].tolist() == [40.0] * 3
    width = 4096
    vals = _fp16_exact(torch.randn(width, 2, generator=g))
    top = torch.randperm(width, generator=g)[:52]
    vals[top[:47], :] = torch.arange(47, dtype=torch.float32)[:, None] + 10.0
    vals[top[47:], :] = 5.0                                       # ranks 48 .. 52 tie, rank 50 among them
    st = _run_sampler(3, width, 3 + width + 8192, vals.to(DEV), 0.8, 50, 0.95)
    st["run"]()
    torch.cuda.synchronize()
    _check_sampler("sample five ties at rank 50", st, width, 0.8, 50, 0.95)
    assert st["dbg"][:, 1].tolist() == [52.0, 52.0], "every tie at the k-th value is kept"


def test_lm_head_sample_mass_ties(lib):
    """More ties at the top-k threshold than the sampler can store: 2000 equal top logits (behind 3 larger ones) and an all-equal
    4096 row.  The draw matches the oracle and is the same in three repeated calls and under CUDA-graph replay"""
    width, V = 4096, 3 + 4096 + 8192
    g = torch.Generator().manual_seed(9)
    vals = _fp16_exact(torch.randn(width, 3, generator=g))
    tied = torch.randperm(width, generator=g)[:2003]
    vals[tied[:3], 0] = torch.tensor([9.0, 8.5, 8.25])
    vals[tied[3:], 0] = 8.0
    vals[:, 1] = 0.0                                              # all equal
    vals[:, 2] = 0.25
    vals[tied[:7], 2] = 0.5                                       # 7 above, 4089 tied at the threshold
    for params in ((0.8, 50, 0.95), (1.0, 1024, 0.9), (0.3, 7, 1.0)):
        st = _run_sampler(3, width, V, vals.to(DEV), *params)
        runs = []
        for _ in range(3):
            st["run"]()
            torch.cuda.synchronize()
            runs.append(_check_sampler(f"sample mass ties {params}", st, width, *params))
        assert all(torch.equal(r, runs[0]) for r in runs), f"{params}: the draw changed between identical calls"
        assert float(st["dbg"][0, 1]) == 2003
        assert float(st["dbg"][1, 1]) == width
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            st["run"]()
        for _ in range(2):
            st["out_ids"].fill_(-7)
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(st["out_ids"][:, st["slot0"]].cpu(), runs[0]), f"{params}: graph replay drew another token"
