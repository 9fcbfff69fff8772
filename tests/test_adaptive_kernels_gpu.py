"""The H-Codec-1.5 adaptive kernels of csrc/adaptive.cu one entry point at a time, through the C ABI: the similarity scan against
torch's fp64 cosine and the oracle's grouping rule run on the kernel's own similarities (so a similarity at the threshold cannot
excuse a mismatch), the alignment one-hot, length packing with the zero lengths of padded groups, de-aggregation by lengths, and
the query-token aggregator's interleave / gather.  Integer and copy outputs are compared exactly, arithmetic against fp64.  Every
output buffer starts as a sentinel (NaN, or an integer no valid output takes), so an element the kernel never writes fails."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
I32_SENTINEL = -(2 ** 31)            # no index, length or group count takes it
I64_SENTINEL = -(2 ** 62)            # packed codes of these tests stay far above it


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _call(name, *args):
    """one C-ABI entry point on the current stream; tensor arguments become device pointers here, and `args` keeps every tensor
    (temporaries included) alive until the kernel has finished, so the caching allocator cannot hand a block to two arguments"""
    from unified_audio_b200 import _lib
    from unified_audio_b200.ops import _p, _stream
    ptrs = [_p(a) if isinstance(a, torch.Tensor) else a for a in args]
    _lib.check(getattr(_lib.load(), name)(*ptrs, _stream()))
    torch.cuda.synchronize()


def _plan(ns, T, seed):
    """a grouping of T frames per clip into ns[b] contiguous non-empty groups at random cut points:
    (seg [B,T], lengths [B,G] zero past each clip's groups, n_groups [B]) int64 on the host, G = max(ns)"""
    g = _gen(seed)
    B, G = len(ns), max(ns)
    seg, lens = torch.zeros(B, T, dtype=torch.long), torch.zeros(B, G, dtype=torch.long)
    for b, n in enumerate(ns):
        cuts = torch.sort(torch.randperm(T - 1, generator=g)[: n - 1] + 1).values
        ln = torch.diff(torch.cat([torch.zeros(1, dtype=torch.long), cuts, torch.tensor([T])]))
        lens[b, :n] = ln
        seg[b] = torch.repeat_interleave(torch.arange(n), ln)
    return seg, lens, torch.tensor(ns)


def _mixed_counts(T):
    """B = 4 clips: one in a single group, one with no merges (G = T), two in between"""
    return [1, T, max(1, (T + 1) // 2), max(1, T // 7)]


# ------------------------------------------------------------------------------------------------------ qb_similarity_alignment
def _similarity_alignment(h, threshold, cap):
    """the kernel on h [B,T,D] fp32 -> (sim [B,T-1], seg [B,T], lengths [B,T], n_groups [B]) on the host"""
    B, T, D = h.shape
    hd = h.to(DEV).contiguous()
    sim = torch.full((B, T - 1), float("nan"), device=DEV)
    seg = torch.full((B, T), I32_SENTINEL, dtype=torch.int32, device=DEV)
    lengths = torch.full((B, T), I32_SENTINEL, dtype=torch.int32, device=DEV)
    ng = torch.full((B,), I32_SENTINEL, dtype=torch.int32, device=DEV)
    _call("qb_similarity_alignment", hd, B, T, D, float(threshold), int(cap), sim, seg, lengths, ng)
    return sim.cpu(), seg.cpu().long(), lengths.cpu().long(), ng.cpu().long()


def _assert_grouping(got, sim, threshold, cap):
    """seg, the whole [B,T] lengths buffer (zero tail included) and n_groups equal the oracle's scan of `sim`"""
    from oracle import adaptive as oa
    _, seg, lengths, ng = got
    want_seg, want_len, want_ng = oa.segments_from_sim(sim, threshold, cap)
    assert torch.equal(ng, want_ng), f"n_groups {ng.tolist()} != {want_ng.tolist()} (threshold {threshold}, cap {cap})"
    assert torch.equal(seg, want_seg), f"frame -> token map differs (threshold {threshold}, cap {cap})"
    assert torch.equal(lengths, want_len), f"token lengths differ (threshold {threshold}, cap {cap})"


SIM_ERR = {}


@pytest.mark.parametrize("T", [2, 3, 9, 250, 4096])
@pytest.mark.parametrize("D", [1, 31, 32, 33, 512, 1024])
def test_similarity_alignment_against_fp64_cosine_and_scan(lib, T, D):
    """sim within 1e-5 of torch's fp64 cosine (eps-clamped norms); the grouping equals the oracle's scan of the kernel's own sim at
    every cap, including the ones where a similarity lies within float noise of the threshold.  Three clips of correlated frames
    (correlation 0.95, 0.5, 0.2 against the 0.5 threshold) at scales 1, 1e3 and 1e-3."""
    g = _gen(T * 1009 + D)
    B, thr = 3, 0.5
    rho = torch.tensor([0.95, 0.5, 0.2])[:, None]
    noise = torch.randn(B, T, D, generator=g)
    h = torch.empty(B, T, D)
    h[:, 0] = noise[:, 0]
    for t in range(1, T):
        h[:, t] = rho * h[:, t - 1] + (1 - rho ** 2).sqrt() * noise[:, t]
    h = h * torch.tensor([1.0, 1e3, 1e-3])[:, None, None]
    h64 = h.double()
    want = F.cosine_similarity(h64[:, :-1], h64[:, 1:], dim=2)
    first = None
    for cap in (1, 3, 8, T, 0):
        got = _similarity_alignment(h, thr, cap)
        sim = got[0]
        err = float((sim.double() - want).abs().max())
        SIM_ERR[(T, D)] = max(SIM_ERR.get((T, D), 0.0), err)
        assert err < 1e-5, f"similarity error {err:.2e} against the fp64 cosine"
        if first is None:
            first = sim
        assert torch.equal(sim, first), "the similarities must not depend on the cap"
        _assert_grouping(got, sim, thr, cap)
    print(f"[similarity T={T} D={D}] max |sim - fp64| {SIM_ERR[(T, D)]:.2e}")


def _one_hot_frames(T, D, seed):
    """frames that are 0 or a power of two times a one-hot vector, in runs: the cosine of two consecutive frames is exactly 1 (same
    hot index) or exactly 0 (different index, or a zero frame through the eps clamp) -> (h [B,T,D], exact sim [B,T-1])"""
    g = _gen(seed)
    B = 3
    hot = torch.randint(-1, 3, (B, T), generator=g)               # -1: an all-zero frame
    keep = torch.rand(B, T, generator=g) < 0.6                    # runs: repeat the previous frame's index
    for t in range(1, T):
        hot[:, t] = torch.where(keep[:, t], hot[:, t - 1], hot[:, t])
    hot[2] = -1                                                    # one clip of zero frames only
    scale = 2.0 ** torch.randint(-3, 4, (B, T), generator=g).double()
    h = torch.zeros(B, T, D, dtype=torch.float64)
    live = hot >= 0
    bi, ti = live.nonzero(as_tuple=True)
    h[bi, ti, hot[live] * (D // 3)] = scale[live]
    sim = ((hot[:, 1:] == hot[:, :-1]) & live[:, 1:]).float()
    assert torch.equal(F.cosine_similarity(h[:, :-1], h[:, 1:], dim=2).float(), sim)
    return h.float(), sim


@pytest.mark.parametrize("T", [2, 3, 9, 250, 4096])
def test_similarity_alignment_exact_cases(lib, T):
    """exact similarities (one-hot and all-zero frames) at thresholds 0 and 1, where `<=` decides every boundary that sits at the
    threshold, and thresholds -2 / 2 on random frames, where the grouping is known in closed form"""
    D = 33
    h, sim = _one_hot_frames(T, D, T)
    for thr in (0.0, 1.0):
        for cap in (1, 3, 8, T, 0):
            got = _similarity_alignment(h, thr, cap)
            assert torch.equal(got[0], sim), "cosines of one-hot / zero frames must be exactly 0 or 1"
            _assert_grouping(got, sim, thr, cap)
    assert int(_similarity_alignment(h, 1.0, 0)[3].min()) == T        # sim <= 1 everywhere: every frame opens a token
    assert int(_similarity_alignment(h, 0.0, 0)[3][2]) == T           # zero frames: sim 0 <= 0
    hr = torch.randn(2, T, D, generator=_gen(T + 1))
    t = torch.arange(T)
    for cap in (1, 3, 8, T, 0):
        got = _similarity_alignment(hr, 2.0, cap)                      # every frame is a boundary
        assert torch.equal(got[1], t.expand(2, T)) and torch.equal(got[2], torch.ones(2, T, dtype=torch.long))
        assert got[3].tolist() == [T, T]
        got = _similarity_alignment(hr, -2.0, cap)                     # no boundary: only the cap splits
        seg = t // cap if cap > 0 else torch.zeros(T, dtype=torch.long)
        n = int(seg[-1]) + 1
        want_len = torch.zeros(T, dtype=torch.long)
        want_len[:n] = torch.bincount(seg, minlength=n)
        assert torch.equal(got[1], seg.expand(2, T)) and torch.equal(got[2], want_len.expand(2, T))
        assert got[3].tolist() == [n, n]


# ------------------------------------------------------------------------------------------------------ qb_alignment_matrix
@pytest.mark.parametrize("T", [1, 2, 9, 1000])
def test_alignment_matrix_is_the_one_hot_of_seg(lib, T):
    """[B,G,T] one-hot of the frame -> token map, exact, with G above three of the four clips' group counts; T = 1000 takes the
    capped grid through several grid-stride trips"""
    seg, _, ns = _plan(_mixed_counts(T), T, 100 + T)
    B, G = seg.shape[0], int(ns.max())
    align = torch.full((B, G, T), float("nan"), device=DEV)
    _call("qb_alignment_matrix", seg.to(torch.int32).to(DEV), B, T, G, align)
    assert torch.equal(align.cpu(), F.one_hot(seg, G).transpose(1, 2).float())


# ------------------------------------------------------------------------------------------------------ qb_pack / unpack_lengths
def _pack(codes, lengths, K):
    B, nq, G = codes.shape
    out = torch.full_like(codes, I64_SENTINEL, device=DEV)
    _call("qb_pack_lengths", codes.to(DEV), lengths.to(torch.int32).to(DEV), B, nq, G, K, out)
    return out.cpu()


def _unpack(packed, K):
    B, nq, G = packed.shape
    plain = torch.full_like(packed, I64_SENTINEL, device=DEV)
    ln = torch.full((B, G), I32_SENTINEL, dtype=torch.int32, device=DEV)
    _call("qb_unpack_lengths", packed.to(DEV), B, nq, G, K, plain, ln)
    return plain.cpu(), ln.cpu().long()


@pytest.mark.parametrize("K", [1, 7, 1024])
@pytest.mark.parametrize("B,nq,G", [(3, 4, 50), (4, 8, 20000)])
def test_length_packing_round_trips_zero_lengths(lib, K, B, nq, G):
    """lengths 0 (padded groups) .. 8 packed as (length - 1) * K + code, so the codes of zero-length groups are negative and
    unpacking has to floor-divide them as Python does; equal to the oracle.  (4, 8, 20000) is 640000 codes: more than the
    capped grid covers in one trip."""
    from oracle import adaptive as oa
    g = _gen(K * 31 + G)
    codes = torch.randint(0, K, (B, nq, G), generator=g)
    lengths = torch.randint(0, 9, (B, G), generator=g)
    lengths[:, -max(1, G // 5):] = 0                                   # a padded tail, as shorter clips of a batch have
    packed = _pack(codes, lengths, K)
    assert torch.equal(packed, oa.inject_lengths(codes, lengths, K))
    assert bool((packed[:, :, -1] < 0).all())
    plain, ln = _unpack(packed, K)
    want_plain, want_len = oa.extract_lengths(packed, K)
    assert torch.equal(plain, want_plain) and torch.equal(ln, want_len)
    assert torch.equal(plain, codes) and torch.equal(ln, lengths)


@pytest.mark.parametrize("K", [1, 7, 1024])
def test_unpack_reads_the_length_of_quantizer_row_zero(lib, K):
    """every row of a code column unpacks its own code, and only row 0 gives the length, whatever rows q > 0 carry; arbitrary
    negative and positive packed codes against the oracle"""
    from oracle import adaptive as oa
    B, nq, G = 2, 4, 37
    g = _gen(K)
    codes = torch.randint(0, K, (B, nq, G), generator=g)
    row_len = torch.randint(0, 9, (B, nq, G), generator=g)             # a different length in every row
    packed = (row_len - 1) * K + codes
    plain, ln = _unpack(packed, K)
    assert torch.equal(plain, codes) and torch.equal(ln, row_len[:, 0])
    wild = torch.randint(-50 * K, 50 * K, (B, nq, G), generator=g)
    plain, ln = _unpack(wild, K)
    want_plain, want_len = oa.extract_lengths(wild, K)
    assert torch.equal(plain, want_plain) and torch.equal(ln, want_len)


# ------------------------------------------------------------------------------------------------------ qb_length_offsets + qb_deaggregate
@pytest.mark.parametrize("dtype", [torch.float32, torch.int64])
@pytest.mark.parametrize("B,C,G", [(3, 24, 17), (2, 1024, 300)])
def test_deaggregate_by_lengths_against_repeat_interleave(lib, dtype, B, C, G):
    """offsets are the exclusive prefix sums of the lengths; each clip's tokens repeated `length` times, cut at T_out when the clip
    is longer and zero-filled when it is shorter, with trailing zero-length groups; bit-exact against per-clip repeat_interleave.
    (2, 1024, 300) is 614400 tokens: more than the capped grid covers in one trip."""
    g = _gen(B * C + G)
    lengths = torch.randint(0, 9, (B, G), generator=g)
    lengths[0, -3:] = 0
    lengths[1, G // 2:] = 0                                            # the shortest clip: zero-filled in every T_out below
    ln32 = lengths.to(torch.int32).to(DEV)
    off = torch.full((B, G), I32_SENTINEL, dtype=torch.int32, device=DEV)
    tot = torch.full((B,), I32_SENTINEL, dtype=torch.int32, device=DEV)
    _call("qb_length_offsets", ln32, B, G, off, tot)
    totals = lengths.sum(1)
    assert torch.equal(off.cpu().long(), torch.cumsum(lengths, 1) - lengths) and torch.equal(tot.cpu().long(), totals)
    if dtype == torch.float32:
        x = torch.randn(B, C, G, generator=g)
    else:
        x = torch.randint(-2 ** 40, 2 ** 40, (B, C, G), generator=g)
    full = [torch.repeat_interleave(x[b], lengths[b], dim=1) for b in range(B)]
    for T_out in (int(totals.max()), int(totals[0]) - 5, int(totals.max()) + 7):
        sentinel = float("nan") if dtype == torch.float32 else I64_SENTINEL
        out = torch.full((B, C, T_out), sentinel, dtype=dtype, device=DEV)
        _call("qb_deaggregate", x.to(DEV), x.element_size(), ln32, off, B, C, G, T_out, out)
        want = torch.zeros(B, C, T_out, dtype=dtype)
        for b in range(B):
            n = min(T_out, full[b].shape[1])
            want[b, :, :n] = full[b][:, :n]
        assert torch.equal(out.cpu(), want), f"de-aggregation differs at T_out {T_out} (clip totals {totals.tolist()})"


# ------------------------------------------------------------------------------------------------------ qb_agg_interleave / qb_agg_gather
MEAN_ERR = {}


def _interleave(feats, seg, lengths, ns, qemb):
    B, T, D = feats.shape
    G = lengths.shape[1]
    offsets = torch.cumsum(lengths, 1) - lengths
    i32 = lambda t: t.to(torch.int32).to(DEV).contiguous()
    out = torch.full((B, T + G, D), float("nan"), device=DEV)
    qpos = torch.full((B, G), I32_SENTINEL, dtype=torch.int32, device=DEV)
    _call("qb_agg_interleave", feats.to(DEV), i32(seg), i32(lengths), i32(offsets), i32(ns), qemb.to(DEV),
          B, T, G, D, out, qpos)
    return out.cpu(), qpos.cpu().long()


@pytest.mark.parametrize("T", [1, 2, 3, 250, 1000])
@pytest.mark.parametrize("D", [64, 130, 512, 1024])
def test_agg_interleave_and_gather(lib, T, D):
    """the T + G sequence of the query-token aggregator against oracle.hcodec15.interleave_plan: frames copied bit for bit to their
    rows, the query of each live group at its row holding the fp64 group mean + the embedding (within 1e-6 of the row's largest
    value), padded groups the bare embedding, no row left unwritten (T + G blocks writing T + G distinct rows: each exactly once);
    then the gather reads the live query rows back exactly and zeros for padded groups"""
    from oracle import hcodec15 as o15
    ns = _mixed_counts(T)
    seg, lengths, n = _plan(ns, T, 7 * T + D)
    B, G = len(ns), int(n.max())
    g = _gen(T + D)
    feats = torch.randn(B, T, D, generator=g)
    qemb = torch.randn(D, generator=g)
    out, qpos = _interleave(feats, seg, lengths, n, qemb)
    align = F.one_hot(seg, G).transpose(1, 2).float()
    fpos, want_qpos, gmask = o15.interleave_plan(align, n)
    assert torch.equal(qpos, want_qpos)
    rows = torch.cat([fpos, want_qpos], 1)
    assert torch.equal(torch.sort(rows, 1).values, torch.arange(T + G).expand(B, T + G))    # the plan is a permutation of rows
    assert not bool(out.isnan().any()), "rows of the T + G sequence left unwritten"
    bi = torch.arange(B)[:, None]
    assert torch.equal(out[bi, fpos], feats), "frame rows must be exact copies"
    mean = torch.einsum("bgt,btd->bgd", align.double(), feats.double()) / lengths.clamp(min=1).double()[..., None]
    want_q = mean + qemb.double()
    got_q = out[bi, want_qpos].double()
    worst = 0.0
    for b in range(B):
        live = int(n[b])
        err = ((got_q[b, :live] - want_q[b, :live]).abs().amax(1) / want_q[b, :live].abs().amax(1)).max()
        worst = max(worst, float(err))
        assert torch.equal(got_q[b, live:].float(), qemb.expand(G - live, D)), "padded query rows must be the bare embedding"
    MEAN_ERR[(T, D)] = worst
    print(f"[agg_interleave T={T} D={D}] groups {ns}: max relative error of the query rows {worst:.2e}")
    assert worst < 1e-6
    # gather from a sequence whose rows all differ, so a wrong row cannot pass
    x = torch.randn(B, T + G, D, generator=g).to(DEV)
    tok = torch.full((B * G, D), float("nan"), device=DEV)
    _call("qb_agg_gather", x, qpos.to(torch.int32).to(DEV), n.to(torch.int32).to(DEV), B, T + G, G, D, tok)
    tok = tok.cpu().reshape(B, G, D)
    want = x.cpu()[bi, want_qpos] * gmask[..., None]
    assert torch.equal(tok, want)
    for b in range(B):
        assert bool((tok[b, int(n[b]):] == 0).all())
