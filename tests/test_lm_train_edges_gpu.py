"""The UniSE LM's training path at the batch, seeds, tiles and loss scales training uses (csrc/lm_train.cu, the split-K 3-term weight
gradients, llm._LMLoss), each against fp64 or exactly:
  - the dropout masks the attention kernels really apply, read back bit for bit (forward through out, backward through dV) and
    compared with oracle/llama_train.dropout_keep at seeds whose high word is set, large layers and the threshold edge;
  - training attention at L next to and on its 32-row tiles, 8 heads and B = 3;
  - transpose_split, weight_grad, lm_loss_bwd, embedding_bwd, col_sum, SwiGLU and RMSNorm backward at the shipped shapes and edges;
  - whole-model gradients at B = 8 and 32 against the oracle run on the GPU, and the batch gradient as the mean of per-utterance ones;
  - the autograd contract: (c * loss).backward() is c times the gradient, micro-batches add exactly, and a parameter changed in place
    between forward and backward is refused."""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import llama, llama_train
from test_lm_train_edges_host import EDGE, HEADS, edge_word
from test_lm_train_gpu import K, lm_inputs, make_face

pytestmark = pytest.mark.gpu

SEEDS = (0, 2 ** 32 - 1, 2 ** 32, 2 ** 62 - 1, 2 ** 64 - 1)
LAYERS = (0, 11, 2 ** 31 - 1)
BIG_SEED = 2 ** 40 + 12345                # a seed whose high word (seed >> 32) is not zero


def frob(a, b):
    """relative Frobenius error of a against b, in fp64 on b's device"""
    a, b = torch.as_tensor(a).to(b.device).double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


@pytest.fixture
def no_tf32():
    """fp32 oracle GEMMs in full fp32 (no TF32), restored afterwards"""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# ------------------------------------------------------------------------------------------------------------------- dropout masks
def read_masks(B, L, heads, p, seed, layer):
    """(forward, backward) keep masks bool [B, heads, L, L] as the kernels apply them.  With q = k = 0 every causal score is 0, so
    P[i, j] = 1 / (i + 1) whatever RoPE does.  Forward: v row j = e_(j - 64w) for the keys of window w, so out[i, d] > 0 exactly
    when key 64w + d of query i is kept.  Backward: dO row i = e_(i - 64w) for the queries of window w, so dV[j, d] =
    P_dropped[64w + d, j] > 0 exactly when query 64w + d keeps key j."""
    from unified_audio_b200 import ops
    H = heads * 64
    cos, sin = ops.rope_tables(max(L, 64), 64, "cuda")
    d = lambda *s: torch.empty(*s, device="cuda")
    qs, kr, v, o, lse = d(B * heads, L, 64), d(B * heads, L, 64), d(B * heads, L, 64), d(B * L, H), d(B * heads, L)
    qkv = torch.zeros(B, L, 3, heads, 64, device="cuda")
    fwd = torch.zeros(B, heads, L, L, dtype=torch.bool, device="cuda")
    bwd = torch.zeros(B, heads, L, L, dtype=torch.bool, device="cuda")
    for w0 in range(0, L, 64):
        n = min(64, L - w0)
        qkv.zero_()
        qkv[:, w0:w0 + n, 2, :, :n] = torch.eye(n, device="cuda")[:, None, :]
        ops.lm_attn_train_fwd(qkv.view(B * L, 3 * H), B, L, heads, cos, sin, p, seed, layer, qs, kr, v, o, lse)
        fwd[..., w0:w0 + n] = o.view(B, L, heads, 64)[..., :n].permute(0, 2, 1, 3) > 0
    qkv.zero_()
    ops.lm_attn_train_fwd(qkv.view(B * L, 3 * H), B, L, heads, cos, sin, p, seed, layer, qs, kr, v, o, lse)
    dout, dqkv, ws = torch.zeros(B, L, heads, 64, device="cuda"), d(B * L, 3 * H), d(B * heads * L)
    for w0 in range(0, L, 64):
        n = min(64, L - w0)
        dout.zero_()
        dout[:, w0:w0 + n, :, :n] = torch.eye(n, device="cuda")[:, None, :]
        ops.lm_attn_train_bwd(qs, kr, v, o, dout.view(B * L, H), lse, B, L, heads, cos, sin, p, seed, layer, dqkv, ws)
        bwd[..., w0:w0 + n, :] = dqkv.view(B, L, 3, heads, 64)[:, :, 2, :, :n].permute(0, 2, 3, 1) > 0
    return fwd, bwd


def check_mask(got, keep, what):
    L = keep.shape[-1]
    tri = torch.ones(L, L, dtype=torch.bool, device="cuda").tril()
    want = torch.as_tensor(keep).cuda()
    assert not got[..., ~tri].any(), f"{what}: a key after its query contributes"
    bad = int((got[..., tri] != want[..., tri]).sum())
    assert bad == 0, f"{what}: {bad} of {int(tri.sum()) * keep.shape[0] * keep.shape[1]} mask bits differ from dropout_keep"


@pytest.mark.parametrize("layer", LAYERS)
@pytest.mark.parametrize("seed", SEEDS)
def test_dropout_mask_exact(lib, seed, layer):
    """B = 3, 8 heads, L = 786 (13 windows of 64) at p = 0.1 and L = 130 at p = 0.5 and 0.9: both kernels' masks equal
    dropout_keep bit for bit over the whole causal triangle"""
    B = 3
    for p, L in ((0.1, 786), (0.5, 130), (0.9, 130)):
        words = llama_train.dropout_words(seed, layer, B, HEADS, L)
        keep = words >= np.uint64(llama_train.dropout_threshold(p))
        assert np.array_equal(keep, llama_train.dropout_keep(seed, layer, B, HEADS, L, p))
        fwd, bwd = read_masks(B, L, HEADS, p, seed, layer)
        check_mask(fwd, keep, f"forward seed={seed} layer={layer} p={p}")
        check_mask(bwd, keep, f"backward seed={seed} layer={layer} p={p}")
        # the kept fraction is 1 - p within 5 sigma over the causal triangle
        n = B * HEADS * L * (L + 1) // 2
        kept = int(fwd.sum())
        assert abs(kept - n * (1 - p)) < 5 * (n * p * (1 - p)) ** 0.5, (kept, n, p)


def test_dropout_mask_edges(lib):
    B, L = 3, 200
    fwd, bwd = read_masks(B, L, HEADS, 0.0, BIG_SEED, 3)
    check_mask(fwd, np.ones((B, HEADS, L, L), dtype=bool), "p = 0 forward")
    check_mask(bwd, np.ones((B, HEADS, L, L), dtype=bool), "p = 0 backward")
    # seeds that differ only in the high word draw different masks, each the oracle's
    lo = 0x0BADC0DE
    a, _ = read_masks(B, L, HEADS, 0.1, (1 << 32) | lo, 3)
    b, _ = read_masks(B, L, HEADS, 0.1, (2 << 32) | lo, 3)
    c, _ = read_masks(B, L, HEADS, 0.1, lo, 3)
    assert not torch.equal(a, b) and not torch.equal(a, c)
    check_mask(b, llama_train.dropout_keep((2 << 32) | lo, 3, B, HEADS, L, 0.1), "high word 2")


@pytest.mark.parametrize("p,word,t", EDGE)
def test_dropout_threshold_edge(lib, p, word, t):
    """a key whose word equals the threshold is kept, one at threshold - 1 dropped; at p = 0.09 the threshold is float32(p) * 2^24
    rounded (1509950), not the double's (1509949)"""
    seed, b, h, i, j, layer = t
    assert edge_word(*t) == word                               # recomputed on the CPU before it is used
    thr = llama_train.dropout_threshold(p)
    B, L = 3, 96
    fwd, bwd = read_masks(B, L, HEADS, p, seed, layer)
    assert bool(fwd[b, h, i, j]) == (word >= thr) and bool(bwd[b, h, i, j]) == (word >= thr), (p, word, thr)
    keep = llama_train.dropout_keep(seed, layer, B, HEADS, L, p)
    check_mask(fwd, keep, f"forward p={p}")
    check_mask(bwd, keep, f"backward p={p}")


# ------------------------------------------------------------------------------------------------------------------- attention tiles
def attention_fp64(qkv, B, L, heads, keep, p):
    """causal attention with RoPE as the LM runs it, fp64 on qkv's device, differentiable in qkv"""
    H = heads * 64
    q, k, v = (qkv.view(B, L, 3, heads, 64)[:, :, i].transpose(1, 2) for i in range(3))
    cos, sin = (t.to(qkv.device) for t in llama._rope(torch.arange(L), 64, torch.float64))
    q, k = q * cos + llama._rot(q) * sin, k * cos + llama._rot(k) * sin
    s = (q @ k.transpose(2, 3)) / 8.0
    s = s.masked_fill(~torch.ones(L, L, dtype=torch.bool, device=qkv.device).tril(), float("-inf"))
    lse = torch.logsumexp(s, -1)
    a = torch.softmax(s, -1)
    if keep is not None:
        a = a * torch.as_tensor(keep).to(qkv.device).double() / (1 - p)
    return (a @ v).transpose(1, 2).reshape(B * L, H), lse.reshape(B * heads, L)


@pytest.mark.parametrize("L", [31, 32, 33, 63, 64, 65, 96, 97, 535, 786])
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("scale", [1.0, 6.0])
def test_attention_train_tiles_vs_fp64(lib, L, p, scale):
    from unified_audio_b200 import ops
    B, heads, layer = 3, HEADS, 7
    H = heads * 64
    g = torch.Generator().manual_seed(1000 * L + int(10 * p) + int(scale))
    qkv = (scale * torch.randn(B * L, 3 * H, generator=g)).cuda()          # different content for every (b, h)
    dout = torch.randn(B * L, H, generator=g).cuda()
    cos, sin = ops.rope_tables(max(L, 64), 64, "cuda")
    d = lambda *s: torch.empty(*s, device="cuda")
    qs, kr, v, o, lse = d(B * heads, L, 64), d(B * heads, L, 64), d(B * heads, L, 64), d(B * L, H), d(B * heads, L)
    ops.lm_attn_train_fwd(qkv, B, L, heads, cos, sin, p, BIG_SEED, layer, qs, kr, v, o, lse)
    dqkv = d(B * L, 3 * H)
    ops.lm_attn_train_bwd(qs, kr, v, o, dout, lse, B, L, heads, cos, sin, p, BIG_SEED, layer, dqkv, d(B * heads * L))
    keep = llama_train.dropout_keep(BIG_SEED, layer, B, heads, L, p) if p > 0 else None
    x = qkv.double().requires_grad_(True)
    o64, lse64 = attention_fp64(x, B, L, heads, keep, p)
    o64.backward(dout.double())
    errs = dict(out=frob(o, o64.detach()), lse=frob(lse, lse64.detach()), dqkv=frob(dqkv, x.grad))
    print(f"L={L} p={p} scale={scale}", errs)
    assert errs["out"] < 2e-6 and errs["lse"] < 2e-6 and errs["dqkv"] < 2e-5, errs


# ------------------------------------------------------------------------------------------------------------------- kernels
def bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("rows,cols,ldx,ks", [(31, 33, 40, 64), (1000, 77, 77, 64), (1000, 513, 600, 512), (9056, 12291, 12352, 64),
                                              (9056, 12291, 12352, 1536), (17120, 1536, 1536, 512), (25152, 512, 512, 1536)])
def test_transpose_split_bitwise(lib, rows, cols, ldx, ks):
    """planes [S, cols, ks] equal split_f16 of the zero-padded transpose bit for bit, zeroed rows past `rows` included; the pitch
    columns past `cols` (NaN here) are never read"""
    from unified_audio_b200 import ops
    g = torch.Generator().manual_seed(rows + cols)
    x = torch.randn(rows, ldx, generator=g)
    x[::7, ::5] *= 1e5                                        # beyond fp16's range: hi saturates
    x[1::7, ::3] *= 1e-6                                      # fp16 subnormals
    x[:, cols:] = float("nan")
    x = x.cuda()
    got = ops.transpose_split(x, rows, cols, ks, ldx)
    S = -(-rows // ks)
    assert got.hi.shape == (S, cols, ks)
    xt = torch.zeros(S * ks, cols, device="cuda")
    xt[:rows] = x[:, :cols]
    t = xt.view(S, ks, cols).transpose(1, 2).contiguous()
    ref = ops.Planes.zeros(t.shape, True, "cuda")
    ops.split_f16(t, ref)
    assert torch.equal(bits(got.hi), bits(ref.hi)) and torch.equal(bits(got.lo), bits(ref.lo))


WG_SHAPES = [(1536, 512), (512, 2048), (4096, 512)]


@pytest.mark.parametrize("tokens", [9056, 17120, 25152])
def test_weight_grad_training_batch_vs_fp64(lib, tokens):
    """dW = dY^T X with ks from grad_slice at B * L of the training batch (several split-K slices), and the head's gradient over
    B * Lt = 9 056 tokens with dY's row pitch 12 352 (pitch columns NaN: never read)"""
    from unified_audio_b200 import ops
    g = torch.Generator().manual_seed(tokens)
    cases = [(n_out, n_in, n_out) for n_out, n_in in WG_SHAPES] + ([(12291, 512, 12352)] if tokens == 9056 else [])
    for n_out, n_in, ld in cases:
        dy = torch.randn(tokens, ld, generator=g)
        dy[:, n_out:] = float("nan")
        x = torch.randn(tokens, n_in, generator=g)
        dy, x = dy.cuda(), x.cuda()
        ks = ops.grad_slice(tokens, n_out, n_in)
        w = ops.weight_grad(dy, x, tokens, n_out, n_in, torch.empty(n_out, n_in, device="cuda"), dy_ld=ld)
        ref = dy[:, :n_out].double().T @ x.double()
        e = frob(w, ref)
        # each slice accumulates its ks tokens in the tensor cores' fp32 accumulator, whose error relative to the sum grows about
        # linearly in ks: 3.5e-9 * ks measured on an H100 SXM at 700 W (1.1e-5 at ks = 3 072, 3.2e-5 for the head's single slice of
        # 9 088); a lost slice, a wrong row offset or a missing lo plane is 1e-3 or more
        bound = 6e-9 * ks
        print(f"tokens={tokens} ({n_out}, {n_in}) ks={ks} slices={-(-tokens // ks)}: rel {e:.2e} (bound {bound:.2e})")
        assert torch.isfinite(w).all() and e < bound, (n_out, n_in, ks, e)


@pytest.mark.parametrize("grad_loss", [2.0 ** -16, 1.0, 5.0, 16.0, 2.0 ** 16])
def test_lm_loss_bwd_shipped_vocab(lib, grad_loss):
    """V = 12 291 with ld_out = 12 352, rows confidently right and confidently wrong (logit gaps of 40 nats): the fp32 rows are
    fp32-grade for every grad_loss and the padding columns exactly 0; the planes are fp32-grade at the unit grad_loss the LM passes
    (their range is |grad_loss| * 2^14 inside fp16's: include/quark_b200.h)"""
    from unified_audio_b200 import ops
    M, V, Vp = 48, 12291, 12352
    g = torch.Generator().manual_seed(17)
    logits, tg = 4 * torch.randn(M, V, generator=g, dtype=torch.float64), torch.randint(0, V, (M,), generator=g)
    rows = torch.arange(M)
    logits[rows[:16], tg[:16]] += 40.0                                     # confident and right
    wrong = (tg[16:32] + 1 + rows[16:32]) % V
    logits[rows[16:32], wrong] += 40.0                                     # confident and wrong
    logits = logits.float().cuda()
    scale = ops.lm_loss_scale(V)
    out = torch.full((M, Vp), float("nan"), device="cuda")
    pl = ops.Planes(torch.full((M, Vp), float("nan"), dtype=torch.float16, device="cuda"),
                    torch.full((M, Vp), float("nan"), dtype=torch.float16, device="cuda"))
    ops.lm_loss_bwd(logits, V, M, V, tg.cuda(), 0.1, torch.tensor([grad_loss], device="cuda"), out, pl, Vp, scale)
    ld = logits.double().requires_grad_(True)
    true = torch.full((M, V), 0.1 / (V - 1), dtype=torch.float64, device="cuda").scatter_(1, tg.cuda()[:, None], 0.9)
    (grad_loss * F.kl_div(torch.log_softmax(ld, -1), true, reduction="batchmean")).backward()
    e_rows = frob(out[:, :V] / (M * scale), ld.grad)
    e_planes = frob(pl.float()[:, :V] / (M * scale), ld.grad)
    print(f"grad_loss={grad_loss}: rows rel {e_rows:.2e}, planes rel {e_planes:.2e}")
    assert e_rows < 1e-6
    for t in (out[:, V:], pl.hi[:, V:], pl.lo[:, V:]):
        assert bool((t == 0).all()), "padding columns must be written as 0"
    if grad_loss == 1.0:
        assert e_planes < 1e-6


@pytest.mark.parametrize("H", [512, 1024])
def test_embedding_bwd_training_batch(lib, H):
    """V = 12 291, n = B * Lt = 9 056 (B = 32): an id at 313 positions (across the kernel's 256-wide chunks), ids 0 and V - 1,
    written and accumulated"""
    from unified_audio_b200 import ops
    B, P, Lt, V = 32, 252, 283, 12291
    L = P + Lt
    g = torch.Generator().manual_seed(H)
    dx = torch.randn(B * L, H, generator=g).cuda()
    ids = torch.randint(1, V - 1, (B, Lt), generator=g)
    ids.view(-1)[::29] = 5
    ids[0, 0], ids[7, 100], ids[-1, -1] = 0, V - 1, V - 1
    assert int((ids == 5).sum()) > 256
    ids = ids.cuda()
    ref = torch.zeros(V, H, dtype=torch.float64, device="cuda").index_add_(
        0, ids.reshape(-1), dx.double().view(B, L, H)[:, P:].reshape(-1, H)) * 0.25
    out = torch.empty(V, H, device="cuda")
    ops.embedding_bwd(dx, ids, ids.numel(), Lt, L, P, H, V, out, scale=0.25)
    assert frob(out, ref) < 1e-7 and frob(out[5], ref[5]) < 1e-7
    assert frob(out[0], ref[0]) < 1e-7 and frob(out[V - 1], ref[V - 1]) < 1e-7
    base = torch.randn(V, H, generator=g).cuda()
    acc = base.clone()
    ops.embedding_bwd(dx, ids, ids.numel(), Lt, L, P, H, V, acc, accumulate=True, scale=0.25)
    assert frob(acc, base.double() + ref) < 1e-7


def test_col_sum_chunks_pitch_accumulate(lib):
    from unified_audio_b200 import ops
    g = torch.Generator().manual_seed(8)
    for rows, C, ld in ((1000, 513, 600), (129, 77, 77), (17120, 512, 515)):
        x = torch.randn(rows, ld, generator=g)
        x[:, C:] = float("nan")                                 # pitch columns are never read
        x = x.cuda()
        ref = x[:, :C].double().sum(0)
        out = torch.empty(C, device="cuda")
        ops.col_sum(x, rows, C, ld, out, scale=0.5)
        assert frob(out, 0.5 * ref) < 1e-7, (rows, C)
        base = torch.randn(C, generator=g).cuda()
        acc = base.clone()
        ops.col_sum(x, rows, C, ld, acc, accumulate=True, scale=0.5)
        assert frob(acc, base.double() + 0.5 * ref) < 1e-7, (rows, C)


def test_swiglu_saturated_gates(lib):
    """gates of +-20 and +-90 (expf(-g) overflows to inf at -90): forward and backward finite and fp32-grade"""
    from unified_audio_b200 import ops
    M, I = 64, 256
    g = torch.Generator().manual_seed(9)
    gu, dh = 3 * torch.randn(M, 2 * I, generator=g), torch.randn(M, I, generator=g)
    gate = gu[:, 0::2]
    gate[::4] = 20.0
    gate[1::4] = -20.0
    gate[2::4] = 90.0
    gate[3::4, ::2] = -90.0
    gu[:, 0::2] = gate
    h, hp = torch.empty(M, I, device="cuda"), ops.Planes.zeros((M, I), True, "cuda")
    dgu, dp = torch.empty(M, 2 * I, device="cuda"), ops.Planes.zeros((M, 2 * I), True, "cuda")
    ops.swiglu(gu.cuda(), M, I, h, hp)
    ops.swiglu_bwd(gu.cuda(), dh.cuda(), M, I, dgu, dp)
    gud = gu.double().cuda().requires_grad_(True)
    hd = F.silu(gud[:, 0::2]) * gud[:, 1::2]
    hd.backward(dh.double().cuda())
    for t in (h, hp.float(), dgu, dp.float()):
        assert torch.isfinite(t).all()
    assert frob(h, hd.detach()) < 1e-6 and frob(hp.float(), hd.detach()) < 1e-6
    assert frob(dgu, gud.grad) < 1e-6 and frob(dp.float(), gud.grad) < 1e-6


@pytest.mark.parametrize("accumulate", [False, True])
def test_rmsnorm_bwd_rows_near_eps(lib, accumulate):
    """C = 512 with rows whose RMS is 0.5, 1 and 2 times sqrt(eps), all-zero rows and ordinary rows"""
    from unified_audio_b200 import ops
    M, C = 300, 512
    g = torch.Generator().manual_seed(10)
    x, dy, dx0 = (torch.randn(M, C, generator=g) for _ in range(3))
    for k, f in enumerate((0.5, 1.0, 2.0)):
        x[100 + 30 * k:130 + 30 * k] *= f * 1e-3                          # sqrt(1e-6) = 1e-3
    x[190:200] = 0.0
    w = 1 + 0.1 * torch.randn(C, generator=g)
    dx, gw, dw = dx0.cuda().clone(), torch.empty(M, C, device="cuda"), torch.empty(C, device="cuda")
    ops.rmsnorm_bwd(x.cuda(), w.cuda(), dy.cuda(), M, C, dx, gw, accumulate)
    ops.col_sum(gw, M, C, C, dw)
    xd, wd = x.double().cuda().requires_grad_(True), w.double().cuda().requires_grad_(True)
    F.rms_norm(xd, (C,), wd, 1e-6).backward(dy.double().cuda())
    want = xd.grad + (dx0.double().cuda() if accumulate else 0)
    assert frob(dx, want) < 1e-6 and frob(dw, wd.grad) < 1e-6
    assert frob(dx[100:190], want[100:190]) < 1e-6 and frob(dx[190:200], want[190:200]) < 1e-6


# ------------------------------------------------------------------------------------------------------------------- whole model
def face_grads(lm, task, x, seed, rows=slice(None)):
    lm.zero_grad(set_to_none=True)
    enr = x["enroll"][rows].cuda() if task == "tse" else None
    loss, _ = lm(task, enr, enr, None, x["mix"][rows].cuda(), x["gids"][rows].cuda(), x["sids"][rows].cuda(), dropout_seed=seed)
    loss.backward()
    return loss.detach(), {n: p.grad for n, p in lm.named_parameters() if p.grad is not None}


def oracle_grads_gpu(cfg, sd, task, x, dtype, p, seed, chunk=None):
    """the oracle's loss and gradients on the GPU; with `chunk`, over chunks of that many utterances weighted by their share of the
    rows (every utterance has the same number of target rows, so the batch loss is the mean of the chunk losses)"""
    B = x["mix"].shape[0]
    chunk = chunk or B
    loss, grads = 0.0, {}
    for c0 in range(0, B, chunk):
        r = slice(c0, c0 + chunk)
        osd = {k: v.to("cuda", dtype).requires_grad_(True) for k, v in sd.items()}
        cx = {k: v[r].cuda() for k, v in x.items()}
        l, _ = llama_train.sft_forward(osd, cfg, task, cx["enroll"].to(dtype) if task == "tse" else None, cx["mix"].to(dtype),
                                       cx["gids"], cx["sids"], dropout_p=p, dropout_seed=seed)
        l.backward()
        w = cx["mix"].shape[0] / B
        loss += w * float(l)
        for n, t in osd.items():
            if t.grad is not None:
                grads[n] = grads[n] + w * t.grad if n in grads else w * t.grad
        del osd, l
    return loss, grads


def bounds(g64, g32):
    gaps = {n: frob(g32[n], g64[n]) for n in g64}
    floor = sorted(gaps.values())[len(gaps) // 2]
    return {n: K * max(gaps[n], floor) for n in g64}, gaps


def check_against(tag, g, g64, bound, gaps):
    assert set(g) == set(g64), set(g) ^ set(g64)
    worst, worst_n = 0.0, None
    for n in g64:
        e = frob(g[n], g64[n])
        print(f"{tag} {n}: rel {e:.2e} (fp32 oracle gap {gaps[n]:.2e}, bound {bound[n]:.2e})")
        assert e < bound[n], (tag, n, e, bound[n])
        if e / bound[n] > worst:
            worst, worst_n = e / bound[n], n
    print(f"{tag}: worst error / bound {worst:.3f} ({worst_n})")
    return worst


@pytest.mark.parametrize("task,Te,L", [("se", 1, 535), ("tse", 250, 786)])
def test_model_grads_b8_dropout_vs_oracle(lib, no_tf32, task, Te, L):
    """shipped widths, B = 8, attention dropout 0.1 at a seed above 2^32"""
    cfg = llama.LM_FULL
    sd = llama.make_lm_state_dict(cfg, 7, 2.0)
    x = lm_inputs(cfg, 8, 250, Te, 249, 31)
    lm = make_face(cfg, sd).requires_grad_(True).train()
    loss, g = face_grads(lm, task, x, BIG_SEED)
    l64, g64 = oracle_grads_gpu(cfg, sd, task, x, torch.float64, 0.1, BIG_SEED)
    _, g32 = oracle_grads_gpu(cfg, sd, task, x, torch.float32, 0.1, BIG_SEED)
    bound, gaps = bounds(g64, g32)
    check_against(f"B=8 {task} L={L} p=0.1", g, g64, bound, gaps)
    assert abs(float(loss) - l64) < 1e-5 * abs(l64)


def test_model_grads_b32_vs_oracle_and_per_utterance(lib, no_tf32):
    """shipped widths, B = 32 'se' (L = 535, 17 120 tokens; 9 056 target rows), no dropout: the face's gradient against the oracle's
    (computed in chunks of 8 utterances), and against the mean of the 32 single-utterance gradients of the face"""
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    cfg = llama.LM_FULL
    sd = llama.make_lm_state_dict(cfg, 7, 2.0)
    B = 32
    x = lm_inputs(cfg, B, 250, 1, 249, 32)
    lm = make_face(cfg, sd).requires_grad_(True).eval()
    loss, g = face_grads(lm, "se", x, 0)
    g = {n: t.clone() for n, t in g.items()}
    l64, g64 = oracle_grads_gpu(cfg, sd, "se", x, torch.float64, 0.0, None, chunk=8)
    _, g32 = oracle_grads_gpu(cfg, sd, "se", x, torch.float32, 0.0, None, chunk=8)
    bound, gaps = bounds(g64, g32)
    check_against("B=32 se p=0", g, g64, bound, gaps)
    assert abs(float(loss) - l64) < 1e-5 * abs(l64)
    del g32
    mean = {n: torch.zeros_like(t, dtype=torch.float64) for n, t in g.items()}
    for b in range(B):
        _, gb = face_grads(lm, "se", x, 0, rows=slice(b, b + 1))
        for n, t in gb.items():
            mean[n] += t.double() / B
    worst = 0.0
    for n in g:
        e = frob(g[n], mean[n])
        assert e < bound[n], ("batch vs mean of single utterances", n, e, bound[n])
        worst = max(worst, e / bound[n])
    print(f"B=32 batch gradient vs mean of 32 single-utterance gradients: worst error / bound {worst:.3f}")
    torch.cuda.synchronize()
    print(f"B=32 test: {time.perf_counter() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB")


# ------------------------------------------------------------------------------------------------------------------- autograd contract
def shipped_face_b2():
    cfg = llama.LM_FULL
    lm = make_face(cfg, llama.make_lm_state_dict(cfg, 7, 2.0)).requires_grad_(True).train()
    return lm, lm_inputs(cfg, 2, 250, 1, 249, 41), lm_inputs(cfg, 2, 250, 1, 249, 42)


def se_loss(lm, x, seed):
    return lm("se", None, None, None, x["mix"].cuda(), x["gids"].cuda(), x["sids"].cuda(), dropout_seed=seed)[0]


def grads_of(lm):
    return {n: p.grad.clone() for n, p in lm.named_parameters() if p.grad is not None}


def test_loss_scale_homogeneity(lib):
    """(c * loss).backward() gives c times the gradient of loss: bitwise for powers of two, within 1 ulp of fl(c * g) otherwise,
    finite at a GradScaler's 2^16"""
    lm, x, _ = shipped_face_b2()
    lm.zero_grad(set_to_none=True)
    l1 = se_loss(lm, x, BIG_SEED)
    l1.backward()
    g1 = grads_of(lm)
    for c in (2.0 ** -16, 2.0 ** -8, 1 / 3, 5.0, 16.0, -2.0, 2.0 ** 16):
        lm.zero_grad(set_to_none=True)
        lc = se_loss(lm, x, BIG_SEED)
        assert torch.equal(lc, l1)
        (c * lc).backward()
        cf = torch.tensor(c, dtype=torch.float32, device="cuda")
        pow2 = abs(c) == 2.0 ** round(np.log2(abs(c)))
        assert set(grads_of(lm)) == set(g1)
        for n in g1:
            got, want = lm.get_parameter(n).grad, g1[n] * cf
            assert torch.isfinite(got).all(), (c, n)
            if pow2:
                assert torch.equal(got, want), (c, n, frob(got, want))
            else:
                ulps = (got.view(torch.int32).long() - want.view(torch.int32).long()).abs()
                assert bool(((got == want) | (ulps <= 1)).all()), (c, n, frob(got, want))


def test_micro_batches_add_exactly(lib):
    """two forwards then (l1 + l2).backward(), and two backward() calls accumulating into .grad, both equal the sum of the separate
    gradients bit for bit"""
    lm, x1, x2 = shipped_face_b2()
    sep = []
    for x, s in ((x1, BIG_SEED), (x2, BIG_SEED + 1)):
        lm.zero_grad(set_to_none=True)
        se_loss(lm, x, s).backward()
        sep.append(grads_of(lm))
    want = {n: sep[0][n] + sep[1][n] for n in sep[0]}
    lm.zero_grad(set_to_none=True)
    (se_loss(lm, x1, BIG_SEED) + se_loss(lm, x2, BIG_SEED + 1)).backward()
    got = grads_of(lm)
    assert set(got) == set(want) and all(torch.equal(got[n], want[n]) for n in want)
    lm.zero_grad(set_to_none=True)
    se_loss(lm, x1, BIG_SEED).backward()
    se_loss(lm, x2, BIG_SEED + 1).backward()
    got = grads_of(lm)
    assert set(got) == set(want) and all(torch.equal(got[n], want[n]) for n in want)


def test_parameter_changed_after_forward_is_refused(lib):
    lm, x, _ = shipped_face_b2()
    prm = dict(lm.named_parameters())
    loss = se_loss(lm, x, BIG_SEED)
    with torch.no_grad():
        prm["layers.3.mlp.down_proj.weight"].mul_(1.01)                    # e.g. an optimizer step before the backward
    with pytest.raises(RuntimeError, match="changed in place"):
        loss.backward()
    loss = se_loss(lm, x, BIG_SEED)
    prm["output_head.weight"].data = prm["output_head.weight"].data.clone()  # same values, new storage
    with pytest.raises(RuntimeError, match="changed in place"):
        loss.backward()
    lm.zero_grad(set_to_none=True)
    se_loss(lm, x, BIG_SEED).backward()                                      # a fresh forward works
    assert all(p.grad is not None for n, p in prm.items() if "enroll_sos" not in n)
