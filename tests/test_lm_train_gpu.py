"""Gradients of the UniSE LM's teacher-forced loss on the GPU (csrc/lm_train.cu + the 3-term split qb_gemm) against fp64.

Kernels one by one against fp64 torch autograd, then whole-model gradients against oracle/llama_train.py's fp64 autograd (the oracle is
pinned against the reference's own LLM_SFT.forward + backward by tests/test_lm_train_host.py), with and without attention dropout,
determinism, train vs eval, three AdamW steps through unise.Model.configure_optimizers, and the composed training_step."""
import pytest
import torch

from oracle import llama, llama_train

pytestmark = pytest.mark.gpu


def frob(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------------------------- kernels
def attention_fp64(qkv, B, L, heads, keep, p):
    """causal attention with RoPE as the LM runs it, fp64, differentiable in qkv"""
    H = heads * 64
    q, k, v = (qkv.view(B, L, 3, heads, 64)[:, :, i].transpose(1, 2) for i in range(3))
    cos, sin = llama._rope(torch.arange(L), 64, torch.float64)
    q, k = q * cos + llama._rot(q) * sin, k * cos + llama._rot(k) * sin
    s = (q @ k.transpose(2, 3)) / 8.0
    s = s.masked_fill(~torch.ones(L, L, dtype=torch.bool).tril(), float("-inf"))
    lse = torch.logsumexp(s, -1)
    a = torch.softmax(s, -1)
    if keep is not None:
        a = a * torch.as_tensor(keep).double() / (1 - p)
    return (a @ v).transpose(1, 2).reshape(B * L, H), lse.reshape(B * heads, L)


@pytest.mark.parametrize("L", [1, 45, 786])
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("scale", [1.0, 6.0])          # 6: scores of several tens, the range trained weights produce
def test_attention_train_vs_fp64(lib, L, p, scale):
    from unified_audio_b200 import ops
    B, heads, seed, layer = (1 if L == 786 else 2), 2, 1234567, 5
    H = heads * 64
    g = torch.Generator().manual_seed(L + int(10 * p))
    qkv = scale * torch.randn(B * L, 3 * H, generator=g)
    dout = torch.randn(B * L, H, generator=g)
    cos, sin = ops.rope_tables(max(L, 64), 64, "cuda")
    d = lambda *s: torch.empty(*s, device="cuda")
    qs, kr, v, o, lse = d(B * heads, L, 64), d(B * heads, L, 64), d(B * heads, L, 64), d(B * L, H), d(B * heads, L)
    ops.lm_attn_train_fwd(qkv.cuda(), B, L, heads, cos, sin, p, seed, layer, qs, kr, v, o, lse)
    dqkv = d(B * L, 3 * H)
    ops.lm_attn_train_bwd(qs, kr, v, o, dout.cuda(), lse, B, L, heads, cos, sin, p, seed, layer, dqkv, d(B * heads * L))
    keep = llama_train.dropout_keep(seed, layer, B, heads, L, p) if p > 0 else None
    x = qkv.double().requires_grad_(True)
    o64, lse64 = attention_fp64(x, B, L, heads, keep, p)
    o64.backward(dout.double())
    errs = dict(out=frob(o, o64.detach()), lse=frob(lse, lse64.detach()), dqkv=frob(dqkv, x.grad))
    print(f"L={L} p={p} scale={scale}", errs)
    assert errs["out"] < 2e-6 and errs["lse"] < 2e-6 and errs["dqkv"] < 2e-5, errs
    if p == 0:          # the training forward at p = 0 is the eval kernel to fp32 noise
        op = ops.Planes.zeros((B * L, H), True, "cuda")
        ws = torch.zeros(ops.attention_umma_workspace_bytes(B, L, heads, 64, True), dtype=torch.uint8, device="cuda")
        ops.attention_umma(qkv.cuda(), B, L, heads, 64, cos, sin, op, ws, split=True, causal=True)
        assert frob(op.float(), o) < 1e-5


def test_small_kernels_vs_fp64(lib):
    from unified_audio_b200 import ops
    g = torch.Generator().manual_seed(3)
    M, C, I, V = 300, 256, 384, 203
    # RMSNorm backward + the fixed-order column sum
    x, w, dy, dx0 = (torch.randn(M, C, generator=g) for _ in range(4))
    w = 1 + 0.1 * w[0]
    dx, gw, dw = dx0.cuda().clone(), torch.empty(M, C, device="cuda"), torch.empty(C, device="cuda")
    ops.rmsnorm_bwd(x.cuda(), w.cuda(), dy.cuda(), M, C, dx, gw, True)
    ops.col_sum(gw, M, C, C, dw)
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    torch.nn.functional.rms_norm(xd, (C,), wd, 1e-6).backward(dy.double())
    assert frob(dx, dx0.double() + xd.grad) < 1e-6 and frob(dw, wd.grad) < 1e-6
    # SwiGLU forward / backward over interleaved (gate, up) columns
    gu, dh = 3 * torch.randn(M, 2 * I, generator=g), torch.randn(M, I, generator=g)
    h, hp = torch.empty(M, I, device="cuda"), ops.Planes.zeros((M, I), True, "cuda")
    dgu, dp = torch.empty(M, 2 * I, device="cuda"), ops.Planes.zeros((M, 2 * I), True, "cuda")
    ops.swiglu(gu.cuda(), M, I, h, hp)
    ops.swiglu_bwd(gu.cuda(), dh.cuda(), M, I, dgu, dp)
    gud = gu.double().requires_grad_(True)
    hd = torch.nn.functional.silu(gud[:, 0::2]) * gud[:, 1::2]
    hd.backward(dh.double())
    assert frob(h, hd.detach()) < 1e-6 and frob(dgu, gud.grad) < 1e-6 and frob(dp.float(), gud.grad) < 1e-6
    # loss backward: label-smoothed KL (batchmean) w.r.t. the logits, scaled by the incoming gradient
    logits, tg = 4 * torch.randn(M, V, generator=g), torch.randint(0, V, (M,), generator=g)
    Vp = 256
    out, op = torch.empty(M, Vp, device="cuda"), ops.Planes.zeros((M, Vp), True, "cuda")
    scale = ops.lm_loss_scale(V)
    ops.lm_loss_bwd(logits.cuda(), V, M, V, tg.cuda(), 0.1, torch.tensor([0.7], device="cuda"), out, op, Vp, scale)
    out, opf = out / (M * scale), op.float() / (M * scale)
    ld = logits.double().requires_grad_(True)
    true = torch.full((M, V), 0.1 / (V - 1), dtype=torch.float64).scatter_(1, tg[:, None], 0.9)
    (0.7 * torch.nn.functional.kl_div(torch.log_softmax(ld, -1), true, reduction="batchmean")).backward()
    assert frob(out[:, :V], ld.grad) < 1e-6 and float(out[:, V:].abs().max()) == 0.0 and frob(opf[:, :V], ld.grad) < 1e-6


def test_embedding_and_weight_grad_vs_fp64(lib):
    from unified_audio_b200 import ops
    g = torch.Generator().manual_seed(4)
    B, P, Lt, H, V = 3, 5, 40, 128, 50
    L = P + Lt
    dx = torch.randn(B * L, H, generator=g)
    ids = torch.randint(0, V, (B, Lt), generator=g)
    ids[:, :10] = 7                                         # a repeated id
    out = torch.empty(V, H, device="cuda")
    ops.embedding_bwd(dx.cuda(), ids.cuda(), ids.numel(), Lt, L, P, H, V, out, scale=0.5)
    ref = torch.zeros(V, H, dtype=torch.float64).index_add_(0, ids.reshape(-1), dx.double().view(B, L, H)[:, P:].reshape(-1, H)) * 0.5
    assert frob(out, ref) < 1e-7
    # split-K weight gradient dW = dY^T X over 1000 tokens: one slice and several slices of 192 tokens agree with fp64
    T, n_out, n_in = 1000, 320, 192
    dy, x = torch.randn(T, n_out, generator=g), torch.randn(T, n_in, generator=g)
    ref = dy.double().T @ x.double()
    for ks in (1024, 192, None):
        w = ops.weight_grad(dy.cuda(), x.cuda(), T, n_out, n_in, torch.empty(n_out, n_in, device="cuda"), ks=ks)
        assert frob(w, ref) < 1e-5, ks            # fp32 accumulation over up to 1000 tokens


# ------------------------------------------------------------------------------------------------------------------- whole model
def make_face(cfg, sd, dropout_p=None):
    from unified_audio_b200.llm import LLM_SFT
    b = dict(cfg["llm_base_config"])
    if dropout_p is not None:
        b["dropout_p"] = dropout_p
    lm = LLM_SFT(num_tasks=cfg["num_tasks"], task_map=cfg["task_map"], feats_dim=cfg["feats_dim"], llm_base_config=b)
    lm.load_state_dict(sd, strict=True)
    return lm.cuda()


def lm_inputs(cfg, B, Tm, Te, Ts, seed):
    b = cfg["llm_base_config"]
    g = torch.Generator().manual_seed(seed)
    return dict(mix=torch.randn(B, Tm, cfg["feats_dim"], generator=g), enroll=torch.randn(B, Te, cfg["feats_dim"], generator=g),
                gids=torch.randint(0, b["global_size"], (B, 32), generator=g), sids=torch.randint(0, b["semantic_size"], (B, Ts), generator=g))


def face_grads(lm, task, x, seed):
    lm.zero_grad(set_to_none=True)
    enr = x["enroll"].cuda() if task == "tse" else None
    loss, acc = lm(task, enr, enr, None, x["mix"].cuda(), x["gids"].cuda(), x["sids"].cuda(), dropout_seed=seed)
    loss.backward()
    return loss.detach(), {n: p.grad for n, p in lm.named_parameters() if p.grad is not None}


def oracle_grads(cfg, sd, task, x, dtype, p, seed):
    osd = {k: v.to(dtype).requires_grad_(True) for k, v in sd.items()}
    loss, _ = llama_train.sft_forward(osd, cfg, task, x["enroll"] if task == "tse" else None, x["mix"], x["gids"], x["sids"],
                                      dropout_p=p, dropout_seed=seed)
    loss.backward()
    return loss.detach(), {n: t.grad for n, t in osd.items() if t.grad is not None}


# The bound: K times the gap between the oracle's own fp32 and fp64 gradients, measured on the CPU for the same tensor (floored at
# the median gap over all tensors, so that a tensor whose fp32 gradient happens to be unusually exact does not set a bound below the
# noise of fp32 arithmetic itself).
K = 10.0


def check_grads(cfg, sd, task, x, p, seed, train=True):
    lm = make_face(cfg, sd).requires_grad_(True)
    lm.train(train)
    loss, g = face_grads(lm, task, x, seed)
    l64, g64 = oracle_grads(cfg, sd, task, x, torch.float64, p, seed)
    _, g32 = oracle_grads(cfg, sd, task, x, torch.float32, p, seed)
    assert set(g) == set(g64), set(g) ^ set(g64)
    gaps = {n: frob(g32[n], g64[n]) for n in g64}
    floor = sorted(gaps.values())[len(gaps) // 2]
    worst = 0.0
    for n in g64:
        e, bound = frob(g[n], g64[n]), K * max(gaps[n], floor)
        print(f"{task} p={p} {n}: rel {e:.2e} (fp32 oracle gap {gaps[n]:.2e}, bound {bound:.2e})")
        assert e < bound, (n, e, bound)
        worst = max(worst, e / bound)
    assert abs(float(loss) - float(l64)) < 1e-5 * abs(float(l64))
    return worst


@pytest.mark.parametrize("task", ["se", "tse"])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_model_grads_small_vs_oracle(lib, task, p):
    cfg = llama.lm_small()
    cfg["llm_base_config"]["dropout_p"] = p
    sd = llama.make_lm_state_dict(cfg, 5, 4.0)
    check_grads(cfg, sd, task, lm_inputs(cfg, 2, 12, 7, 12, 21), p, 99, train=p > 0)


@pytest.mark.parametrize("task,Te", [("se", 0), ("tse", 250)])
def test_model_grads_shipped_widths_vs_oracle(lib, task, Te):
    """B = 1, 5 s of WavLM frames (250) and 249 semantic tokens: L = 535 for 'se', 786 for 'tse'; attention dropout 0.1"""
    cfg = llama.LM_FULL
    sd = llama.make_lm_state_dict(cfg, 7, 2.0)
    check_grads(cfg, sd, task, lm_inputs(cfg, 1, 250, max(Te, 1), 249, 8), 0.1, 2024)


def test_determinism_and_seed(lib):
    cfg = llama.lm_small()
    sd = llama.make_lm_state_dict(cfg, 5, 4.0)
    x = lm_inputs(cfg, 2, 12, 7, 12, 21)
    lm = make_face(cfg, sd).requires_grad_(True).train()
    l1, g1 = face_grads(lm, "tse", x, 11)
    l2, g2 = face_grads(lm, "tse", x, 11)
    assert torch.equal(l1, l2) and all(torch.equal(g1[n], g2[n]) for n in g1)
    l3, g3 = face_grads(lm, "tse", x, 12)
    assert not torch.equal(l1, l3) and not torch.equal(g1["layers.0.self_attn.v_proj.weight"], g3["layers.0.self_attn.v_proj.weight"])


def test_train_vs_eval(lib):
    cfg = llama.lm_small()
    sd = llama.make_lm_state_dict(cfg, 5, 4.0)
    x = lm_inputs(cfg, 2, 12, 7, 12, 21)
    lm = make_face(cfg, sd, dropout_p=0.0)
    args = ("tse", x["enroll"].cuda(), x["enroll"].cuda(), None, x["mix"].cuda(), x["gids"].cuda(), x["sids"].cuda())
    le, ae = lm(*args)                                  # eval: the inference path
    lm.requires_grad_(True).train()
    lt, at = lm(*args)
    assert lt.grad_fn is not None and abs(float(lt) - float(le)) < 1e-6 * abs(float(le)) and float(at) == float(ae)
    lt.backward()
    lm.eval().requires_grad_(False)
    le2, ae2 = lm(*args)                                # weights unchanged: bit-identical
    assert torch.equal(le, le2) and torch.equal(ae, ae2)


def test_three_adamw_steps_then_generate(lib):
    """configure_optimizers + clip_grad_norm_(5.0) for three steps on the face and on the fp64 oracle; generate afterwards must use the
    updated weights (the packed-weight cache is rebuilt when the parameters' version counters move)"""
    from unified_audio_b200.unise import Model
    cfg = llama.lm_small()
    sd = llama.make_lm_state_dict(cfg, 5, 4.0)
    x = lm_inputs(cfg, 2, 12, 7, 12, 21)
    # lr large enough that three steps change the greedy tokens
    conf = dict(opt=dict(lr=2e-2), sch=dict(warmup_steps=2, step_decay=0.99998, min_factor=0.02))
    lm = make_face(cfg, sd)
    before = lm.generate("tse", x["enroll"].cuda(), x["enroll"].cuda(), torch.zeros(2, 12, 80, device="cuda"), x["mix"].cuda(), do_sample=False)
    model = Model(conf, tokenizer=None, dnn=lm, semantic_model=None)
    [opt], [sch] = model.configure_optimizers()
    osd = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    oopt = torch.optim.AdamW(list(osd.values()), **conf["opt"])
    osch = torch.optim.lr_scheduler.LambdaLR(oopt, sch["scheduler"].lr_lambdas[0])
    lm.train()
    for step in range(3):
        opt.zero_grad(set_to_none=True)
        face_grads(lm, "tse", x, 100 + step)[0]
        torch.nn.utils.clip_grad_norm_(lm.parameters(), 5.0)
        opt.step()
        sch["scheduler"].step()
        oopt.zero_grad(set_to_none=True)
        loss, _ = llama_train.sft_forward(osd, cfg, "tse", x["enroll"], x["mix"], x["gids"], x["sids"], 0.1, 100 + step)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(list(osd.values()), 5.0)
        oopt.step()
        osch.step()
    lm.eval()
    worst = max(frob(p.detach(), osd[n].detach()) for n, p in lm.named_parameters())
    print("max relative parameter difference after 3 steps", worst)
    assert worst < 1e-3
    new_sd = {k: v.detach().float() for k, v in osd.items()}
    gg, ss = lm.generate("tse", x["enroll"].cuda(), x["enroll"].cuda(), torch.zeros(2, 12, 80, device="cuda"), x["mix"].cuda(), do_sample=False)
    go, so = llama.sft_generate(new_sd, cfg, "tse", x["enroll"], x["mix"], 12)
    assert torch.equal(gg.cpu(), go) and torch.equal(ss.cpu(), so)
    assert not (torch.equal(before[0], gg) and torch.equal(before[1], ss))


# ------------------------------------------------------------------------------------------------------------------- training_step
@pytest.mark.parametrize("mode", ["se", "tse"])
def test_training_step_small_composition(lib, mode):
    from test_unise_validation_gpu import build_small, capture_lm_inputs, small_batch, to_cuda
    model, z, o = build_small()
    batch = to_cuda(small_batch(mode, torch.from_numpy(z["e2e_wav"]), 60))
    frozen = {n: p.detach().clone() for n, p in list(model.tokenizer.named_parameters()) + list(model.semantic_model.named_parameters())}
    model.dnn.requires_grad_(True)
    seen = capture_lm_inputs(model)
    out = model.training_step(batch, 0, dropout_seed=77)
    assert set(out) == {"loss", "train_acc"} and out["loss"].grad_fn is not None and not model.dnn.training
    out["loss"].backward()
    assert all(p.grad is not None for n, p in model.dnn.named_parameters() if mode == "tse" or "enroll_sos" not in n)
    assert all(p.grad is None for p in list(model.tokenizer.parameters()) + list(model.semantic_model.parameters()))
    assert all(torch.equal(p, frozen[n]) for n, p in list(model.tokenizer.named_parameters()) + list(model.semantic_model.named_parameters()))
    kw = seen[-1]
    # the LM's loss on the captured inputs, from the fp64 oracle with the same dropout mask
    lcfg, lsd = o["lcfg"], o["lsd"]
    osd = {k: v.double() for k, v in lsd.items()}
    ef = kw["enroll_feats"].cpu().double() if kw["enroll_feats"] is not None else None
    l64, _ = llama_train.sft_forward(osd, lcfg, mode, ef, kw["mix_feats"].cpu().double(), kw["global_ids"].cpu(), kw["semantic_ids"].cpu(),
                                     dropout_p=lcfg["llm_base_config"]["dropout_p"], dropout_seed=77)
    assert abs(float(out["loss"]) - float(l64)) < 1e-5 * abs(float(l64))
