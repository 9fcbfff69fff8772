"""Differentiable CPU restatement of the UniSE AR-LM's teacher-forced loss, for checking gradients.

TEST INFRASTRUCTURE - see oracle/__init__.py.  oracle/llama.py's `sft_forward` runs under no_grad and casts the logits to fp32; this
one keeps the dtype of the state dict it is given (fp64 for a reference gradient) and builds an autograd graph, so `loss.backward()`
gives every parameter's gradient.  Attention dropout follows transformers' Llama attention in train mode (dropout on the softmax
output, before `@ V`, kept values scaled by 1 / (1 - p)) with the mask the library draws (include/quark_b200.h), restated in NumPy by
`dropout_keep`.  Pinned against the reference's own `LLM_SFT.forward` + `loss.backward()` by oracle/make_golden_lm_grads.py.
"""
from __future__ import annotations

import zlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle.llama import _prefix, _rope, _rot

_M0, _M1, _W0, _W1, _MASK = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF


def philox4x32_10_np(key, c0, c1, c2, c3):
    """oracle.llama.philox4x32_10 over NumPy arrays of counters (uint64 holding 32-bit values) -> 4 uint64 arrays"""
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) for c in (c0, c1, c2, c3))
    m = np.uint64(_MASK)
    for _ in range(10):
        p0, p1 = np.uint64(_M0) * c0, np.uint64(_M1) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & m, p1 & m, ((p0 >> np.uint64(32)) ^ c3 ^ k1) & m, p0 & m
        k0, k1 = (k0 + np.uint64(_W0)) & m, (k1 + np.uint64(_W1)) & m
    return c0, c1, c2, c3


def dropout_threshold(p: float) -> int:
    """the mask's 24-bit threshold: float32(p) * 2^24 (exact in a double) rounded to the nearest integer, ties to even.  The library
    receives p as a C float, so a Python double that float32 rounds (0.09, 0.058, 0.16, ...) can land one step away from round(p * 2^24)."""
    return int(np.rint(np.float64(np.float32(p)) * 2.0 ** 24))


def dropout_words(seed: int, layer: int, B: int, heads: int, L: int) -> np.ndarray:
    """uint64 [B, heads, L, L]: the 24-bit word of key j of query i, word (j & 3) of Philox4x32-10(key = seed lo / hi, counter = {i,
    j >> 2, b * heads + h, layer}) >> 8"""
    J4 = -(-L // 4)
    bh = np.arange(B * heads, dtype=np.uint64)[:, None, None]
    i = np.arange(L, dtype=np.uint64)[None, :, None]
    j4 = np.arange(J4, dtype=np.uint64)[None, None, :]
    shape = (B * heads, L, J4)
    words = philox4x32_10_np((seed & _MASK, (seed >> 32) & _MASK), np.broadcast_to(i, shape), np.broadcast_to(j4, shape),
                             np.broadcast_to(bh, shape), np.full(shape, layer & _MASK, dtype=np.uint64))
    r = np.stack(words, -1).reshape(B * heads, L, 4 * J4)[..., :L]
    return (r >> np.uint64(8)).reshape(B, heads, L, L)


def dropout_keep(seed: int, layer: int, B: int, heads: int, L: int, p: float) -> np.ndarray:
    """bool [B, heads, L, L]: key j of query i kept iff its dropout_words word >= dropout_threshold(p)"""
    return dropout_words(seed, layer, B, heads, L) >= np.uint64(dropout_threshold(p))


def llm_forward(sd, cfg, x, masks=None, p=0.0):
    """llm.py:150-228 without a cache, differentiable, in x's dtype; masks[layer] = bool [B, heads, L, L] keep mask or None"""
    b = cfg["llm_base_config"]
    H, nh = b["hidden_size"], b["num_attention_heads"]
    hd = H // nh
    B, L, _ = x.shape
    cos, sin = (t.to(x.device) for t in _rope(torch.arange(L), hd, x.dtype))
    causal = torch.ones(L, L, dtype=torch.bool, device=x.device).tril()
    for i in range(b["num_layers"]):
        pre = f"layers.{i}."
        h = F.rms_norm(x, (H,), sd[pre + "input_layernorm.weight"], 1e-6)
        q, k, v = (F.linear(h, sd[pre + f"self_attn.{n}_proj.weight"]).view(B, L, nh, hd).transpose(1, 2) for n in "qkv")
        q = q * cos + _rot(q) * sin
        k = k * cos + _rot(k) * sin
        att = torch.softmax((q @ k.transpose(2, 3) * hd ** -0.5).masked_fill(~causal, float("-inf")), -1)
        if masks is not None and masks[i] is not None:
            att = att * torch.as_tensor(masks[i]).to(att.device, att.dtype) / (1.0 - p)
        o = (att @ v).transpose(1, 2).reshape(B, L, H)
        x = x + F.linear(o, sd[pre + "self_attn.o_proj.weight"])
        h = F.rms_norm(x, (H,), sd[pre + "post_attention_layernorm.weight"], 1e-6)
        x = x + F.linear(F.silu(F.linear(h, sd[pre + "mlp.gate_proj.weight"])) * F.linear(h, sd[pre + "mlp.up_proj.weight"]),
                         sd[pre + "mlp.down_proj.weight"])
    return F.rms_norm(x, (H,), sd["norm.weight"], 1e-6)


def sft_forward(sd, cfg, task_name, enroll_feats, mix_feats, global_ids, semantic_ids, dropout_p=0.0, dropout_seed=None):
    """llm_sft.py:37-89 + llm.py:87-104 -> (loss, acc), differentiable and in the state dict's dtype.  With dropout_p > 0 every layer's
    attention uses dropout_keep(dropout_seed, layer, ...)."""
    b = cfg["llm_base_config"]
    goff, soff = 3, 3 + b["global_size"]
    g, s = global_ids.long() + goff, semantic_ids.long() + soff
    B = g.shape[0]
    col = lambda v: torch.full((B, 1), v, dtype=torch.long, device=g.device)
    input_ids = torch.cat([col(0), g, col(1), s], 1)
    target_ids = torch.cat([g, col(1), s, col(2)], 1)
    dt = sd["norm.weight"].dtype
    emb = torch.cat([_prefix(sd, cfg, task_name, None if enroll_feats is None else enroll_feats.to(dt), mix_feats.to(dt)),
                     sd["codec_embedding.weight"][input_ids]], 1)
    masks = None
    if dropout_p > 0:
        L = emb.shape[1]
        masks = [dropout_keep(dropout_seed, i, B, b["num_attention_heads"], L, dropout_p) for i in range(b["num_layers"])]
    hs = llm_forward(sd, cfg, emb, masks, dropout_p)[:, -target_ids.shape[1]:]
    logits = F.linear(hs, sd["output_head.weight"])
    V = logits.shape[-1]
    ls = b["label_smoothing"]
    flat, tgt = logits.reshape(-1, V), target_ids.reshape(-1)
    true = torch.full_like(flat, ls / (V - 1))
    true.scatter_(1, tgt[:, None], 1.0 - ls)
    loss = F.kl_div(F.log_softmax(flat, -1), true, reduction="batchmean")
    acc = (logits.argmax(-1) == target_ids).to(dt).mean()
    return loss, acc


SKETCH_FULL, SKETCH_DIM = 4096, 256


def grad_sketch(name: str, grad: torch.Tensor) -> torch.Tensor:
    """What the gradient fixture keeps of one gradient: the tensor itself (fp64, flattened) up to SKETCH_FULL elements, otherwise its
    SKETCH_DIM projections onto Gaussian vectors seeded by the parameter's name.  Projections preserve the Frobenius norm of a
    difference in expectation (Johnson-Lindenstrauss), so ||sketch(a) - sketch(b)|| / ||sketch(b)|| estimates the relative Frobenius
    error of a against b (to ~10 % at 256 projections) at a few KB per tensor."""
    g = grad.detach().double().reshape(-1).cpu()
    if g.numel() <= SKETCH_FULL:
        return g
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.randn(SKETCH_DIM, g.numel(), generator=gen, dtype=torch.float64) @ g / SKETCH_DIM ** 0.5
