"""CPU restatement of the UniSE AR-LM (decoder-only Llama-style LM with conditioning prefix).

TEST INFRASTRUCTURE - see oracle/__init__.py.  The reference's `CustomLlamaModel` cannot be constructed
under the installed transformers (U/model/llm/llm.py:79 `_update_causal_mask` no longer exists; SURVEY 7.6),
so its semantics are restated here and pinned against `transformers.LlamaModel` run in the build
container (oracle/make_golden_lm.py): with mask None + SDPA the reference's layers are plain causal
Llama decoder layers (llm.py:153 comment, :195-216).

Paths relative to /root/reference/QuarkAudio-UniSE/:
  model/llm/llm.py:40-83    vocab layout, embeddings, layers (hidden 512, 12 layers, 8 heads x 64, FFN 4*hidden
                            SwiGLU, RMSNorm eps 1e-6, RoPE theta 1e4, no biases), output_head
  model/llm/llm.py:150-228  llm_forward (causal stack on inputs_embeds, final norm, KV cache)
  model/llm/llm.py:87-104   label-smoothed KL loss
  model/llm/llm.py:253-289  sample_logits (greedy == arg-max of the range-masked logits)
  model/llm/llm_sft.py:29-33, 37-89, 93-195   task / sos embeddings, adapter, forward, generate
"""
from __future__ import annotations

import zlib
from collections import OrderedDict

import torch
import torch.nn.functional as F

LM_FULL = dict(num_tasks=3, task_map=dict(se=0, tse=1, rtse=2), feats_dim=768,
               llm_base_config=dict(cond_dim=80, global_size=4096, semantic_size=8192, hidden_size=512, num_layers=12,
                                    num_attention_heads=8, dropout_p=0.1, max_position_embeddings=4096,
                                    label_smoothing=0.1))


def lm_small(hidden=128, layers=2, heads=2, gsize=64, ssize=128, feats=64):
    return dict(num_tasks=3, task_map=dict(se=0, tse=1, rtse=2), feats_dim=feats,
                llm_base_config=dict(cond_dim=80, global_size=gsize, semantic_size=ssize, hidden_size=hidden,
                                     num_layers=layers, num_attention_heads=heads, dropout_p=0.1,
                                     max_position_embeddings=4096, label_smoothing=0.1))


def lm_param_specs(cfg):
    b = cfg["llm_base_config"]
    H, L = b["hidden_size"], b["num_layers"]
    V = 3 + b["global_size"] + b["semantic_size"]
    out = OrderedDict()
    out["mix_sos_embedding.weight"] = ((1, H), "emb")
    out["codec_embedding.weight"] = ((V, H), "emb")
    for i in range(L):
        p = f"layers.{i}."
        for n in "qkvo":
            out[p + f"self_attn.{n}_proj.weight"] = ((H, H), "w")
        out[p + "mlp.gate_proj.weight"] = ((4 * H, H), "w")
        out[p + "mlp.up_proj.weight"] = ((4 * H, H), "w")
        out[p + "mlp.down_proj.weight"] = ((H, 4 * H), "w")
        out[p + "input_layernorm.weight"] = ((H,), "norm")
        out[p + "post_attention_layernorm.weight"] = ((H,), "norm")
    out["norm.weight"] = ((H,), "norm")
    out["output_head.weight"] = ((V, H), "w")
    out["task_embedding.weight"] = ((cfg["num_tasks"], H), "emb")
    out["enroll_sos_embedding.weight"] = ((1, H), "emb")
    out["adapter.weight"] = ((H, cfg["feats_dim"]), "w")
    out["adapter.bias"] = ((H,), "b")
    return out


def make_lm_state_dict(cfg, seed=0, weight_gain=1.0):
    """Seeded weights; `weight_gain` > 1 sharpens the logits (HF default init std 0.02 gives
    near-uniform logits and therefore arg-max margins at the fp32 noise floor, SURVEY 8d)."""
    sd = OrderedDict()
    for name, (shape, kind) in lm_param_specs(cfg).items():
        g = torch.Generator()
        g.manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2**63 - 1))
        if kind == "w":
            sd[name] = torch.randn(shape, generator=g) * (weight_gain / shape[-1] ** 0.5)
        elif kind == "emb":
            sd[name] = torch.randn(shape, generator=g)
        elif kind == "norm":
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            sd[name] = 0.05 * torch.randn(shape, generator=g)
    return sd


def _rope(pos, head_dim, dtype, theta=10000.0):
    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).float() / head_dim))
    fr = pos.float()[:, None] * inv[None, :]
    emb = torch.cat((fr, fr), -1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def _rot(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), -1)


def llm_forward(sd, cfg, inputs_embeds, cache=None):
    """llm.py:150-228.  inputs_embeds [B,L,H]; cache = list of (k,v) [B,nh,T,hd] per layer or None.
    Returns (last_hidden_state [B,L,H], new_cache)."""
    b = cfg["llm_base_config"]
    H, nh = b["hidden_size"], b["num_attention_heads"]
    hd = H // nh
    x = inputs_embeds
    B, L, _ = x.shape
    past = 0 if cache is None else cache[0][0].shape[2]
    cos, sin = _rope(torch.arange(past, past + L), hd, x.dtype)
    new_cache = []
    for i in range(b["num_layers"]):
        p = f"layers.{i}."
        h = F.rms_norm(x, (H,), sd[p + "input_layernorm.weight"], 1e-6)
        q = F.linear(h, sd[p + "self_attn.q_proj.weight"]).view(B, L, nh, hd).transpose(1, 2)
        k = F.linear(h, sd[p + "self_attn.k_proj.weight"]).view(B, L, nh, hd).transpose(1, 2)
        v = F.linear(h, sd[p + "self_attn.v_proj.weight"]).view(B, L, nh, hd).transpose(1, 2)
        q = q * cos + _rot(q) * sin
        k = k * cos + _rot(k) * sin
        if cache is not None:
            k = torch.cat([cache[i][0], k], 2)
            v = torch.cat([cache[i][1], v], 2)
        new_cache.append((k, v))
        att = torch.matmul(q, k.transpose(2, 3)) * hd ** -0.5
        T = k.shape[2]
        mask = torch.ones(L, T, dtype=torch.bool).tril(diagonal=T - L)
        att = att.masked_fill(~mask, float("-inf"))
        att = torch.softmax(att, -1)
        o = torch.matmul(att, v).transpose(1, 2).reshape(B, L, H)
        x = x + F.linear(o, sd[p + "self_attn.o_proj.weight"])
        h = F.rms_norm(x, (H,), sd[p + "post_attention_layernorm.weight"], 1e-6)
        h = F.linear(F.silu(F.linear(h, sd[p + "mlp.gate_proj.weight"])) * F.linear(h, sd[p + "mlp.up_proj.weight"]),
                     sd[p + "mlp.down_proj.weight"])
        x = x + h
    return F.rms_norm(x, (H,), sd["norm.weight"], 1e-6), new_cache


def _prefix(sd, cfg, task_name, enroll_feats, mix_feats):
    """llm_sft.py:58-78 / 108-128: [task | (enroll_sos, enroll) | mix_sos, mix]."""
    B = mix_feats.shape[0]
    task = sd["task_embedding.weight"][cfg["task_map"][task_name]][None, None].expand(B, 1, -1)
    mix = F.linear(mix_feats, sd["adapter.weight"], sd["adapter.bias"])
    mix_sos = sd["mix_sos_embedding.weight"][0][None, None].expand(B, 1, -1)
    if enroll_feats is not None:
        enr = F.linear(enroll_feats, sd["adapter.weight"], sd["adapter.bias"])
        esos = sd["enroll_sos_embedding.weight"][0][None, None].expand(B, 1, -1)
        return torch.cat([task, esos, enr, mix_sos, mix], 1)
    return torch.cat([task, mix_sos, mix], 1)


@torch.no_grad()
def sft_forward(sd, cfg, task_name, enroll_feats, mix_feats, global_ids, semantic_ids, return_logits=False):
    """llm_sft.py:37-89 + llm.py:87-104 -> (loss, acc) [, logits]."""
    b = cfg["llm_base_config"]
    goff, soff = 3, 3 + b["global_size"]
    g = global_ids.long() + goff
    s = semantic_ids.long() + soff
    B = g.shape[0]
    col = lambda v: torch.full((B, 1), v, dtype=torch.long)
    input_ids = torch.cat([col(0), g, col(1), s], 1)
    target_ids = torch.cat([g, col(1), s, col(2)], 1)
    emb = torch.cat([_prefix(sd, cfg, task_name, enroll_feats, mix_feats), sd["codec_embedding.weight"][input_ids]], 1)
    hs, _ = llm_forward(sd, cfg, emb)
    hs = hs[:, -target_ids.shape[1]:]
    logits = F.linear(hs, sd["output_head.weight"])
    V = logits.shape[-1]
    ls = b["label_smoothing"]
    flat, tgt = logits.float().reshape(-1, V), target_ids.reshape(-1)
    true = torch.full_like(flat, ls / (V - 1))
    true.scatter_(1, tgt[:, None], 1.0 - ls)
    loss = F.kl_div(F.log_softmax(flat, -1), true, reduction="batchmean")
    acc = (logits.argmax(-1) == target_ids).float().mean()
    return (loss, acc, logits) if return_logits else (loss, acc)


@torch.no_grad()
def sft_generate(sd, cfg, task_name, enroll_feats, mix_feats, semantic_length, global_length=32, return_margins=False):
    """llm_sft.py:93-195 with do_sample=False (greedy, the shipped test setting model.py:173):
    arg-max of the logits restricted to the global / semantic token range."""
    b = cfg["llm_base_config"]
    goff, soff = 3, 3 + b["global_size"]
    hs, cache = llm_forward(sd, cfg, _prefix(sd, cfg, task_name, enroll_feats, mix_feats))
    B = mix_feats.shape[0]
    margins = []

    def run(first_id, steps, lo, hi):
        nonlocal cache
        ids = torch.full((B, 1), first_id, dtype=torch.long)
        out = []
        for _ in range(steps):
            h, cache = llm_forward(sd, cfg, sd["codec_embedding.weight"][ids], cache)
            logits = F.linear(h[:, 0], sd["output_head.weight"])[:, lo:hi]
            top2 = torch.topk(logits.double(), 2, -1).values
            margins.append((top2[:, 0] - top2[:, 1]) / logits.abs().max(-1).values.double())
            ids = logits.argmax(-1, keepdim=True) + lo
            out.append(ids)
        return out

    gout = run(0, global_length + 1, goff, goff + b["global_size"])
    global_ids = torch.cat(gout[:-1], -1) - goff
    sout = run(1, semantic_length, soff, soff + b["semantic_size"])
    semantic_ids = torch.cat(sout, -1) - soff
    if return_margins:
        return global_ids, semantic_ids, torch.stack(margins, 1)
    return global_ids, semantic_ids


# --------------------------------------------------------------------------- sampled decoding (llm.py:253-289)
def sample_filter(logits, temperature=0.8, top_k=50, top_p=0.95):
    """The reference's sample_logits up to (not including) the multinomial draw: returns the final probabilities
    [B, V'] (zeros where a token was filtered out).  Steps, in the reference's order: top-k by threshold value
    (`logits < topk[-1]` removed, ties at the k-th value stay) -> top-p on the descending sort of the survivors
    (a token goes when the cumulative softmax BEFORE it exceeds top_p; the first always stays) -> / temperature ->
    softmax."""
    logits = logits.clone().float()
    if top_k > 0:
        kth = torch.topk(logits, top_k)[0][..., -1, None]
        logits[logits < kth] = float("-inf")
    if top_p < 1.0:
        # stable: when the cut falls inside a run of equal logits, the lower token ids are the ones kept, the order the
        # device sampler defines (an unstable sort keeps an arbitrary subset of the run)
        sorted_logits, sorted_indices = torch.sort(logits, descending=True, stable=True)
        cum = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
        rem = cum > top_p
        rem[..., 1:] = rem[..., :-1].clone()
        rem[..., 0] = 0
        logits[rem.scatter(-1, sorted_indices, rem)] = float("-inf")
    assert 0 < temperature <= 1.0
    return F.softmax(logits / temperature, dim=-1)


def philox4x32_10(key, counter):
    """Philox-4x32 with 10 rounds (Salmon et al. 2011): key (k0, k1), counter (c0, c1, c2, c3) -> 4 uint32."""
    M0, M1, W0, W1, mask = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF
    k0, k1 = key
    c0, c1, c2, c3 = counter
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & mask, p1 & mask, ((p0 >> 32) ^ c3 ^ k1) & mask, p0 & mask
        k0, k1 = (k0 + W0) & mask, (k1 + W1) & mask
    return c0, c1, c2, c3


def sample_uniform(seed, call, step, row):
    """The uniform in [0,1) the device sampler uses for (generate call chunk, decode step, batch row):
    24 high bits of Philox4x32-10(key = seed split lo/hi, counter = {step, row, call, 0}).x (include/quark_b200.h)."""
    r = philox4x32_10((seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF), (step, row, call, 0))[0]
    return (r >> 8) / 16777216.0


def inverse_cdf_pick(probs_row, u):
    """Inverse-CDF draw over the kept tokens in descending-probability order (ties: ascending id), the order the device
    sampler defines.  Returns (token, distance of u*S to the nearest CDF boundary / S)."""
    idx = torch.nonzero(probs_row > 0).flatten()
    p = probs_row[idx].double()
    order = sorted(range(len(idx)), key=lambda i: (-float(p[i]), int(idx[i])))
    cdf = torch.cumsum(p[order], 0)
    t = u * float(cdf[-1])
    k = int(torch.searchsorted(cdf, torch.tensor(t, dtype=torch.float64), right=True))
    k = min(k, len(order) - 1)
    near = float((cdf - t).abs().min() / cdf[-1])
    return int(idx[order[k]]), near
