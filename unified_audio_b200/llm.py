"""UniSE AR-LM (`LLM_SFT`) with the reference's surface, running on libquark_b200.

Mirrors QuarkAudio-UniSE/model/llm/llm_sft.py:13-195 and llm.py:13-228:
    LLM_SFT(num_tasks, task_map, feats_dim, llm_base_config)
    .llm_forward(inputs_embeds, past_key_values=None, use_cache=False) -> .last_hidden_state / .past_key_values
    .forward(task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, global_ids, semantic_ids) -> (loss, acc)
    .generate(task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, global_length=32, ..., do_sample) -> (global, semantic)
state_dict keys are the reference's (HF Llama layer names under `layers.*`, `norm.weight`, `codec_embedding`,
`output_head`, `adapter`, `task_embedding`, `enroll_sos_embedding`, `mix_sos_embedding`); the conformer
condition encoder (`cond_*`, built but never executed: llm_sft.py:62-65,112-115) is accepted at load and ignored.

Prefill / teacher-forced forward: wgmma GEMMs (3-term split) + causal split-precision flash attention over a static fp32 KV cache.
Decode: fused skinny kernels (3-term fp16-split mma.sync over pre-packed weights with the RMSNorm weights folded in,
programmatic dependent launch), captured in CUDA graphs and replayed for the 33 + T steps; greedy (do_sample=False, the shipped
setting U/model/model.py:173) or sampled on the device.  No PyTorch / CPU fallback for the transformer stack.
"""
from __future__ import annotations

import copy
import operator
from dataclasses import dataclass
import os
from typing import Optional

import torch

from . import ops
from .codec import _Face, _Tree, _pad_to
from .ops import ACT_SWIGLU, Planes, rowmap


def lm_spec(cfg_base: dict, num_tasks: int, feats_dim: int):
    H, L = cfg_base["hidden_size"], cfg_base["num_layers"]
    V = 3 + cfg_base["global_size"] + cfg_base["semantic_size"]
    out = {"mix_sos_embedding.weight": (1, H), "codec_embedding.weight": (V, H)}
    for i in range(L):
        p = f"layers.{i}."
        for n in "qkvo":
            out[p + f"self_attn.{n}_proj.weight"] = (H, H)
        out[p + "mlp.gate_proj.weight"] = (4 * H, H)
        out[p + "mlp.up_proj.weight"] = (4 * H, H)
        out[p + "mlp.down_proj.weight"] = (H, 4 * H)
        out[p + "input_layernorm.weight"] = (H,)
        out[p + "post_attention_layernorm.weight"] = (H,)
    out["norm.weight"] = (H,)
    out["output_head.weight"] = (V, H)
    out["task_embedding.weight"] = (num_tasks, H)
    out["enroll_sos_embedding.weight"] = (1, H)
    out["adapter.weight"] = (H, feats_dim)
    out["adapter.bias"] = (H,)
    return out


class StaticKVCache:
    """Pre-allocated fp32 cache [layers][B, heads, Lmax, 64]; replaces HF DynamicCache's torch.cat growth."""

    def __init__(self, layers, B, heads, Lmax, device):
        self.k = [torch.zeros(B, heads, Lmax, 64, dtype=torch.float32, device=device) for _ in range(layers)]
        self.v = [torch.zeros(B, heads, Lmax, 64, dtype=torch.float32, device=device) for _ in range(layers)]
        self.B, self.heads, self.layers, self.Lmax, self.length = B, heads, layers, Lmax, 0
        self.pos = torch.zeros(B, dtype=torch.int32, device=device)     # row b's position, read (and bumped) by the decode kernels

    def get_seq_length(self):
        return self.length

    def reserve(self, n_positions: int):
        """Make room for `n_positions` in total (HF DynamicCache grows without bound, llm.py:189-193): reallocate to the
        next multiple of 256 and copy the filled prefix.  Captured graphs never call this (their capacity is fixed)."""
        if n_positions <= self.Lmax:
            return
        new = -(-n_positions // 256) * 256
        for buf in (self.k, self.v):
            for i, t in enumerate(buf):
                g = torch.zeros(self.B, self.heads, new, 64, dtype=t.dtype, device=t.device)
                g[:, :, :self.length] = t[:, :, :self.length]
                buf[i] = g
        self.Lmax = new


@dataclass
class LMOutput:
    last_hidden_state: torch.Tensor
    past_key_values: Optional[StaticKVCache] = None


class LLM_SFT(_Face):
    _IGNORED_KEYS = ("cond_", "rotary_emb.")         # the conformer condition encoder is never executed

    def __init__(self, num_tasks: int = 1, task_map: dict = None, feats_dim: int = 768, llm_base_config: dict = None):
        super().__init__()
        b = dict(llm_base_config or {})
        self.cfg = b
        self.task_map = dict(task_map or {"se": 0})
        self.hidden, self.n_layers, self.heads = b["hidden_size"], b["num_layers"], b["num_attention_heads"]
        if self.hidden != self.heads * 64 or self.hidden % 128:
            raise ValueError("kernels assume head_dim 64 and hidden % 128 == 0 (shipped config: 512 = 8 x 64)")
        self.global_size, self.semantic_size = b["global_size"], b["semantic_size"]
        self.vocab_size = 3 + self.global_size + self.semantic_size
        self.global_offset, self.semantic_offset = 3, 3 + self.global_size
        self.global_sos_token_id, self.semantic_sos_token_id, self.semantic_eos_token_id = 0, 1, 2
        self.label_smoothing = b.get("label_smoothing", 0.1)
        self.max_pos = b.get("max_position_embeddings", 4096)
        tree = _Tree.build(lm_spec(b, num_tasks, feats_dim))
        for name, child in tree.named_children():
            self.add_module(name, child)
        self.graph_steps = int(os.environ.get("QB_LM_GRAPH_STEPS", "8"))     # decode steps per replayed CUDA graph
        self._gen_state = {}
        # generate() walks a batch in chunks of <= `chunk` sequences; `lanes` > 1 runs that many chunks CONCURRENTLY, each on its own
        # CUDA stream with its own KV cache / workspace / captured graphs (the decode step is a chain of ~62 short dependent kernels:
        # one chain leaves most of the GPU idle, independent chains fill it).  Tokens do not depend on either setting.
        # A chain costs about the same for 8, 16 or 32 rows, so a batch of <= 32 is not cut into smaller chunks: chunk = 32.
        self.lanes = max(1, int(os.environ.get("QB_LM_LANES", "4")))
        # K / V rows a lane of the decode attention keeps in flight: 8 for one chain (latency-bound), 4 on concurrent lanes
        # (throughput-bound); QB_LM_ATT_U pins it.  Fixed per decode state (it is baked into the captured graphs).
        self.att_unroll = int(os.environ.get("QB_LM_ATT_U", "8"))
        self.lane_att_unroll = int(os.environ.get("QB_LM_ATT_U", "4"))
        self.chunk = min(32, max(1, int(os.environ.get("QB_LM_CHUNK", "32"))))
        self._lane_views = None
        self.eval()

    # ------------------------------------------------------------------ state
    def _drop_prepared(self):
        super()._drop_prepared()
        self._gen_state, self._lane_views = {}, None          # captured graphs point into the dropped weights and workspace

    def _param_versions(self):
        """(version counter, storage) of every parameter: an optimizer step changes them in place, which bumps the counters"""
        return tuple((p._version, p.data_ptr()) for p in self.parameters())

    def _prepare(self):
        if self._w is not None and self._w["versions"] == self._param_versions():
            return self._w
        if self._w is not None:
            self._drop_prepared()                  # the parameters changed in place since the weights were packed
        self._require_cuda()
        versions = self._param_versions()
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        layers = []
        for i in range(self.n_layers):
            p = f"layers.{i}."
            wqkv = torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0).contiguous()
            wg, wu = sd[p + "mlp.gate_proj.weight"].contiguous(), sd[p + "mlp.up_proj.weight"].contiguous()
            in_w, post_w = sd[p + "input_layernorm.weight"].contiguous(), sd[p + "post_attention_layernorm.weight"].contiguous()
            layers.append(dict(
                in_w=in_w, post_w=post_w,
                wqkv=Planes.from_f32(wqkv, True), wo=Planes.from_f32(sd[p + "self_attn.o_proj.weight"], True),
                wgu=Planes.from_f32(torch.stack([wg, wu], 1).reshape(-1, self.hidden), True),
                wd=Planes.from_f32(sd[p + "mlp.down_proj.weight"], True),
                # decode path: the preceding RMSNorm weight folded in (W' = W diag(g)), packed as fp16 {hi[4], lo[4]} groups
                wqkv_p=ops.lm_pack_weight(wqkv * in_w[None, :]),
                wo_p=ops.lm_pack_weight(sd[p + "self_attn.o_proj.weight"]),
                wg_p=ops.lm_pack_weight(wg * post_w[None, :]),
                wu_p=ops.lm_pack_weight(wu * post_w[None, :]),
                wd_p=ops.lm_pack_weight(sd[p + "mlp.down_proj.weight"])))
        self._w = dict(layers=layers, norm=sd["norm.weight"].contiguous(), head=Planes.from_f32(sd["output_head.weight"], True),
                       head_p=ops.lm_pack_weight(sd["output_head.weight"] * sd["norm.weight"][None, :]),
                       emb=sd["codec_embedding.weight"].contiguous(),
                       adapter=ops.pad_k_planes(sd["adapter.weight"], _pad_to(sd["adapter.weight"].shape[1], 64)),
                       adapter_b=sd["adapter.bias"].contiguous(), cos=None, sin=None, rope_rows=0, versions=versions)
        self._ensure_rope(self.max_pos)
        return self._w

    def _ensure_rope(self, n_positions: int):
        """cos/sin tables cover positions [0, rope_rows).  The reference's HF rotary embedding computes them from position_ids
        on the fly and has no length limit (llm.py:187), so the table grows on demand (the kernels index it unguarded:
        every caller checks pos0 + L against it first).  Growing replaces the tensors, so captured decode graphs that hold
        the old pointers are dropped."""
        W = self._w
        if W["rope_rows"] >= n_positions:
            return
        rows = max(self.max_pos, -(-n_positions // 1024) * 1024)
        W["cos"], W["sin"] = ops.rope_tables(rows, 64, self._dev())
        W["rope_rows"] = rows
        self._gen_state = {}

    # ------------------------------------------------------------------ transformer stack
    def _prefill(self, x: torch.Tensor, B: int, L: int, cache: StaticKVCache):
        """x [B*L, hidden] fp32, updated in place by the 12 layers; K/V written at cache.length..  cache None = a teacher-forced
        forward that nobody will decode from: no KV cache is allocated or written."""
        W = self._prepare()
        H, heads, inter, M = self.hidden, self.heads, 4 * self.hidden, B * L
        pos0 = cache.length if cache is not None else 0
        if cache is not None:
            if pos0 + L > cache.Lmax:
                raise ValueError("KV cache too small")
            if cache.B != B or cache.heads != heads or cache.layers != self.n_layers:
                raise ValueError(f"KV cache built for batch {cache.B} x {cache.heads} heads x {cache.layers} layers, "
                                 f"got batch {B} x {heads} heads x {self.n_layers} layers")
        self._ensure_rope(pos0 + L)
        W = self._w
        t1 = self._planes("t1", (M, H))
        hid = self._planes("hid", (M, inter))
        qkv = self._buf("qkv", (M, 3 * H))
        q16 = self._buf("q32", (B, heads, L, 64)) if cache is not None else None
        xm = rowmap(x, H, M, 0)
        lin = lambda a, w, n, K, **kw: ops.gemm(a, w, n, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, **kw)
        # a prefill from an empty cache (every call of llm_forward / forward / generate) attends within its own L positions: the causal
        # wgmma attention (csrc/attention_umma.cu) reads the qkv GEMM's output directly; lm_qkv_prep still fills the fp32 KV cache for
        # the decode steps.  A continuation (pos0 > 0) keeps the cache-reading mma.sync kernel.
        umma = pos0 == 0
        att_ws = self._buf("att5_ws", (ops.attention_umma_workspace_bytes(B, L, heads, 64, True),), torch.uint8) if umma else None
        for i, Lw in enumerate(W["layers"]):
            ops.rmsnorm(x, Lw["in_w"], M, H, t1)
            lin(t1, Lw["wqkv"], 3 * H, H, out_f32=rowmap(qkv, 3 * H, M, 0))
            if cache is not None:
                ops.lm_qkv_prep(qkv, B, L, heads, pos0, W["cos"], W["sin"], q16, cache.k[i], cache.v[i], cache.Lmax)
            if umma:
                ops.attention_umma(qkv, B, L, heads, 64, W["cos"], W["sin"], t1, att_ws, split=True, causal=True)
            else:
                ops.lm_flash_attn(q16, cache.k[i], cache.v[i], B, L, heads, pos0, cache.Lmax, t1)
            lin(t1, Lw["wo"], H, H, residual=xm, out_f32=xm)
            ops.rmsnorm(x, Lw["post_w"], M, H, t1)
            lin(t1, Lw["wgu"], 2 * inter, H, act=ACT_SWIGLU, out_planes=hid, out_planes_map=(inter, M, 0))
            lin(hid, Lw["wd"], H, inter, residual=xm, out_f32=xm)
        if cache is not None:
            cache.length = pos0 + L
            cache.pos.fill_(cache.length)

    def _decode_layers(self, x: torch.Tensor, B: int, cache: StaticKVCache):
        W = self._prepare()
        ops.lm_set_att_unroll(self.att_unroll)
        H, heads, inter = self.hidden, self.heads, 4 * self.hidden
        qb, ab, mb = self._buf("dq", (B, H)), self._buf("da", (B, H)), self._buf("dm", (B, inter))
        for i, Lw in enumerate(W["layers"]):
            ops.lm_decode_layer_tc(x, B, H, heads, inter, Lw, cache.k[i], cache.v[i], cache.Lmax, cache.pos, W["cos"], W["sin"], qb, ab, mb)

    @torch.no_grad()
    def llm_forward(self, inputs_embeds, attention_mask=None, past_key_values: Optional[StaticKVCache] = None,
                    use_cache: bool = False, max_new_tokens: Optional[int] = None, **unused) -> LMOutput:
        """llm.py:150-228 (mask None + SDPA == causal).  `max_new_tokens` (optional) sizes a newly created cache; a cache
        that fills up is grown (reallocate + copy) like the reference's DynamicCache."""
        if attention_mask is not None:
            raise NotImplementedError("only the reference's causal (mask=None) path is implemented")
        W = self._prepare()
        B, L, H = inputs_embeds.shape
        cache = past_key_values
        if cache is None and not use_cache:
            # teacher-forced forward (LLM_SFT.forward, llm_sft.py:93-135): nothing decodes from it, so no KV cache at all
            self._ensure_rope(L)
            x = inputs_embeds.float().reshape(B * L, H).contiguous().clone()
            self._prefill(x, B, L, None)
            out = torch.empty(B * L, H, device=x.device)
            ops.rmsnorm(x, self._w["norm"], B * L, H, out_f32=out)
            return LMOutput(out.reshape(B, L, H), None)
        if cache is None:
            extra = (max_new_tokens if max_new_tokens is not None else 1024) if use_cache else 0
            cache = StaticKVCache(self.n_layers, B, self.heads, max(64, -(-(L + extra) // 64) * 64), self._dev())
        if cache.B != B or cache.heads != self.heads or cache.layers != self.n_layers:
            raise ValueError(f"KV cache built for batch {cache.B} x {cache.heads} heads x {cache.layers} layers, "
                             f"got batch {B} x {self.heads} heads x {self.n_layers} layers")
        cache.reserve(cache.length + L)
        self._ensure_rope(cache.length + L)
        W = self._w
        x = inputs_embeds.float().reshape(B * L, H).contiguous().clone()
        if L == 1 and B <= 32 and cache.length > 0:
            self._decode_layers(x, B, cache)
            cache.length += 1
            cache.pos.fill_(cache.length)
        else:
            self._prefill(x, B, L, cache)
        out = torch.empty(B * L, H, device=x.device)
        ops.rmsnorm(x, W["norm"], B * L, H, out_f32=out)
        return LMOutput(out.reshape(B, L, H), cache if use_cache else None)

    # ------------------------------------------------------------------ conditioning prefix (llm_sft.py:58-78)
    def _adapter(self, feats):
        W = self._prepare()
        B, T, Fd = feats.shape
        if Fd != self.adapter.weight.shape[1]:
            raise ValueError(f"features have {Fd} channels, the adapter takes {self.adapter.weight.shape[1]}")
        fpad = W["adapter"].hi.shape[1]
        a = Planes.zeros((B * T, fpad), True, feats.device)
        ops.rows_to_planes(feats.float().contiguous(), 1, B * T, Fd, a, fpad, B * T, 0)
        out = torch.empty(B * T, self.hidden, device=feats.device)
        ops.gemm(a, W["adapter"], self.hidden, a_batch=1, a_rows_per_batch=B * T, a_ld=fpad, m_per_batch=B * T, bias=W["adapter_b"],
                 out_f32=rowmap(out, self.hidden, B * T, 0))
        return out.reshape(B, T, self.hidden)

    def _prefix(self, task_name, enroll_feats, mix_feats, enroll_lengths=None):
        """[B, P, hidden]: task, (enroll_sos, adapter(enroll)), mix_sos, adapter(mix).  With `enroll_lengths` (host ints, one per row
        of a right-padded enroll_feats) row b keeps only its first enroll_lengths[b] enrollment frames, so that its own prefix of
        P_b = 3 + enroll_lengths[b] + T_mix positions has no padding inside it; zero rows fill positions P_b..P, P = the padded width."""
        if enroll_lengths is not None:
            return self._ragged_prefix(self._prefix(task_name, enroll_feats, mix_feats), enroll_lengths, enroll_feats.shape[1])
        B = mix_feats.shape[0]
        e = lambda w: w.detach().float()
        task = e(self.task_embedding.weight)[self.task_map[task_name]][None, None].expand(B, 1, -1)
        mix_sos = e(self.mix_sos_embedding.weight)[0][None, None].expand(B, 1, -1)
        parts = [task]
        if enroll_feats is not None:
            parts += [e(self.enroll_sos_embedding.weight)[0][None, None].expand(B, 1, -1), self._adapter(enroll_feats)]
        parts += [mix_sos, self._adapter(mix_feats)]
        return torch.cat(parts, 1)

    @staticmethod
    def _ragged_prefix(prefix, lengths, te_max):
        """uniform prefix [B, P, H] = task, enroll_sos, enroll (te_max), mix_sos, mix -> row b moves its mix_sos + mix up to
        right after its own lengths[b] enrollment frames; the positions after them gather a zero row"""
        B, P, H = prefix.shape
        idx = torch.full((B, P), P, dtype=torch.long)
        for b, n in enumerate(lengths):
            idx[b, :2 + n] = torch.arange(2 + n)
            idx[b, 2 + n:P - (te_max - n)] = torch.arange(2 + te_max, P)
        z = torch.cat([prefix, prefix.new_zeros(B, 1, H)], 1)
        return torch.gather(z, 1, idx.to(prefix.device)[..., None].expand(B, P, H))

    # ------------------------------------------------------------------ teacher-forced forward (llm_sft.py:37-89)
    def _ids(self, global_ids, semantic_ids):
        g = global_ids.long() + self.global_offset
        s = semantic_ids.long() + self.semantic_offset
        B = g.shape[0]
        col = lambda v: torch.full((B, 1), v, dtype=torch.long, device=g.device)
        return torch.cat([col(0), g, col(1), s], 1), torch.cat([g, col(1), s, col(2)], 1)

    def forward(self, task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, global_ids, semantic_ids, return_logits=False,
                dropout_seed: Optional[int] = None):
        """llm_sft.py:37-89 -> (loss, acc[, logits]).  In eval mode with no parameter requiring grad: the inference path (no autograd).
        In train mode, or when grad mode is on and the parameters require grad: the training path, whose loss has a grad_fn
        (`loss.backward()` accumulates fp32 gradients into every parameter's .grad) and which applies attention dropout with
        probability llm_base_config["dropout_p"] in train mode (mask: include/quark_b200.h, from `dropout_seed`, default a draw of
        torch's CPU generator).  No gradient flows into enroll_feats / mix_feats (the reference detaches them, model.py:37-51)."""
        if self.training or (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())):
            return self._train_forward(task_name, enroll_feats if enroll_mel is not None else None, mix_feats, global_ids, semantic_ids,
                                       return_logits, dropout_seed)
        with torch.no_grad():
            return self._eval_forward(task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, global_ids, semantic_ids, return_logits)

    def _eval_forward(self, task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, global_ids, semantic_ids, return_logits=False):
        W = self._prepare()
        input_ids, target_ids = self._ids(global_ids, semantic_ids)
        B = input_ids.shape[0]
        emb = torch.cat([self._prefix(task_name, enroll_feats if enroll_mel is not None else None, mix_feats),
                         W["emb"][input_ids]], 1)
        hs = self.llm_forward(emb).last_hidden_state[:, -target_ids.shape[1]:].contiguous()
        Lt, V = hs.shape[1], self.vocab_size
        M = B * Lt
        hp = Planes.zeros((M, self.hidden), True, hs.device)
        ops.split_f16(hs.reshape(M, self.hidden), hp)
        vpad = (V + 3) // 4 * 4
        logits = torch.empty(M, vpad, device=hs.device)
        ops.gemm(hp, W["head"], V, a_batch=1, a_rows_per_batch=M, a_ld=self.hidden, m_per_batch=M,
                 out_f32=rowmap(logits, vpad, M, 0))
        # label-smoothed KL + accuracy (llm.py:87-104) in one pass over the produced logits (csrc/llm.cu lm_loss_*)
        la = ops.lm_loss(logits, vpad, M, V, target_ids.reshape(-1).contiguous(), self.label_smoothing)
        loss, acc = la[0], la[1]
        if return_logits:
            logits = logits[:, :V].reshape(B, Lt, V)
        return (loss, acc, logits) if return_logits else (loss, acc)

    # ------------------------------------------------------------------ training path: forward that keeps activations, backward
    def _train_forward(self, task_name, enroll_feats, mix_feats, global_ids, semantic_ids, return_logits, dropout_seed):
        self._require_cuda()
        if dropout_seed is None:
            dropout_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        input_ids, target_ids = self._ids(global_ids, semantic_ids)
        run = dict(task=task_name, enroll=None if enroll_feats is None else enroll_feats.detach().float().contiguous(),
                   mix=mix_feats.detach().float().contiguous(), input_ids=input_ids.contiguous(),
                   targets=target_ids.reshape(-1).contiguous(), seed=int(dropout_seed),
                   p=float(self.cfg.get("dropout_p", 0.1)) if self.training else 0.0)
        names = list(dict(self.named_parameters()))
        loss, acc, logits = _LMLoss.apply(self, run, names, *[p for _, p in self.named_parameters()])
        if return_logits:
            B, Lt = input_ids.shape
            return loss, acc, logits[:, :self.vocab_size].reshape(B, Lt, self.vocab_size)
        return loss, acc

    def _train_rope(self, L):
        rows = max(self.max_pos, -(-L // 1024) * 1024)
        return self._cached(("train_rope", rows), lambda: ops.rope_tables(rows, 64, self._dev()))

    @staticmethod
    def _split(w: torch.Tensor) -> Planes:
        """live fp32 parameter [n, k] -> hi / lo planes (k padded with zeros to a multiple of 64)"""
        n, k = w.shape
        kp = _pad_to(k, 64)
        out = Planes(torch.empty(n, kp, dtype=torch.float16, device=w.device), torch.empty(n, kp, dtype=torch.float16, device=w.device))
        if kp == k:
            ops.split_f16(w, out)
        else:
            ops.rows_to_planes(w, 1, n, k, out, kp, n, 0)
        return out

    @staticmethod
    def _transposed(w: torch.Tensor) -> Planes:
        """live fp32 parameter [n, k] -> planes of W^T [k, pad64(n)]: the weight operand of the data gradient dX = dY W"""
        t = ops.transpose_split(w, w.shape[0], w.shape[1], _pad_to(w.shape[0], 64))
        return Planes(t.hi[0], t.lo[0])

    def _train_fwd(self, run, prm):
        H, heads, I, nl = self.hidden, self.heads, 4 * self.hidden, self.n_layers
        mix, enr = run["mix"], run["enroll"]
        B, Tm, Fd = mix.shape
        if Fd != self.adapter.weight.shape[1]:
            raise ValueError(f"features have {Fd} channels, the adapter takes {self.adapter.weight.shape[1]}")
        if enr is not None and enr.shape[0] != B:
            raise ValueError(f"enroll_feats has {enr.shape[0]} rows, mix_feats {B}")
        Te = 0 if enr is None else enr.shape[1]
        dev = mix.device
        feats = mix.reshape(-1, Fd) if enr is None else torch.cat([enr.reshape(-1, Fd), mix.reshape(-1, Fd)], 0)
        Nf = feats.shape[0]
        fa = self._split(feats)
        ad = torch.empty(Nf, H, device=dev)
        ops.gemm(fa, self._split(prm["adapter.weight"]), H, a_batch=1, a_rows_per_batch=Nf, a_ld=fa.hi.shape[1], m_per_batch=Nf,
                 bias=prm["adapter.bias"], out_f32=rowmap(ad, H, Nf, 0))
        row = lambda w: w[None, None].expand(B, 1, H)
        parts = [row(prm["task_embedding.weight"][self.task_map[run["task"]]])]
        if enr is not None:
            parts += [row(prm["enroll_sos_embedding.weight"][0]), ad[:B * Te].reshape(B, Te, H)]
        parts += [row(prm["mix_sos_embedding.weight"][0]), ad[B * Te:].reshape(B, Tm, H)]
        P = 2 + Tm + (1 + Te if enr is not None else 0)
        ids = run["input_ids"]
        Lt = ids.shape[1]
        L, M, Mt = P + Lt, B * (P + Lt), B * Lt
        x = torch.cat(parts + [prm["codec_embedding.weight"][ids]], 1).reshape(M, H).contiguous()
        cos, sin = self._train_rope(L)
        t1 = Planes(torch.empty(M, H, dtype=torch.float16, device=dev), torch.empty(M, H, dtype=torch.float16, device=dev))
        hp = Planes(torch.empty(M, I, dtype=torch.float16, device=dev), torch.empty(M, I, dtype=torch.float16, device=dev))
        qkv = torch.empty(M, 3 * H, device=dev)
        lin = lambda a, w, n, K, **kw: ops.gemm(a, w, n, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, **kw)
        xm = rowmap(x, H, M, 0)
        saved = []
        for i in range(nl):
            p = f"layers.{i}."
            s = dict(x=x.clone())
            ops.rmsnorm(x, prm[p + "input_layernorm.weight"], M, H, t1)
            wqkv = torch.cat([prm[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0)
            lin(t1, self._split(wqkv), 3 * H, H, out_f32=rowmap(qkv, 3 * H, M, 0))
            s.update(qs=torch.empty(B * heads, L, 64, device=dev), kr=torch.empty(B * heads, L, 64, device=dev),
                     v=torch.empty(B * heads, L, 64, device=dev), o=torch.empty(M, H, device=dev), lse=torch.empty(B * heads, L, device=dev))
            ops.lm_attn_train_fwd(qkv, B, L, heads, cos, sin, run["p"], run["seed"], i, s["qs"], s["kr"], s["v"], s["o"], s["lse"])
            ops.split_f16(s["o"], t1)
            lin(t1, self._split(prm[p + "self_attn.o_proj.weight"]), H, H, residual=xm, out_f32=xm)
            s["xm"] = x.clone()
            ops.rmsnorm(x, prm[p + "post_attention_layernorm.weight"], M, H, t1)
            wgu = torch.stack([prm[p + "mlp.gate_proj.weight"], prm[p + "mlp.up_proj.weight"]], 1).reshape(2 * I, H)
            s["gu"], s["h"] = torch.empty(M, 2 * I, device=dev), torch.empty(M, I, device=dev)
            lin(t1, self._split(wgu), 2 * I, H, out_f32=rowmap(s["gu"], 2 * I, M, 0))
            ops.swiglu(s["gu"], M, I, s["h"], hp)
            lin(hp, self._split(prm[p + "mlp.down_proj.weight"]), H, I, residual=xm, out_f32=xm)
            saved.append(s)
        hs = torch.empty(M, H, device=dev)
        ops.rmsnorm(x, prm["norm.weight"], M, H, out_f32=hs)
        hst = hs.reshape(B, L, H)[:, P:].reshape(Mt, H).contiguous()
        V = self.vocab_size
        vpad = (V + 3) // 4 * 4
        logits = torch.empty(Mt, vpad, device=dev)
        lin_t = self._split(hst)
        ops.gemm(lin_t, self._split(prm["output_head.weight"]), V, a_batch=1, a_rows_per_batch=Mt, a_ld=H, m_per_batch=Mt,
                 out_f32=rowmap(logits, vpad, Mt, 0))
        la = ops.lm_loss(logits, vpad, Mt, V, run["targets"], self.label_smoothing)
        ctx = dict(layers=saved, xL=x, hst=hst, logits=logits, feats=feats, B=B, L=L, P=P, Lt=Lt, Te=Te, Tm=Tm)
        return la[0], la[1], logits, ctx

    def _train_bwd(self, run, prm, sv, grad_loss):
        H, heads, I, nl, V = self.hidden, self.heads, 4 * self.hidden, self.n_layers, self.vocab_size
        B, L, P, Lt, Te, Tm = (sv[k] for k in ("B", "L", "P", "Lt", "Te", "Tm"))
        M, Mt = B * L, B * Lt
        dev = grad_loss.device
        cos, sin = self._train_rope(L)
        g = {}
        # head + loss: dlogits once, as fp32 rows (for dW) and planes (for dX), written times Mt * scale (qb_lm_loss_bwd: its ~1/V
        # entries stay out of fp16's subnormal range).  The head's data-gradient GEMM takes `scale` back out (gamma, a power of two), so
        # the rest of the backward pass runs in units of Mt, where a row's gradients are O(1) in fp16 planes; every parameter gradient
        # is written times `unscale`.  The pass runs for a unit loss gradient: grad_loss (a loss weight, 1 / N of an accumulation, a
        # GradScaler's 2^16) multiplies the finished gradients, so the planes never see it and (c * loss).backward() is c times the
        # gradient for any c.
        Vp = _pad_to(V, 64)
        scale = ops.lm_loss_scale(V)
        unscale = 1.0 / Mt
        dlog = torch.empty(Mt, Vp, device=dev)
        dlp = Planes(torch.empty(Mt, Vp, dtype=torch.float16, device=dev), torch.empty(Mt, Vp, dtype=torch.float16, device=dev))
        ops.lm_loss_bwd(sv["logits"], sv["logits"].shape[1], Mt, V, run["targets"], self.label_smoothing,
                        self._cached(("unit_grad", dev), lambda: torch.ones(1, device=dev)), dlog, dlp, Vp, scale)
        g["output_head.weight"] = ops.weight_grad(dlog, sv["hst"], Mt, V, H, torch.empty(V, H, device=dev), dy_ld=Vp,
                                                  scale=unscale / scale)
        dhs = torch.zeros(M, H, device=dev)
        ops.gemm(dlp, self._transposed(prm["output_head.weight"]), H, a_batch=B, a_rows_per_batch=Lt, a_ld=Vp, m_per_batch=Lt,
                 gamma=torch.full((H,), 1.0 / scale, device=dev), out_f32=rowmap(dhs, H, L, P))
        dx, gw = torch.empty(M, H, device=dev), torch.empty(M, H, device=dev)
        nrm = torch.empty(M, H, device=dev)

        def norm_bwd(x, name, dy, accumulate):
            ops.rmsnorm_bwd(x, prm[name], dy, M, H, dx, gw, accumulate)
            g[name] = torch.empty(H, device=dev)
            ops.col_sum(gw, M, H, H, g[name], scale=unscale)

        def planes(t):
            out = Planes(torch.empty(t.shape, dtype=torch.float16, device=dev), torch.empty(t.shape, dtype=torch.float16, device=dev))
            ops.split_f16(t, out)
            return out

        lin = lambda a, w, n, K, out: ops.gemm(a, w, n, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, out_f32=rowmap(out, n, M, 0))
        norm_bwd(sv["xL"], "norm.weight", dhs, False)
        for i in reversed(range(nl)):
            p, s = f"layers.{i}.", sv["layers"][i]
            # MLP: x_out = xm + down(swiglu(gate_up(rmsnorm(xm))))
            g[p + "mlp.down_proj.weight"] = ops.weight_grad(dx, s["h"], M, H, I, torch.empty(H, I, device=dev), scale=unscale)
            dh = torch.empty(M, I, device=dev)
            lin(planes(dx), self._transposed(prm[p + "mlp.down_proj.weight"]), I, H, dh)
            dgu = torch.empty(M, 2 * I, device=dev)
            dgp = Planes(torch.empty(M, 2 * I, dtype=torch.float16, device=dev), torch.empty(M, 2 * I, dtype=torch.float16, device=dev))
            ops.swiglu_bwd(s["gu"], dh, M, I, dgu, dgp)
            del dh
            ops.rmsnorm(s["xm"], prm[p + "post_attention_layernorm.weight"], M, H, out_f32=nrm)
            ggu = ops.weight_grad(dgu, nrm, M, 2 * I, H, torch.empty(2 * I, H, device=dev), scale=unscale)
            g[p + "mlp.gate_proj.weight"], g[p + "mlp.up_proj.weight"] = ggu[0::2].contiguous(), ggu[1::2].contiguous()
            wgu = torch.stack([prm[p + "mlp.gate_proj.weight"], prm[p + "mlp.up_proj.weight"]], 1).reshape(2 * I, H)
            dn = torch.empty(M, H, device=dev)
            lin(dgp, self._transposed(wgu), H, 2 * I, dn)
            del dgu, dgp
            norm_bwd(s["xm"], p + "post_attention_layernorm.weight", dn, True)
            # attention: xm = x + o_proj(attn(qkv(rmsnorm(x))))
            g[p + "self_attn.o_proj.weight"] = ops.weight_grad(dx, s["o"], M, H, H, torch.empty(H, H, device=dev), scale=unscale)
            do = torch.empty(M, H, device=dev)
            lin(planes(dx), self._transposed(prm[p + "self_attn.o_proj.weight"]), H, H, do)
            dqkv = torch.empty(M, 3 * H, device=dev)
            ops.lm_attn_train_bwd(s["qs"], s["kr"], s["v"], s["o"], do, s["lse"], B, L, heads, cos, sin, run["p"], run["seed"], i, dqkv,
                                  torch.empty(B * heads * L, device=dev))
            ops.rmsnorm(s["x"], prm[p + "input_layernorm.weight"], M, H, out_f32=nrm)
            gqkv = ops.weight_grad(dqkv, nrm, M, 3 * H, H, torch.empty(3 * H, H, device=dev), scale=unscale)
            for j, n in enumerate("qkv"):
                g[p + f"self_attn.{n}_proj.weight"] = gqkv[j * H:(j + 1) * H]
            wqkv = torch.cat([prm[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0)
            lin(planes(dqkv), self._transposed(wqkv), H, 3 * H, dn)
            del dqkv
            norm_bwd(s["x"], p + "input_layernorm.weight", dn, True)
            sv["layers"][i] = None                 # free this layer's activations as soon as they are used
        # inputs_embeds = [task | (enroll_sos, adapter(enroll)) | mix_sos, adapter(mix) | codec_embedding[input_ids]]
        g["codec_embedding.weight"] = torch.empty(V, H, device=dev)
        ids = run["input_ids"]
        ops.embedding_bwd(dx, ids, ids.numel(), Lt, L, P, H, V, g["codec_embedding.weight"], scale=unscale)
        colrow = lambda pos, out: ops.col_sum(dx[pos:], B, H, L * H, out, scale=unscale)
        g["task_embedding.weight"] = torch.zeros_like(prm["task_embedding.weight"])
        colrow(0, g["task_embedding.weight"][self.task_map[run["task"]]])
        x3 = dx.reshape(B, L, H)
        if Te:
            g["enroll_sos_embedding.weight"] = torch.empty(1, H, device=dev)
            colrow(1, g["enroll_sos_embedding.weight"])
            da = torch.cat([x3[:, 2:2 + Te].reshape(-1, H), x3[:, 3 + Te:P].reshape(-1, H)], 0).contiguous()
        else:
            da = x3[:, 2:P].reshape(-1, H).contiguous()
        g["mix_sos_embedding.weight"] = torch.empty(1, H, device=dev)
        colrow(P - Tm - 1, g["mix_sos_embedding.weight"])
        feats = sv["feats"]
        Nf, Fd = feats.shape
        g["adapter.weight"] = ops.weight_grad(da, feats, Nf, H, Fd, torch.empty(H, Fd, device=dev), scale=unscale)
        g["adapter.bias"] = torch.empty(H, device=dev)
        ops.col_sum(da, Nf, H, H, g["adapter.bias"], scale=unscale)
        torch._foreach_mul_(list(g.values()), grad_loss.float().reshape(()))          # on the device: no host read of grad_loss
        return g

    # ------------------------------------------------------------------ generate (llm_sft.py:93-195)
    @torch.no_grad()
    def generate(self, task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, global_length: int = 32,
                 temperature: float = 0.8, top_k: int = 50, top_p: float = 0.95, do_sample: bool = True,
                 use_cuda_graph: bool = True, seed: Optional[int] = None, enroll_lengths=None, row_seeds=None):
        """llm_sft.py:93-195 with the reference's signature and defaults.  do_sample=True draws every token on the device
        (top-k -> top-p -> temperature -> multinomial, csrc/llm.cu lm_sample_embed_kernel / lm_sample_full_embed_kernel); `seed`
        (default: torch's global generator) makes the draw reproducible.  Greedy decoding ignores temperature / top_k / top_p /
        seed / row_seeds exactly as the reference's arg-max does (filters never remove the arg-max, llm.py:263-287).

        top_k takes what the reference's `torch.topk` over the range-masked vocabulary row takes: 0 (or below) applies no top-k
        filter, any k up to the vocabulary size (12 291 at the shipped widths) is valid, and a k at or above the range width
        (4096 global / 8192 semantic tokens) keeps every token of the range; a k above the vocabulary raises as torch.topk does
        (except k <= 1024, which a reduced-width model keeps accepting as it always has).
        top_p >= 1 applies no top-p filter.

        `row_seeds` (ints [B], tensor or sequence; not together with `seed`): one 64-bit key per row.  Row b's uniforms are then a
        function of row_seeds[b] and the decode step only, so its tokens do not depend on its place in the batch, the chunk of 32
        it falls in, the lane or the batch size: a row draws the same tokens in any batch, and alone.  With `seed` the stream is
        one per call, and a row's uniforms depend on its row and chunk.

        `enroll_lengths` (ints [B], tensor or sequence): the valid frames of each row of a right-padded enroll_feats [B, Te_max, F],
        for rows whose enrollments differ in length.  Row b then decodes exactly as if it were generated alone with
        enroll_feats[b, :enroll_lengths[b]]: its prefix holds no padding, the padding sits after its own P_b positions, and the decode
        kernels keep one position per row (starting at P_b).  A causal prefill never lets a real position see the padded tail, and
        decode writes position P_b + s before it reads it, so the tail is never read.  None keeps the uniform path."""
        if enroll_lengths is not None:
            enroll_lengths = self._check_enroll_lengths(enroll_lengths, enroll_mel, enroll_feats, mix_feats.shape[0])
        if row_seeds is not None:
            row_seeds = self._check_row_seeds(row_seeds, seed, mix_feats.shape[0])
        sampling = None
        if do_sample:
            if not (0.0 < temperature <= 1.0):
                raise AssertionError("0 < temperature <= 1.0 (llm.py:278)")
            if top_k > max(self.vocab_size, 1024):     # 1..1024 were accepted at every width before the full-range sampler
                raise RuntimeError(f"top_k = {top_k} is out of range for the vocabulary of {self.vocab_size} tokens "
                                   "(torch.topk, llm.py:262)")
            sampling = dict(temperature=float(temperature), top_k=max(0, int(top_k)), top_p=float(top_p))
            if row_seeds is not None:
                sampling["row_keys"] = ops.row_keys_words(row_seeds)
            else:
                sampling["seed"] = int(torch.randint(0, 2 ** 62, (1,)).item()) if seed is None else int(seed)
        semantic_length = mix_mel.size(1)
        Ball = mix_feats.shape[0]
        starts = list(range(0, Ball, self.chunk))         # decode kernels keep <= 32 sequences' rows in registers
        n_lanes = min(self.lanes, len(starts))
        outs = []
        lens = lambda sl: None if enroll_lengths is None else enroll_lengths[sl]
        if n_lanes <= 1:
            for ci, b0 in enumerate(starts):
                sl = slice(b0, min(b0 + self.chunk, Ball))
                if sampling is not None:
                    sampling["call"] = ci
                    sampling["rows"] = sl
                outs.append(self._generate_chunk(task_name, None if enroll_mel is None else enroll_feats[sl], mix_feats[sl],
                                                 semantic_length, global_length, use_cuda_graph, sampling, lens(sl)))
        else:
            # chunk ci runs on lane ci % n_lanes: the host enqueues one chunk after the other, the device overlaps the lanes
            n_pos = 2 + mix_feats.shape[1] + (0 if enroll_mel is None else 1 + enroll_feats.shape[1]) + global_length + 1 + semantic_length
            views = self._lanes(n_lanes, n_pos)
            cur = torch.cuda.current_stream()
            ready = torch.cuda.Event()
            ready.record(cur)
            for ci, b0 in enumerate(starts):
                sl = slice(b0, min(b0 + self.chunk, Ball))
                view, stream = views[ci % n_lanes]
                if sampling is not None:
                    sampling["call"] = ci
                    sampling["rows"] = sl
                if ci < n_lanes:
                    stream.wait_event(ready)             # the inputs were produced on the caller's stream
                with torch.cuda.stream(stream):
                    outs.append(view._generate_chunk(task_name, None if enroll_mel is None else enroll_feats[sl], mix_feats[sl],
                                                     semantic_length, global_length, use_cuda_graph, sampling, lens(sl)))
            for _, stream in views[:n_lanes]:
                cur.wait_stream(stream)
            for gi, si in outs:                           # allocated on a lane's stream, consumed on the caller's
                gi.record_stream(cur)
                si.record_stream(cur)
        return torch.cat([o[0] for o in outs], 0), torch.cat([o[1] for o in outs], 0)

    @staticmethod
    def _check_enroll_lengths(enroll_lengths, enroll_mel, enroll_feats, B):
        """-> host list of B ints in 1..Te_max (read once: the prefix layout is built on the host)"""
        if enroll_mel is None or enroll_feats is None:
            raise ValueError("enroll_lengths needs an enrollment (enroll_mel and enroll_feats)")
        lens = [int(n) for n in (enroll_lengths.tolist() if torch.is_tensor(enroll_lengths) else enroll_lengths)]
        te_max = enroll_feats.shape[1]
        if len(lens) != B or any(n < 1 or n > te_max for n in lens):
            raise ValueError(f"enroll_lengths must hold {B} lengths in 1..{te_max} (the padded enrollment), got {lens}")
        return lens

    @staticmethod
    def _check_row_seeds(row_seeds, seed, B):
        """-> host list of B ints (one 64-bit key per row)"""
        if seed is not None:
            raise ValueError("give either `seed` (one random stream per call) or `row_seeds` (one per row), not both")
        if torch.is_tensor(row_seeds) and (row_seeds.is_floating_point() or row_seeds.is_complex()):
            raise ValueError(f"row_seeds must be integers, got a {row_seeds.dtype} tensor")
        keys = row_seeds.reshape(-1).tolist() if torch.is_tensor(row_seeds) else list(row_seeds)
        try:
            keys = [operator.index(k) for k in keys]
        except TypeError:
            raise ValueError(f"row_seeds must be integers, got {keys}") from None
        if len(keys) != B:
            raise ValueError(f"row_seeds must hold {B} keys, one per row, got {len(keys)}")
        return keys

    def _lanes(self, n: int, n_positions: int):
        """Lane = (shallow view of this module with its own workspace, decode state and captured graphs; its own stream).  The
        prepared weights and RoPE tables are shared read-only, so the tables are sized BEFORE the lanes exist (growing them
        replaces the tensors captured graphs point at)."""
        self._prepare()
        self._ensure_rope(n_positions)
        rows = self._w["rope_rows"]
        if self._lane_views is None or self._lane_views[0] != rows:
            self._lane_views = (rows, [])
        lanes = self._lane_views[1]
        while len(lanes) < n:
            v = copy.copy(self)
            v._ws, v._gen_state, v._lane_views = {}, {}, None
            v.lanes = 1
            v.att_unroll = self.lane_att_unroll
            lanes.append((v, torch.cuda.Stream(device=self._dev())))
        return lanes

    def _generate_chunk(self, task_name, enroll_feats, mix_feats, semantic_length, global_length, use_graph, sampling=None,
                        enroll_lengths=None):
        """enroll_lengths: host ints, one per row (ragged prefixes), or None.  P below is the padded prefix width: with ragged rows it
        is the same for every chunk of a call, so the chunks share one decode state and its captured graphs."""
        W = self._prepare()
        dev = mix_feats.device
        prefix = self._prefix(task_name, enroll_feats, mix_feats, enroll_lengths)
        B, P, H = prefix.shape
        n_steps = global_length + 1 + semantic_length
        Lmax = -(-(P + n_steps) // 64) * 64
        self._ensure_rope(P + n_steps)
        W = self._w
        max_cols = _pad_to(max(self.global_size, self.semantic_size), 16)     # the head runs 16 columns per CTA
        samp_key = None if sampling is None else (sampling["temperature"], sampling["top_k"], sampling["top_p"], "row_keys" in sampling)
        # Decode state (KV cache, counters, output ids) and the captured graphs are kept per shape: capturing and
        # instantiating ~560 kernel nodes costs the host 10-50 ms, as much as the whole generation takes on the device.
        key = (B, P, n_steps, bool(use_graph), int(self.graph_steps), str(dev), samp_key)
        st = self._gen_state.get(key)
        if st is None:
            self._gen_state.clear()                    # one shape at a time (the cache is ~0.9 GB at B=32)
            st = dict(cache=StaticKVCache(self.n_layers, B, self.heads, Lmax, dev),
                      xs=torch.zeros(B, H, device=dev),
                      rng=torch.zeros(2, dtype=torch.int32, device=dev), slot=torch.zeros(2, dtype=torch.int32, device=dev),
                      out_ids=torch.zeros(B, n_steps, dtype=torch.int64, device=dev),
                      pv=torch.zeros(max_cols // 16 + 1, 32, device=dev),
                      pi=torch.zeros(max_cols // 16 + 1, 32, dtype=torch.int32, device=dev), g1=None, gk=None, captured=False,
                      logits=torch.zeros(B, max_cols, device=dev) if sampling is not None else None,
                      seed=torch.zeros(4, dtype=torch.int32, device=dev), row_keys=torch.zeros(B, 2, dtype=torch.int32, device=dev),
                      dbg=torch.zeros(B, 4, device=dev))
            self._gen_state[key] = st
        cache, xs, rng, slot, out_ids, pv, pi = (st[k] for k in ("cache", "xs", "rng", "slot", "out_ids", "pv", "pi"))
        cache.length = 0
        cache.pos.zero_()
        slot.zero_()
        if sampling is not None and "row_keys" in sampling:       # per-row Philox keys, also in device memory
            st["row_keys"].copy_(sampling["row_keys"][sampling["rows"]], non_blocking=True)
        elif sampling is not None:      # Philox key / call counter live in device memory: the captured graph is reused across seeds
            sd_ = sampling["seed"]
            to_i32 = lambda v: v - (1 << 32) if v >= (1 << 31) else v
            st["seed"].copy_(torch.tensor([to_i32(sd_ & 0xFFFFFFFF), to_i32((sd_ >> 32) & 0xFFFFFFFF), sampling["call"], 0],
                                          dtype=torch.int32), non_blocking=True)
        rng.copy_(torch.tensor([self.global_offset, self.global_offset + self.global_size], dtype=torch.int32), non_blocking=True)
        x = prefix.reshape(B * P, H).contiguous().clone()
        self._prefill(x, B, P, cache)
        # the first decode step of row b writes position P_b (P for every row without ragged prefixes)
        starts = torch.tensor([P] * B if enroll_lengths is None else [3 + n + mix_feats.shape[1] for n in enroll_lengths],
                              dtype=torch.int32)

        def reset_pos():
            cache.pos.copy_(starts, non_blocking=True)
        reset_pos()

        def step():
            self._decode_layers(xs, B, cache)
            if sampling is not None and "row_keys" in sampling:
                ops.lm_head_sample_rows_tc(xs, B, H, W["head_p"], rng, max_cols, W["emb"], xs, out_ids, n_steps, cache.pos, slot, pv,
                                           pi, st["logits"], sampling["temperature"], sampling["top_k"], sampling["top_p"],
                                           st["row_keys"], st["dbg"])
            elif sampling is not None:
                ops.lm_head_sample_tc(xs, B, H, W["head_p"], rng, max_cols, W["emb"], xs, out_ids, n_steps, cache.pos, slot, pv, pi,
                                      st["logits"], sampling["temperature"], sampling["top_k"], sampling["top_p"], st["seed"], st["dbg"])
            else:
                ops.lm_head_argmax_tc(xs, B, H, W["head_p"], rng, max_cols, W["emb"], xs, out_ids, n_steps, cache.pos, slot, pv, pi)

        # All decode state is on the device, so a graph may hold any number of consecutive steps: one single-step graph
        # plus one of `graph_steps` steps (fewer replays per generation).
        K = max(1, int(self.graph_steps))
        if use_graph and not st["captured"]:
            # warm-up outside capture (one-time cudaFuncSetAttribute calls), then restore the mutated state
            xs.copy_(W["emb"][self.global_sos_token_id][None].expand(B, H))
            step()
            torch.cuda.synchronize()
            st["g1"] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(st["g1"]):
                step()
            if K > 1 and n_steps >= K:
                st["gk"] = torch.cuda.CUDAGraph()
                with torch.cuda.graph(st["gk"]):
                    for _ in range(K):
                        step()
            st["captured"] = True
            reset_pos()
            slot.zero_()
        g1, gk = (st["g1"], st["gk"]) if use_graph else (None, None)

        def run(n):
            while n > 0:
                if gk is not None and n >= K:
                    gk.replay()
                    n -= K
                else:
                    g1.replay() if g1 is not None else step()
                    n -= 1

        xs.copy_(W["emb"][self.global_sos_token_id][None].expand(B, H))
        run(global_length + 1)
        rng.copy_(torch.tensor([self.semantic_offset, self.semantic_offset + self.semantic_size], dtype=torch.int32))
        xs.copy_(W["emb"][self.semantic_sos_token_id][None].expand(B, H))
        run(semantic_length)
        cache.length += n_steps
        global_ids = out_ids[:, :global_length] - self.global_offset          # (new tensors: out_ids is reused by the next call)
        semantic_ids = out_ids[:, global_length + 1:] - self.semantic_offset
        return global_ids, semantic_ids


class _LMLoss(torch.autograd.Function):
    """The teacher-forced loss as one autograd node: forward runs the LM keeping the activations its backward needs, backward runs the
    library's gradient kernels and returns an fp32 gradient for every parameter (None for one the step did not use).  The backward
    reads the parameters the forward saw (aliases, not copies), so it refuses to run once one of them has been changed in place or
    replaced since the forward, as torch's own saved-tensor check does."""

    @staticmethod
    def forward(ctx, face, run, names, *params):
        prm = {n: p.detach().float().contiguous() for n, p in zip(names, params)}
        loss, acc, logits, saved = face._train_fwd(run, prm)
        ctx.face, ctx.run, ctx.names, ctx.prm, ctx.saved = face, run, names, prm, saved
        ctx.params, ctx.versions = params, tuple((p._version, p.data_ptr()) for p in params)
        ctx.mark_non_differentiable(acc, logits)
        return loss, acc, logits

    @staticmethod
    def backward(ctx, grad_loss, grad_acc, grad_logits):
        if ctx.saved is None:
            raise RuntimeError("LLM_SFT training forward: backward called twice on the same graph")
        changed = [n for n, p, v in zip(ctx.names, ctx.params, ctx.versions) if (p._version, p.data_ptr()) != v]
        if changed:
            raise RuntimeError(f"LLM_SFT training forward: {len(changed)} parameter(s) changed in place between the forward and the "
                               f"backward (first: {changed[0]}); run the backward before the optimizer step")
        g = ctx.face._train_bwd(ctx.run, ctx.prm, ctx.saved, grad_loss)
        ctx.saved = ctx.prm = ctx.params = None
        return (None, None, None) + tuple(g.get(n) for n in ctx.names)
