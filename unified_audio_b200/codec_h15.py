"""H-Codec-1.5 adaptive frame-rate `Codec` (SURVEY.md 8f.4) with the reference's surface, running on libquark_b200.

Mirrors QuarkAudio-HCodec/HCodec-1.5/vq/codec_adaptive.py:32-207:
    Codec(encoder_kwargs, decoder_kwargs, quantizer_kwargs, adaptive_kwargs)      # the four blocks of conf/config_adaptive_v3.yaml
    .encode(x [B,1,T] @16 kHz, feat [B,1024,T/320], threshold=0.0) -> {'acoustic_codes', 'semantic_codes'}: int64 [B,nq,G], the
        token length packed into every index, index = (length - 1) * codebook_size + code (negative in the padded groups of
        the shorter items of a batch, exactly as the reference produces them)
    .decode(acoustic_codes, semantic_codes, token_lengths=None) -> wav [B, T]
state_dict keys are the reference's.  No PyTorch / CPU fallback.

What runs where:
  * SEANet encoder / semantic encoder / RVQ / decoder blocks: the H-Codec-1.0 kernels (`codec_h1.py`) at this config's widths
    (vq/encoder_modules, vq/codec_decoder.py and vq/semantic_module.py are byte-identical between HCodec-1.0 and HCodec-1.5);
  * similarity alignment, length packing, de-aggregation: csrc/adaptive.cu (`adaptive.py`);
  * `QueryTokenAggregator` (adaptive/model_blocks/mimi/transformer.py:701-826): qb_agg_interleave builds the T + G sequence, the
    transformer runs on it, qb_agg_gather reads the query rows;
  * mimi `ProjectedTransformer` (transformer.py:436-596, 828-880; 32 layers each for the two aggregators and the bottleneck):
    LayerNorm(1e-5) -> bias-free in_proj GEMM -> full attention with RoPE -> out_proj GEMM with the LayerScale + residual
    epilogue -> LayerNorm -> linear1 GEMM + exact GELU epilogue -> linear2 GEMM with the LayerScale + residual epilogue.
    `causal=False` makes the reference's `attn_bias` None (transformer.py:403-415): `context` is inert and attention is full.
    The reference rotates interleaved pairs (2i, 2i+1) (module/rope.py:47-64); q.k is invariant under a common permutation of
    the head dims, so the Q and K rows of in_proj are permuted (evens first, then odds) once at load and the rotate-half
    attention kernels of the rest of the library apply unchanged.
One host read per encode (the batch's largest group count G, which the reference also reads: modeling_flexicodec_new.py:905)
sizes the T + G sequences; decode reads the largest total length the same way (pad_sequence in the reference).
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from . import _lib, adaptive, ops
from .codec import _Tree
from .codec_h1 import CodecH1, H1
from .ops import ACT_GELU, Planes, _p, _stream, rowmap

H15 = dict(H1, ratios=[8, 5, 4, 2], dec_dim=1024, sem_in=1024, sem_ch=1024,
           agg=dict(dim=512, heads=8, layers=32, ff=2048), bottleneck=dict(dim=1024, heads=8, layers=32, ff=2048),
           threshold=0.6, max_group=8)
# which GEMM operands of the mimi transformers carry the fp16 hi + lo split (3 tensor-core passes) - same meaning as
# codec.PRECISION_POLICIES.  The aggregators sit in front of the RVQ (index identity is decided by their output) and keep
# fp32-grade arithmetic in every policy but "fast"; the bottleneck sits behind the indices.
MIMI_POLICIES = {"mixed": dict(agg=True, bottleneck=True), "accurate": dict(agg=True, bottleneck=True),
                 "mixed_dec16": dict(agg=True, bottleneck=False), "fast": dict(agg=False, bottleneck=False)}


def config_from_kwargs(encoder_kwargs, decoder_kwargs, quantizer_kwargs, adaptive_kwargs) -> dict:
    """conf/config_adaptive_v3.yaml blocks -> the flat config of this file (only the fields the reference's constructors read)"""
    e, s = encoder_kwargs["encoder"], encoder_kwargs["semantic_encoder"]
    d, q, a = decoder_kwargs["decoder"], quantizer_kwargs["quantizer"], adaptive_kwargs
    if not (a.get("use_similarity_alignment") and a.get("use_query_token_aggregator") and a.get("use_bottleneck_transformer")):
        raise ValueError("CodecH15 builds the shipped adaptive configuration: similarity alignment + query-token aggregators + "
                         "bottleneck transformer must all be enabled")
    ag, bt = a["aggregators"]["semantic_aggregator"], a["transformer_kwargs"]
    if a["aggregators"]["acoustic_aggregator"] != ag:
        raise ValueError("the two aggregators must share one shape")
    for t in (ag, bt):
        if t.get("causal", False):
            raise ValueError("causal mimi transformers are not built (the shipped config is non-causal)")
    if bt.get("gating", "none") != "none" or bt.get("norm", "layer_norm") != "layer_norm" or bt.get("positional_embedding", "rope") != "rope":
        raise ValueError("bottleneck transformer: only gating none / layer_norm / rope (the shipped config) is built")
    if bt["input_dimension"] != bt["d_model"] or list(bt["output_dimensions"]) != [bt["d_model"]] or ag["in_out_dim"] != ag["dim"]:
        raise ValueError("input / output projections of ProjectedTransformer are not built (the shipped config has none)")
    return dict(n_filters=e["n_filters"], dimension=e["dimension"], ratios=list(reversed(e["ratios"])),
                dec_dim=d["dim"], dec_inter=d["intermediate_dim"], dec_layers=d.get("convnext_layers", 12),
                n_fft=d.get("n_fft", 1280), hop=d.get("hop_length", 320), nq=q["num_quantizers"], codebook_size=q["codebook_size"],
                sem_in=s["input_channels"], sem_ch=s["encode_channels"], sem_strides=list(s["strides"]), tf_layers=2, heads=8,
                agg=dict(dim=ag["dim"], heads=ag["num_heads"], layers=ag["num_layers"], ff=ag["dim_feedforward"]),
                bottleneck=dict(dim=bt["d_model"], heads=bt["num_heads"], layers=bt["num_layers"], ff=bt["dim_feedforward"]),
                threshold=a.get("manual_threshold") if a.get("manual_threshold") is not None else a["similarity_threshold"],
                max_group=a["max_tokens_per_group"])


def mimi_spec(t) -> Dict[str, tuple]:
    out, d, ff = {}, t["dim"], t["ff"]
    for i in range(t["layers"]):
        p = f"transformer.transformer.layers.{i}."
        out[p + "self_attn.in_proj_weight"] = (3 * d, d)
        out[p + "self_attn.out_proj.weight"] = (d, d)
        for n in ("norm1", "norm2"):
            out[p + n + ".weight"] = (d,)
            out[p + n + ".bias"] = (d,)
        out[p + "linear1.weight"] = (ff, d)
        out[p + "linear2.weight"] = (d, ff)
        out[p + "layer_scale_1.scale"] = (d,)
        out[p + "layer_scale_2.scale"] = (d,)
    return out


class CodecH15(CodecH1):
    def __init__(self, encoder_kwargs: dict = None, decoder_kwargs: dict = None, quantizer_kwargs: dict = None,
                 adaptive_kwargs: dict = None, precision: str = "mixed", _cfg: dict = None, semantic_decoder: bool = False):
        c = dict(_cfg) if _cfg is not None else (
            config_from_kwargs(encoder_kwargs, decoder_kwargs, quantizer_kwargs, adaptive_kwargs) if adaptive_kwargs else dict(H15))
        if adaptive_kwargs and decoder_kwargs.get("semantic_decoder") is not None:     # conf/config_adaptive_v3.yaml:38-43
            c["sem_dec"] = dict(decoder_kwargs["semantic_decoder"])
        CodecH1.__init__(self, precision=precision, _cfg=c, semantic_decoder=semantic_decoder)
        agg = dict(mimi_spec(c["agg"]), query_embedding=(1, c["agg"]["dim"], 1))
        self.semantic_aggregator = _Tree.build(agg)
        self.acoustic_aggregator = _Tree.build(agg)
        self.bottleneck_transformer = _Tree.build({k[len("transformer."):]: v for k, v in mimi_spec(c["bottleneck"]).items()})
        self.mimi_policy = dict(MIMI_POLICIES[precision])
        self.codebook_size = c["codebook_size"]
        self.manual_threshold = c["threshold"]
        self.eval()

    # ------------------------------------------------------------------ weight repack
    def _pack_mimi(self, sd, prefix, t, split):
        d, heads = t["dim"], t["heads"]
        hd = d // heads
        # interleaved RoPE pairs (2i, 2i+1) -> rotate-half layout (i, i + hd/2) for the Q and K rows of in_proj
        perm = torch.cat([torch.arange(0, hd, 2), torch.arange(1, hd, 2)])
        rows = torch.cat([(torch.arange(heads)[:, None] * hd + perm[None]).reshape(-1) + blk * d for blk in (0, 1)] +
                         [torch.arange(2 * d, 3 * d)])
        layers = []
        for i in range(t["layers"]):
            p = f"{prefix}transformer.layers.{i}."
            f32 = lambda k: sd[p + k].float().contiguous()
            lw = lambda w: Planes.from_f32(w.float().contiguous(), split)
            layers.append(dict(n1w=f32("norm1.weight"), n1b=f32("norm1.bias"), n2w=f32("norm2.weight"), n2b=f32("norm2.bias"),
                               wqkv=lw(sd[p + "self_attn.in_proj_weight"].float()[rows.to(sd[p + "self_attn.in_proj_weight"].device)]),
                               wo=lw(sd[p + "self_attn.out_proj.weight"]), w1=lw(sd[p + "linear1.weight"]),
                               w2=lw(sd[p + "linear2.weight"]), ls1=f32("layer_scale_1.scale"), ls2=f32("layer_scale_2.scale")))
        return layers

    def _prepare(self):
        if self._w is not None:
            return self._w
        W = CodecH1._prepare(self)
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        c, mp = self.c, self.mimi_policy
        for name in ("semantic_aggregator", "acoustic_aggregator"):
            W[name] = dict(layers=self._pack_mimi(sd, f"{name}.transformer.", c["agg"], mp["agg"]),
                           qemb=sd[f"{name}.query_embedding"].float().reshape(-1).contiguous())
        W["bottleneck"] = dict(layers=self._pack_mimi(sd, "bottleneck_transformer.", c["bottleneck"], mp["bottleneck"]))
        return W

    def _rope_mimi(self, L, hd):
        """module/rope.py:38-40, 57-58 in the rotate-half layout: cos / sin [L, hd] with column j and j + hd/2 = frequency j"""
        freqs = torch.exp(torch.arange(hd // 2, dtype=torch.float32) * (-math.log(10000.0) * 2 / hd))
        ang = torch.arange(L, dtype=torch.float32)[:, None] * freqs[None]
        emb = torch.cat((ang, ang), -1)
        return emb.cos().to(self._dev()).contiguous(), emb.sin().to(self._dev()).contiguous()

    # ------------------------------------------------------------------ mimi transformer
    def _mimi(self, layers, x, B, L, t, split, taps=None, tap_name=None):
        """StreamingTransformer.forward (transformer.py:676-697) without streaming state; x [B*L, C] fp32 updated in place."""
        C, heads, FF = t["dim"], t["heads"], t["ff"]
        hd, M = C // heads, B * L
        t_a = self._planes("mm_a", (M, C), split)
        t_b = self._planes("mm_b", (M, C), split)
        hid = self._planes("mm_hid", (M, FF), split)
        qkv = self._buf("mm_qkv", (M, 3 * C))
        cos, sin = self._cached(("rope_mimi", L, hd), lambda: self._rope_mimi(L, hd))
        att_ws = self._buf("att5_ws", (ops.self_attention_workspace_bytes(B, L, heads, hd, split),), torch.uint8)
        xm = rowmap(x, C, M, 0)
        for i, Lw in enumerate(layers):
            ops.layernorm(x, Lw["n1w"], Lw["n1b"], 1, M, C, eps=1e-5, out=t_a)
            self._linear(t_a, Lw["wqkv"], 3 * C, M, C, out_f32=rowmap(qkv, 3 * C, M, 0))
            ops.self_attention(qkv, B, L, heads, hd, cos, sin, t_b, att_ws, split)
            self._linear(t_b, Lw["wo"], C, M, C, gamma=Lw["ls1"], residual=xm, out_f32=xm)
            ops.layernorm(x, Lw["n2w"], Lw["n2b"], 1, M, C, eps=1e-5, out=t_a)
            self._linear(t_a, Lw["w1"], FF, M, C, act=ACT_GELU, out_planes=hid, out_planes_map=(FF, M, 0))
            self._linear(hid, Lw["w2"], C, M, FF, gamma=Lw["ls2"], residual=xm, out_f32=xm)
            if taps is not None and tap_name and i in (0, len(layers) - 1):
                taps[f"{tap_name}.layer{i}"] = x.reshape(B, L, C).transpose(1, 2).clone()

    def _aggregate(self, name, feats, B, T, plan, taps=None, tap_name=None):
        """QueryTokenAggregator.forward: feats [B*T, D] fp32 rows -> tokens [B*G, D] (zero rows for padded groups)"""
        W = self._prepare()[name]
        t = self.c["agg"]
        D, G = t["dim"], plan["G"]
        L = T + G
        # the kernel takes seg / lengths / offsets as row indices into the T + G sequence: a tensor of another dtype or shape
        # would be read as out-of-range rows, so refuse it here
        for key, shape in (("seg", (B, T)), ("lens32", (B, G)), ("offsets", (B, G)), ("ng32", (B,))):
            v = plan[key]
            if v.dtype != torch.int32 or tuple(v.shape) != shape:
                raise ValueError(f"aggregation plan: {key} must be int32 {shape}, got {v.dtype} {tuple(v.shape)}")
        lib = _lib.load()
        x = self._buf(f"agg_x{L}", (B * L, D))
        qpos = self._buf(f"agg_qpos{G}", (B, G), torch.int32)
        _lib.check(lib.qb_agg_interleave(_p(feats), _p(plan["seg"]), _p(plan["lens32"]), _p(plan["offsets"]), _p(plan["ng32"]),
                                         _p(W["qemb"]), B, T, G, D, _p(x), _p(qpos), _stream()))
        if taps is not None and tap_name:
            taps[f"{tap_name}.interleaved"] = x.reshape(B, L, D).transpose(1, 2).clone()
        self._mimi(W["layers"], x, B, L, t, self.mimi_policy["agg"], taps, tap_name)
        tok = torch.empty(B * G, D, device=feats.device)
        _lib.check(lib.qb_agg_gather(_p(x), _p(qpos), _p(plan["ng32"]), B, L, G, D, _p(tok), _stream()))
        return tok

    # ------------------------------------------------------------------ public surface
    def _threshold(self, threshold: float) -> float:
        if not 0.0 <= threshold <= 1.0:
            raise ValueError("threshold must be in [0, 1]")          # codec_adaptive.py:153
        return float(self.manual_threshold) if threshold <= 0.0 else float(threshold)

    @torch.no_grad()
    def encode(self, x, feat, use_mask=False, domain_split=None, threshold: float = 0.0, taps=None):
        """codec_adaptive.py:150-183"""
        c = self.c
        emb, N = self._encode_emb(x, taps)
        sem, Ns = self._encode_sem(feat, taps)
        if Ns != N:
            raise ValueError(f"semantic stream has {Ns} frames but the acoustic stream has {N}")
        B, D = x.shape[0], c["dimension"]
        seg, sim, ng, lens = adaptive.similarity_alignment(sem.view(B, N, D), self._threshold(threshold), c["max_group"],
                                                           want_matrix=False)
        G = lens.shape[1]
        lens32 = lens.to(torch.int32).contiguous()
        offsets = torch.empty(B, G, dtype=torch.int32, device=x.device)
        totals = torch.empty(B, dtype=torch.int32, device=x.device)
        _lib.check(_lib.load().qb_length_offsets(_p(lens32), B, G, _p(offsets), _p(totals), _stream()))
        plan = dict(seg=seg, lens32=lens32, offsets=offsets, ng32=ng.to(torch.int32).contiguous(), G=G)
        if taps is not None:
            taps["seg"], taps["n_groups"], taps["sim"], taps["token_lengths"] = seg.clone(), ng.clone(), sim.clone(), lens.clone()
        sem_tok = self._aggregate("semantic_aggregator", sem, B, N, plan, taps, "sem_agg")
        ac_tok = self._aggregate("acoustic_aggregator", emb, B, N, plan, taps, "ac_agg")
        if taps is not None:
            taps["sem_agg.out"] = sem_tok.reshape(B, G, D).transpose(1, 2).clone()
            taps["ac_agg.out"] = ac_tok.reshape(B, G, D).transpose(1, 2).clone()
        ia, _ = self.quantizer.encode_rows(ac_tok, want_quantized=False)
        isem, _ = self.semantic_quantizer.encode_rows(sem_tok, want_quantized=False)
        K = self.codebook_size
        return dict(acoustic_codes=adaptive.inject_lengths(ia.reshape(B, G, -1).transpose(1, 2), lens, K),
                    semantic_codes=adaptive.inject_lengths(isem.reshape(B, G, -1).transpose(1, 2), lens, K))

    @torch.no_grad()
    def decode(self, acoustic_codes, semantic_codes, token_lengths=None, taps=None):
        """codec_adaptive.py:186-207"""
        c, K = self.c, self.codebook_size
        if token_lengths is None:
            acoustic_codes, token_lengths = adaptive.extract_lengths(acoustic_codes, K)
            semantic_codes, token_lengths = adaptive.extract_lengths(semantic_codes, K)
        ac = adaptive.deaggregate_by_lengths(acoustic_codes.long(), token_lengths)          # [B, nq, T]
        sc = adaptive.deaggregate_by_lengths(semantic_codes.long(), token_lengths)
        B, nq, T = ac.shape
        Dq = self.quantizer.dim
        z = self._buf(f"dec_z{T}", (B * T, 2 * Dq))
        self.quantizer.decode_rows(ac.transpose(1, 2).reshape(B * T, nq).contiguous(), z, 2 * Dq, 0)
        self.semantic_quantizer.decode_rows(sc.transpose(1, 2).reshape(B * T, nq).contiguous(), z, 2 * Dq, Dq)
        if taps is not None:
            taps["dec.z"] = z.reshape(B, T, 2 * Dq).transpose(1, 2).clone()
        self._mimi(self._prepare()["bottleneck"]["layers"], z, B, T, c["bottleneck"], self.mimi_policy["bottleneck"], taps, "bottleneck")
        if taps is not None:
            taps["bottleneck.out"] = z.reshape(B, T, 2 * Dq).transpose(1, 2).clone()
        return self._decode_z(z, B, T, taps)

    @torch.no_grad()
    def roundtrip(self, x, feat):
        out = self.encode(x, feat)
        return out["acoustic_codes"], out["semantic_codes"], self.decode(out["acoustic_codes"], out["semantic_codes"])

    @torch.no_grad()
    def semantic_decode(self, semantic_codes, token_lengths=None):
        """codec_adaptive.py:132,139: the semantic decoder on the de-aggregated semantic stream.  semantic_codes: the length-packed
        int64 [B,nq,G] of `encode` (or plain codes with token_lengths [B,G]) -> pred_feat fp32 [B, 1024, T * prod(strides)]."""
        self._require_semantic_decoder()
        if token_lengths is None:
            semantic_codes, token_lengths = adaptive.extract_lengths(semantic_codes, self.codebook_size)
        sc = adaptive.deaggregate_by_lengths(semantic_codes.long(), token_lengths)          # [B, nq, T]
        B, nq, T = sc.shape
        z = self._buf(f"sd_zrows{T}", (B * T, self.semantic_quantizer.dim))
        self.semantic_quantizer.decode_rows(sc.transpose(1, 2).reshape(B * T, nq).contiguous(), z, self.semantic_quantizer.dim, 0)
        return self._semantic_decode_rows(z, B, T)

    def forward(self, x, feat, use_mask=False, domain_split=None):
        """codec_adaptive.py:100-147 in evaluation mode, at the threshold encode(threshold=0.0) uses: {'recon' [B, T],
        'pred_feat' fp32 [B, 1024, T_feat], 'commit_loss' 0-d fp32, 'token_lengths' int64 [B, G]}, recon = decode(**encode(x, feat))."""
        self._check_forward()
        with torch.no_grad():
            codes = self.encode(x, feat)
            plain, lens = adaptive.extract_lengths(codes["semantic_codes"], self.codebook_size)
            return dict(recon=self.decode(codes["acoustic_codes"], codes["semantic_codes"]),
                        pred_feat=self.semantic_decode(plain, token_lengths=lens), commit_loss=self._commit_loss(),
                        token_lengths=lens)
