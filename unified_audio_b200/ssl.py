"""SSL feature front ends and tokenizer glue on libquark_b200 (SURVEY.md 8f.2 / 8f.3).

    HCodecTokenizer.extract_ssl_features   QuarkAudio-HCodec/HCodec-2.0/audio_tokenizer.py:47-61
        Resample(48k -> 16k) -> pad 160/160 -> HuBERT-base (`AutoModel "bosonai/hubert_base"`, output_hidden_states) ->
        mean of the 13 hidden states -> sign(x) |x|^0.3                                       [B, T50, 768]
    HCodecTokenizer.pad_wav / tokenize      audio_tokenizer.py:63-75
    HCodecTokenizerH1                       QuarkAudio-HCodec/HCodec-1.0/audio_tokenizer.py:18-66
        pad_wav (640) -> pad 160/160 -> HuBERT-base at 16 kHz -> mean of the 13 hidden states -> sign(x) |x|^0.3 -> CodecH1.encode
    HCodecTokenizerH15                      QuarkAudio-HCodec/HCodec-1.5/audio_tokenizer.py:38-86
        pad_wav (prod(ratios) * 2) -> pad 160/160 -> wav2vec2-large-xlsr-53, no normalisation (WAV2VEC2_XLSR53_RAW) ->
        (hidden_states[11] + hidden_states[14] + hidden_states[16]) / 3 -> sign(x) |x|^0.3 -> CodecH15.encode (length-packed codes)
    Model.extract_semantic_features         QuarkAudio-UniSE/model/model.py:38-51  (WavLM-base-plus, no compression)
    BiCodecTokenizer.extract_wav2vec2_features   QuarkAudio-UniSE/model/bicodec/audio_tokenizer.py:74-90
        Wav2Vec2FeatureExtractor(do_normalize=True) -> wav2vec2-large-xlsr-53 (no padding) ->
        (hidden_states[11] + hidden_states[14] + hidden_states[16]) / 3                       [B, T', 1024]
    wrap padding + 5 s segmenting           QuarkAudio-UniSE/model/model.py:175-181

`SSLFrontEnd(config)` holds the parameters under the key names of `transformers.HubertModel` / `WavLMModel`
(`feature_extractor.conv_layers.{i}.conv.weight`, `feature_projection.*`, `encoder.pos_conv_embed.conv.parametrizations.weight.*`,
`encoder.layers.{i}.attention.{q,k,v,out}_proj.*`, `feed_forward.*`, `layer_norm`, `final_layer_norm`; WavLM adds
`attention.gru_rel_pos_*` and `encoder.layers.0.attention.rel_attn_embed.weight`; `transformers.Wav2Vec2Model` adds
`feature_extractor.conv_layers.{i}.conv.bias` and `.layer_norm.*` for every conv), so a checkpoint's state-dict loads as is.

Kernels: torchaudio's sinc resampler is a stride-3 41-tap FIR = a 2-tap Toeplitz GEMM over 192-sample rows; conv layer 0
(one input channel) + per-channel GroupNorm + GELU are csrc/ssl.cu; conv layers 1-6 are TMA-im2col GEMMs with a GELU epilogue;
the weight-normed grouped positional conv (k = 128, 16 groups) is 16 GEMMs over a group-padded buffer (`a_cols`); the 12 post-LN
layers run on the wgmma GEMMs (3-term split) + the wgmma attention (HuBERT; WavLM's gated relative-position bias keeps the fp32 kernel).
wav2vec2 (feat_extract_norm="layer", do_stable_layer_norm=True): the processor normalisation (fp64 statistics) and conv layer 0 +
bias are csrc/ssl.cu, every conv is followed by LayerNorm over channels + GELU (qb_layernorm_act) written as planes of the next
conv's buffer, and the pre-LN layers run up to the last hidden state the output needs (layers 17-24 and `encoder.layer_norm` of
XLSR-53 are loaded but never computed).  No PyTorch / CPU fallback.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
from torch import nn

from . import ops
from .codec import _Face, _Tree, _pad_to
from .codec_h1 import CodecH1
from .codec_h15 import CodecH15
from .ops import ACT_GELU, Planes, rowmap

HUBERT_BASE = dict(conv_dim=[512] * 7, conv_kernel=[10, 3, 3, 3, 3, 2, 2], conv_stride=[5, 2, 2, 2, 2, 2, 2], hidden=768,
                   layers=12, heads=12, ffn=3072, pos_k=128, pos_groups=16, eps=1e-5, kind="hubert")
WAVLM_BASE_PLUS = dict(HUBERT_BASE, num_buckets=320, max_distance=800, kind="wavlm")
# facebook/wav2vec2-large-xlsr-53 as BiCodec's tokenizer uses it: hidden_state_ids are the averaged hidden states (0 = the
# positional-conv output, k = the residual stream after layer k), do_normalize the feature extractor's per-utterance normalisation
WAV2VEC2_XLSR53 = dict(HUBERT_BASE, hidden=1024, layers=24, heads=16, ffn=4096, kind="wav2vec2", hidden_state_ids=(11, 14, 16),
                       do_normalize=True)
# the same model as H-Codec-1.5's tokenizer calls it (HCodec-1.5/audio_tokenizer.py:53-66): a bare `AutoModel`, no processor
# normalisation; `HCodecTokenizerH15` adds the 160/160 pad and the front end is built with compress=True
WAV2VEC2_XLSR53_RAW = dict(WAV2VEC2_XLSR53, do_normalize=False)


def ssl_spec(c: dict) -> Dict[str, tuple]:
    out: Dict[str, tuple] = {}
    cin = 1
    w2v = c.get("kind") == "wav2vec2"
    for i, (co, k) in enumerate(zip(c["conv_dim"], c["conv_kernel"])):
        out[f"feature_extractor.conv_layers.{i}.conv.weight"] = (co, cin, k)
        if w2v:                                 # conv_bias=True, feat_extract_norm="layer"
            out[f"feature_extractor.conv_layers.{i}.conv.bias"] = (co,)
        if i == 0 or w2v:
            out[f"feature_extractor.conv_layers.{i}.layer_norm.weight"] = (co,)
            out[f"feature_extractor.conv_layers.{i}.layer_norm.bias"] = (co,)
        cin = co
    H = c["hidden"]
    out["feature_projection.layer_norm.weight"] = (cin,)
    out["feature_projection.layer_norm.bias"] = (cin,)
    out["feature_projection.projection.weight"] = (H, cin)
    out["feature_projection.projection.bias"] = (H,)
    out["encoder.pos_conv_embed.conv.bias"] = (H,)
    out["encoder.pos_conv_embed.conv.parametrizations.weight.original0"] = (1, 1, c["pos_k"])
    out["encoder.pos_conv_embed.conv.parametrizations.weight.original1"] = (H, H // c["pos_groups"], c["pos_k"])
    out["encoder.layer_norm.weight"] = (H,)
    out["encoder.layer_norm.bias"] = (H,)
    for i in range(c["layers"]):
        p = f"encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            out[p + f"attention.{n}.weight"] = (H, H)
            out[p + f"attention.{n}.bias"] = (H,)
        if c.get("kind") == "wavlm":
            d = H // c["heads"]
            out[p + "attention.gru_rel_pos_const"] = (1, c["heads"], 1, 1)
            out[p + "attention.gru_rel_pos_linear.weight"] = (8, d)
            out[p + "attention.gru_rel_pos_linear.bias"] = (8,)
        out[p + "layer_norm.weight"] = (H,)
        out[p + "layer_norm.bias"] = (H,)
        out[p + "feed_forward.intermediate_dense.weight"] = (c["ffn"], H)
        out[p + "feed_forward.intermediate_dense.bias"] = (c["ffn"],)
        out[p + "feed_forward.output_dense.weight"] = (H, c["ffn"])
        out[p + "feed_forward.output_dense.bias"] = (H,)
        out[p + "final_layer_norm.weight"] = (H,)
        out[p + "final_layer_norm.bias"] = (H,)
    if c.get("kind") == "wavlm":
        out["encoder.layers.0.attention.rel_attn_embed.weight"] = (c["num_buckets"], c["heads"])
    return out


def resample_kernel(orig: int, new: int, lowpass_filter_width: int = 6, rolloff: float = 0.99):
    """torchaudio.functional._get_sinc_resample_kernel (sinc_interp_hann) in fp64 -> ([new', k] fp32, width, orig', new'), for decimation
    (orig > new) and interpolation (orig < new) alike: row j of the kernel gives output phase j of each input stride of orig' samples"""
    g = math.gcd(orig, new)
    orig, new = orig // g, new // g
    base = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base)
    idx = torch.arange(-width, width + orig, dtype=torch.float64)[None] / orig
    t = torch.arange(0, -new, -1, dtype=torch.float64)[:, None] / new + idx
    t = (t * base).clamp(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t = t * math.pi
    kern = torch.where(t == 0, torch.tensor(1.0, dtype=torch.float64), t.sin() / t) * window * (base / orig)
    return kern.float(), width, orig, new


class SSLFrontEnd(_Face):
    _IGNORED_KEYS = ("masked_spec_embed",)          # pre-training only

    def __init__(self, config: Optional[dict] = None, in_rate: int = 16000, compress: bool = False):
        """config: HUBERT_BASE / WAVLM_BASE_PLUS / WAV2VEC2_XLSR53 (or a reduced dict of the same keys).  in_rate 48000 adds the
        tokenizer's Resample(48k -> 16k); compress adds sign(x)|x|^0.3 (H-Codec tokenizer) - UniSE and BiCodec use neither."""
        super().__init__()
        self.cfg = dict(config or HUBERT_BASE)
        if self.cfg.get("kind") == "wav2vec2":
            ids = self.cfg["hidden_state_ids"]
            if not ids or min(ids) < 0 or max(ids) >= self.cfg["layers"]:
                raise ValueError(f"hidden_state_ids {ids} must lie in [0, layers) (the last state carries encoder.layer_norm)")
        self.in_rate, self.compress = in_rate, compress
        tree = _Tree.build(ssl_spec(self.cfg))
        for name, child in tree.named_children():
            self.add_module(name, child)
        self.eval()

    # ------------------------------------------------------------------ weight repack
    def _prepare(self):
        if self._w is not None:
            return self._w
        dev = self._require_cuda()
        c = self.cfg
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        W: Dict[str, object] = {}
        f32 = lambda k: sd[k].contiguous()

        if self.in_rate != 16000:
            kern, width, o, n = resample_kernel(self.in_rate, 16000)
            if n != 1:
                raise NotImplementedError("Resample: only integer decimation (48 kHz -> 16 kHz) is implemented")
            # y[64 m + j] = sum_i kern[i] x_pad[o (64 m + j) + i]: a 2-tap GEMM over rows of 64*o samples with a Toeplitz weight
            R = 64 * o
            if kern.shape[1] > R + o:
                raise NotImplementedError("resampling kernel longer than one row")
            wt = torch.zeros(64, 2 * R, dtype=torch.float64)
            for j in range(64):
                wt[j, o * j: o * j + kern.shape[1]] = kern[0].double()
            W["resample"] = dict(w=Planes.from_f32(wt.float().to(dev), True), width=width, o=o, R=R, k=kern.shape[1])
        w2v = c.get("kind") == "wav2vec2"
        nconv = len(c["conv_dim"])
        W["conv0_w"] = f32("feature_extractor.conv_layers.0.conv.weight").reshape(c["conv_dim"][0], -1).contiguous()
        W["gn_w"], W["gn_b"] = f32("feature_extractor.conv_layers.0.layer_norm.weight"), f32("feature_extractor.conv_layers.0.layer_norm.bias")
        W["convs"] = [ops.conv_planes(sd[f"feature_extractor.conv_layers.{i}.conv.weight"]) for i in range(1, nconv)]
        if w2v:
            W["conv_b"] = [f32(f"feature_extractor.conv_layers.{i}.conv.bias") for i in range(nconv)]
            W["conv_ln"] = [(f32(f"feature_extractor.conv_layers.{i}.layer_norm.weight"), f32(f"feature_extractor.conv_layers.{i}.layer_norm.bias"))
                            for i in range(nconv)]
        W["fp_ln_w"], W["fp_ln_b"] = f32("feature_projection.layer_norm.weight"), f32("feature_projection.layer_norm.bias")
        W["fp_w"] = ops.pad_k_planes(sd["feature_projection.projection.weight"], _pad_to(c["conv_dim"][-1], 64))
        W["fp_b"] = f32("feature_projection.projection.bias")
        # weight-normed grouped positional conv: w = g * v / ||v|| (norm over (out, in) per tap); per group [Cg, k * 64] planes
        g0, v = sd["encoder.pos_conv_embed.conv.parametrizations.weight.original0"], sd["encoder.pos_conv_embed.conv.parametrizations.weight.original1"]
        w = v * (g0 / v.pow(2).sum((0, 1), keepdim=True).sqrt())
        H, G, K = c["hidden"], c["pos_groups"], c["pos_k"]
        cg = H // G
        if cg > 64:
            raise NotImplementedError("positional conv: more than 64 channels per group")
        wg = torch.zeros(G, cg, K, 64, device=dev)
        wg[:, :, :, :cg] = w.reshape(G, cg, cg, K).permute(0, 1, 3, 2)             # [g, out, tap, in]
        W["pos_w"] = [Planes.from_f32(wg[g].reshape(cg, K * 64), True) for g in range(G)]
        W["pos_b"] = f32("encoder.pos_conv_embed.conv.bias")
        W["enc_ln_w"], W["enc_ln_b"] = f32("encoder.layer_norm.weight"), f32("encoder.layer_norm.bias")
        layers = []
        for i in range(max(c["hidden_state_ids"]) if w2v else c["layers"]):     # wav2vec2: layers past the last state used are dead
            p = f"encoder.layers.{i}."
            wqkv = torch.cat([sd[p + f"attention.{n}_proj.weight"] for n in "qkv"], 0)
            L = dict(wqkv=Planes.from_f32(wqkv, True), bqkv=torch.cat([sd[p + f"attention.{n}_proj.bias"] for n in "qkv"], 0).contiguous(),
                     wo=Planes.from_f32(sd[p + "attention.out_proj.weight"], True), bo=f32(p + "attention.out_proj.bias"),
                     ln_w=f32(p + "layer_norm.weight"), ln_b=f32(p + "layer_norm.bias"),
                     w1=Planes.from_f32(sd[p + "feed_forward.intermediate_dense.weight"], True), b1=f32(p + "feed_forward.intermediate_dense.bias"),
                     w2=Planes.from_f32(sd[p + "feed_forward.output_dense.weight"], True), b2=f32(p + "feed_forward.output_dense.bias"),
                     fln_w=f32(p + "final_layer_norm.weight"), fln_b=f32(p + "final_layer_norm.bias"))
            if c.get("kind") == "wavlm":
                L.update(gru_w=f32(p + "attention.gru_rel_pos_linear.weight"), gru_b=f32(p + "attention.gru_rel_pos_linear.bias"),
                         gru_c=f32(p + "attention.gru_rel_pos_const").reshape(-1).contiguous())
            layers.append(L)
        W["layers"] = layers
        if c.get("kind") == "wavlm":
            W["rel_embed"] = f32("encoder.layers.0.attention.rel_attn_embed.weight")
        self._w = W
        return W

    def _rel_table(self, T):
        """WavLMAttention.compute_bias / _relative_positions_bucket as a per-distance table [heads, 2T - 1]
        (entry (h, r + T - 1) = rel_attn_embed[bucket(r)][h], r = key - query); built once per length (load-time glue)."""
        c = self.cfg
        rel = torch.arange(-(T - 1), T)
        nb = c["num_buckets"] // 2
        bucket = (rel > 0).long() * nb
        a = rel.abs()
        max_exact = nb // 2
        large = torch.log(a.float() / max_exact) / math.log(c["max_distance"] / max_exact) * (nb - max_exact)
        large = torch.min((max_exact + large).long(), torch.full_like(a, nb - 1))
        bucket = bucket + torch.where(a < max_exact, a, large)
        emb = self._prepare()["rel_embed"]                       # [num_buckets, heads]
        return emb[bucket.to(emb.device)].t().contiguous()        # [heads, 2T - 1]

    def _identity_rope(self, T, D):
        return self._cached(("rope1", T, D), lambda: (torch.ones(T, D, device=self._dev()), torch.zeros(T, D, device=self._dev())))

    def _embed(self, feats: torch.Tensor, B: int, Tf: int, taps: Optional[dict] = None) -> torch.Tensor:
        """conv features [B * Tf, Cf] -> feature projection (LayerNorm -> Linear) -> x + GELU(positional conv(x)) [B * Tf, H]"""
        W = self._w
        c = self.cfg
        Cf, H = c["conv_dim"][-1], c["hidden"]
        M = B * Tf
        if taps is not None:
            taps["features"] = feats.reshape(B, Tf, Cf).clone()
        # ---- feature projection: LayerNorm -> Linear
        cfp = _pad_to(Cf, 64)
        pn = self._planes("fp_in", (M, cfp))
        ops.layernorm(feats, W["fp_ln_w"], W["fp_ln_b"], B, Tf, Cf, eps=c["eps"], out=pn, ld=cfp, rows_per_batch=Tf, row_off=0)
        xh = self._buf("x", (M, H))
        # projected features also go, group-padded, into the positional conv's zero-padded buffer
        ops.gemm(pn, W["fp_w"], H, a_batch=1, a_rows_per_batch=M, a_ld=cfp, m_per_batch=M, bias=W["fp_b"], out_f32=rowmap(xh, H, M, 0))
        # ---- positional conv embedding: x + GELU(conv_k128_g16(x))  (HubertPositionalConvEmbedding + SamePad)
        G, K = c["pos_groups"], c["pos_k"]
        cg = H // G
        pad_l = K // 2
        rows_p = Tf + K                                       # pad_l zeros in front, K - pad_l (>= needed K - 1 - pad_l) behind
        pbuf = self._planes("pos_in", (B, rows_p, G * 64))
        xg = self._buf("pos_xg", (M, G * 64))
        xg.view(M, G, 64)[:, :, :cg].copy_(xh.view(M, G, cg))   # group-padded copy (device glue: strided copy, no arithmetic)
        ops.rows_to_planes(xg, B, Tf, G * 64, pbuf, G * 64, rows_p, pad_l)
        x1 = self._buf("x1", (M, H))
        for g in range(G):
            res = ops.RowMap(xh.data_ptr() + 4 * g * cg, H, Tf, 0)
            out = ops.RowMap(x1.data_ptr() + 4 * g * cg, H, Tf, 0)
            ops.gemm(pbuf, W["pos_w"][g], cg, a_batch=B, a_rows_per_batch=rows_p, a_ld=G * 64, m_per_batch=Tf, taps=K,
                     a_cols=64, a_col_off=64 * g, bias=W["pos_b"][g * cg:(g + 1) * cg], act=ACT_GELU, residual=res, out_f32=out)
        return x1

    # ------------------------------------------------------------------ stages
    def resample(self, wav: torch.Tensor) -> torch.Tensor:
        """torchaudio.transforms.Resample(in_rate, 16000) (audio_tokenizer.py:41,50): wav [B,T] -> [B, ceil(T / 3)]"""
        W = self._prepare()
        if self.in_rate == 16000:
            return wav
        r = W["resample"]
        B, T = wav.shape
        o, R, width = r["o"], r["R"], r["width"]
        T_out = math.ceil(T / o)
        rows = math.ceil(T_out / 64)
        # padded input [B, (rows + 1) * R]: `width` zeros in front (torchaudio pads (width, width + orig))
        xp = ops.pad_wav(wav, width, (rows + 1) * R)
        a = self._planes("rs_in", (B, rows + 1, R))
        ops.split_f16(xp, a)
        y = self._buf("rs_out", (B, rows * 64))
        ops.gemm(a, r["w"], 64, a_batch=B, a_rows_per_batch=rows + 1, a_ld=R, m_per_batch=rows, taps=2,
                 out_f32=rowmap(y, 64, rows, 0))
        return y[:, :T_out]

    def hidden_state_mean(self, wav16: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
        """pad 160/160 -> feature encoder -> projection -> positional conv -> encoder; returns the mean of the
        1 + layers hidden states [B, T', H] fp32 (audio_tokenizer.py:51-55 / model.py:43-46).  wav2vec2: no padding, the mean of
        the `hidden_state_ids` states (bicodec/audio_tokenizer.py:85-88)."""
        W = self._prepare()
        c = self.cfg
        if c.get("kind") == "wav2vec2":
            return self._wav2vec2_mean(wav16, taps)
        B, T = wav16.shape
        x = ops.pad_wav(wav16, 160, T + 320)
        Tin = T + 320
        # ---- feature encoder (HubertFeatureEncoder: conv_bias=False, feat_extract_norm='group')
        C0, k0, s0 = c["conv_dim"][0], c["conv_kernel"][0], c["conv_stride"][0]
        Tc = (Tin - k0) // s0 + 1
        s1 = c["conv_stride"][1]
        rpb = _pad_to(Tc, s1)
        cur = self._planes("fe0", (B, rpb, _pad_to(C0, 64)))
        y0 = self._buf("fe_y0", (B, Tc, C0))
        ws0 = self._buf("fe_ws0", (ops.ssl_conv0_workspace_bytes(B, Tc, C0),), torch.uint8)
        ops.ssl_conv0_gn_gelu(x, W["conv0_w"], W["gn_w"], W["gn_b"], 1e-5, k0, s0, cur, _pad_to(C0, 64), rpb, 0, y0, ws0)
        cin_pad = _pad_to(C0, 64)
        feats = None
        nconv = len(c["conv_dim"])
        for i in range(1, nconv):
            k, s, co = c["conv_kernel"][i], c["conv_stride"][i], c["conv_dim"][i]
            Tn = (Tc - k) // s + 1
            last = i == nconv - 1
            if last:
                feats = self._buf("fe_out", (B * Tn, co))
                ops.gemm(cur, W["convs"][i - 1], co, a_batch=B, a_rows_per_batch=rpb, a_ld=cin_pad, m_per_batch=Tn, taps=k, stride=s,
                         act=ACT_GELU, out_f32=rowmap(feats, co, Tn, 0))
            else:
                sn = c["conv_stride"][i + 1]
                rpb_n = _pad_to(Tn, sn)
                nxt = self._planes(f"fe{i}", (B, rpb_n, _pad_to(co, 64)))
                ops.gemm(cur, W["convs"][i - 1], co, a_batch=B, a_rows_per_batch=rpb, a_ld=cin_pad, m_per_batch=Tn, taps=k, stride=s,
                         act=ACT_GELU, out_planes=nxt, out_planes_map=(_pad_to(co, 64), rpb_n, 0))
                cur, rpb, cin_pad = nxt, rpb_n, _pad_to(co, 64)
            Tc = Tn
        Tf, H = Tc, c["hidden"]
        M = B * Tf
        x1 = self._embed(feats, B, Tf, taps)
        xs = self._buf("xs", (M, H))
        xp = self._planes("xp", (M, H))
        ops.layernorm(x1, W["enc_ln_w"], W["enc_ln_b"], B, Tf, H, eps=c["eps"], out_f32=xs, out=xp)
        acc = self._buf("hs_sum", (M, H))
        n_states = c["layers"] + 1
        ops.axpy(xs, 1.0 / n_states, acc, accumulate=False)
        if taps is not None:
            taps["hs0"] = xs.reshape(B, Tf, H).clone()
        heads, hd = c["heads"], H // c["heads"]
        qkv = self._buf("qkv", (M, 3 * H))
        att = self._planes("att", (M, H))
        hid = self._planes("hid", (M, c["ffn"]))
        t32 = self._buf("t32", (M, H))
        cos, sin = self._identity_rope(Tf, hd)
        wavlm = c.get("kind") == "wavlm"
        att_ws = None if wavlm else self._buf("att5_ws", (ops.self_attention_workspace_bytes(B, Tf, heads, hd, True),), torch.uint8)
        if wavlm:
            rel_table = self._cached(("rel", Tf), lambda: self._rel_table(Tf))
            gate = self._buf("gate", (B, heads, Tf))
        for li, L in enumerate(W["layers"]):
            ops.gemm(xp, L["wqkv"], 3 * H, a_batch=1, a_rows_per_batch=M, a_ld=H, m_per_batch=M, bias=L["bqkv"],
                     out_f32=rowmap(qkv, 3 * H, M, 0))
            if wavlm:        # gated relative position bias from the layer INPUT (WavLMAttention.forward)
                ops.wavlm_gate(xs, B, Tf, heads, hd, L["gru_w"], L["gru_b"], L["gru_c"], gate)
                ops.attention_relbias(qkv, B, Tf, heads, hd, rel_table, gate, att)
            else:
                ops.self_attention(qkv, B, Tf, heads, hd, cos, sin, att, att_ws, True)
            ops.gemm(att, L["wo"], H, a_batch=1, a_rows_per_batch=M, a_ld=H, m_per_batch=M, bias=L["bo"],
                     residual=rowmap(xs, H, M, 0), out_f32=rowmap(t32, H, M, 0))
            ops.layernorm(t32, L["ln_w"], L["ln_b"], B, Tf, H, eps=c["eps"], out_f32=xs, out=xp)
            ops.gemm(xp, L["w1"], c["ffn"], a_batch=1, a_rows_per_batch=M, a_ld=H, m_per_batch=M, bias=L["b1"], act=ACT_GELU,
                     out_planes=hid, out_planes_map=(c["ffn"], M, 0))
            ops.gemm(hid, L["w2"], H, a_batch=1, a_rows_per_batch=M, a_ld=c["ffn"], m_per_batch=M, bias=L["b2"],
                     residual=rowmap(xs, H, M, 0), out_f32=rowmap(t32, H, M, 0))
            ops.layernorm(t32, L["fln_w"], L["fln_b"], B, Tf, H, eps=c["eps"], out_f32=xs, out=xp)
            ops.axpy(xs, 1.0 / n_states, acc, accumulate=True)
            if taps is not None:
                taps[f"hs{li + 1}"] = xs.reshape(B, Tf, H).clone()
        return acc.reshape(B, Tf, H)

    def min_samples(self) -> int:
        """receptive field of the conv stack: the shortest input that yields one frame (400 samples for XLSR-53)"""
        n, hop = self.cfg["conv_kernel"][0], 1
        for k, s in zip(self.cfg["conv_kernel"][1:], self.cfg["conv_stride"]):
            hop *= s
            n += (k - 1) * hop
        return n

    def _wav2vec2_mean(self, wav16: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
        """Wav2Vec2Model (conv_bias, feat_extract_norm="layer", do_stable_layer_norm): feature encoder -> projection -> positional
        conv -> pre-LN layers; returns the mean of hidden_states[k] for k in `hidden_state_ids` [B, T', H] fp32."""
        W = self._w
        c = self.cfg
        B, Tin = wav16.shape
        if Tin < self.min_samples():
            raise ValueError(f"wav2vec2 needs at least {self.min_samples()} samples per utterance (the conv stack's receptive "
                             f"field), got {Tin}")
        # ---- feature encoder: conv + bias -> LayerNorm over channels -> GELU, 7 times (Wav2Vec2LayerNormConvLayer, eps 1e-5)
        C0, k0, s0 = c["conv_dim"][0], c["conv_kernel"][0], c["conv_stride"][0]
        Tc = (Tin - k0) // s0 + 1
        y = self._buf("fe_y0", (B, Tc, C0))
        ops.ssl_conv0_bias(wav16, W["conv0_w"], W["conv_b"][0], k0, s0, y)
        nconv = len(c["conv_dim"])
        for i in range(nconv - 1):
            co, cn, k, s = c["conv_dim"][i], c["conv_dim"][i + 1], c["conv_kernel"][i + 1], c["conv_stride"][i + 1]
            rpb, cpad = _pad_to(Tc, s), _pad_to(co, 64)
            cur = self._planes(f"fe{i}", (B, rpb, cpad))
            ops.layernorm_act(y, *W["conv_ln"][i], B, Tc, co, ACT_GELU, eps=1e-5, out=cur, ld=cpad, rows_per_batch=rpb, row_off=0)
            Tn = (Tc - k) // s + 1
            y = self._buf(f"fe_y{i + 1}", (B, Tn, cn))
            ops.gemm(cur, W["convs"][i], cn, a_batch=B, a_rows_per_batch=rpb, a_ld=cpad, m_per_batch=Tn, taps=k, stride=s,
                     bias=W["conv_b"][i + 1], out_f32=rowmap(y, cn, Tn, 0))
            Tc = Tn
        Tf, Cf, H = Tc, c["conv_dim"][-1], c["hidden"]
        M = B * Tf
        feats = self._buf("fe_out", (M, Cf))
        ops.layernorm_act(y, *W["conv_ln"][-1], B, Tf, Cf, ACT_GELU, eps=1e-5, out_f32=feats)
        x = self._embed(feats, B, Tf, taps)                      # hidden_states[0]: no LayerNorm before the pre-LN layers
        x2 = self._buf("x2", (M, H))
        ids = c["hidden_state_ids"]
        acc = self._buf("hs_sum", (M, H))
        first = True
        if 0 in ids:
            ops.axpy(x, 1.0 / len(ids), acc, accumulate=False)
            first = False
        if taps is not None:
            taps["hs0"] = x.reshape(B, Tf, H).clone()
        heads, hd = c["heads"], H // c["heads"]
        qkv = self._buf("qkv", (M, 3 * H))
        xp = self._planes("xp", (M, H))
        att = self._planes("att", (M, H))
        hid = self._planes("hid", (M, c["ffn"]))
        cos, sin = self._identity_rope(Tf, hd)
        att_ws = self._buf("att5_ws", (ops.self_attention_workspace_bytes(B, Tf, heads, hd, True),), torch.uint8)
        for li, L in enumerate(W["layers"]):                      # Wav2Vec2EncoderLayerStableLayerNorm; x <-> x2 ping-pong
            ops.layernorm(x, L["ln_w"], L["ln_b"], B, Tf, H, eps=c["eps"], out=xp)
            ops.gemm(xp, L["wqkv"], 3 * H, a_batch=1, a_rows_per_batch=M, a_ld=H, m_per_batch=M, bias=L["bqkv"],
                     out_f32=rowmap(qkv, 3 * H, M, 0))
            ops.self_attention(qkv, B, Tf, heads, hd, cos, sin, att, att_ws, True)
            ops.gemm(att, L["wo"], H, a_batch=1, a_rows_per_batch=M, a_ld=H, m_per_batch=M, bias=L["bo"],
                     residual=rowmap(x, H, M, 0), out_f32=rowmap(x2, H, M, 0))
            ops.layernorm(x2, L["fln_w"], L["fln_b"], B, Tf, H, eps=c["eps"], out=xp)
            ops.gemm(xp, L["w1"], c["ffn"], a_batch=1, a_rows_per_batch=M, a_ld=H, m_per_batch=M, bias=L["b1"], act=ACT_GELU,
                     out_planes=hid, out_planes_map=(c["ffn"], M, 0))
            ops.gemm(hid, L["w2"], H, a_batch=1, a_rows_per_batch=M, a_ld=c["ffn"], m_per_batch=M, bias=L["b2"],
                     residual=rowmap(x2, H, M, 0), out_f32=rowmap(x, H, M, 0))
            if li + 1 in ids:
                ops.axpy(x, 1.0 / len(ids), acc, accumulate=not first)
                first = False
            if taps is not None:
                taps[f"hs{li + 1}"] = x.reshape(B, Tf, H).clone()
        return acc.reshape(B, Tf, H)

    def normalize(self, wav: torch.Tensor) -> torch.Tensor:
        """Wav2Vec2FeatureExtractor(do_normalize=True): each utterance to zero mean, unit (population) variance, eps 1e-7"""
        out = torch.empty_like(wav)
        ops.wav_normalize(wav, 1e-7, out)
        return out

    @torch.no_grad()
    def forward(self, wavs: torch.Tensor, channel_first: bool = False, taps: Optional[dict] = None) -> torch.Tensor:
        """extract_ssl_features / extract_semantic_features: wavs [B, T] at `in_rate` -> [B, T', H] (or [B, H, T'])."""
        if wavs.device.type != "cuda":
            raise RuntimeError("unified_audio_b200.SSLFrontEnd runs on CUDA only (no CPU fallback)")
        w16 = self.resample(wavs.float().contiguous())
        if self.cfg.get("do_normalize"):
            w16 = self.normalize(w16.contiguous())
        mean = self.hidden_state_mean(w16.contiguous(), taps)
        if taps is not None:
            taps["mean"] = mean.clone()
        B, Tf, H = mean.shape
        out = torch.empty((B, H, Tf) if channel_first else (B, Tf, H), device=mean.device)
        ops.ssl_compress(mean, B, Tf, H, 0.3 if self.compress else 0.0, channel_first, out)
        return out


def pad_wav(wav: torch.Tensor, hop_length: int) -> torch.Tensor:
    """HCodecTokenizer.pad_wav (audio_tokenizer.py:63-66): zero-pad the tail to a multiple of hop_length, on the device."""
    T = wav.shape[-1]
    return ops.pad_wav(wav, 0, math.ceil(T / hop_length) * hop_length)


def wrap_segments(src: torch.Tensor, seg_len: int) -> torch.Tensor:
    """U/model/model.py:175-181: np.pad(src, [(0,0),(0,pad_len)], 'wrap') then reshape(-1, seg_len), without the NumPy round trip."""
    T = src.shape[-1]
    total = math.ceil(T / seg_len) * seg_len
    return ops.pad_wav(src, 0, total, wrap=True).reshape(-1, seg_len)


class HCodecTokenizer(nn.Module):
    """HCodecTokenizer (audio_tokenizer.py:21-79) on the device end to end: pad_wav -> Resample + HuBERT features -> Codec.encode."""

    def __init__(self, codec, feature_extractor: SSLFrontEnd, sampling_rate: int = 48000, target_frame_rate: float = 12.5):
        super().__init__()
        self.model, self.feature_extractor = codec, feature_extractor
        self.hop_length = int(sampling_rate / target_frame_rate)

    @torch.no_grad()
    def extract_ssl_features(self, wavs):
        return self.feature_extractor(wavs)

    def pad_wav(self, wav):
        return pad_wav(wav, self.hop_length)

    @torch.no_grad()
    def tokenize(self, wav):
        wav = self.pad_wav(wav)
        feats = self.feature_extractor(wav, channel_first=True)        # (b, d, t) written channel-first by the kernel
        return self.model.encode(wav, feats)

    @torch.no_grad()
    def detokenize(self, acoustic_codes, semantic_codes):
        return self.model.decode(acoustic_codes, semantic_codes)


def _check_front_end(face: str, codec, fe: SSLFrontEnd, kind: str):
    """the front-end settings a 16 kHz H-Codec tokenizer needs; each mismatch would give plausible codes with no error"""
    c = fe.cfg
    if c.get("kind", "hubert") != kind:                 # SSLFrontEnd runs a config without `kind` as HuBERT
        raise ValueError(f"{face} needs a {kind} front end, got kind={c.get('kind')!r}")
    if fe.in_rate != 16000:
        raise ValueError(f"{face} takes 16 kHz audio: the front end must have in_rate=16000, got {fe.in_rate}")
    if not fe.compress:
        raise ValueError(f"{face} feeds sign(x)|x|^0.3 features to the codec: build the front end with compress=True")
    if c["hidden"] != codec.c["sem_in"]:
        raise ValueError(f"{face}: the front end's hidden width {c['hidden']} differs from the codec's semantic-encoder input "
                         f"width {codec.c['sem_in']}")


def _check_wav(face: str, wav):
    if not isinstance(wav, torch.Tensor) or wav.ndim != 2:
        raise ValueError(f"{face}: wav must be a [B, T] tensor, got {tuple(wav.shape) if isinstance(wav, torch.Tensor) else type(wav)}")
    if wav.device.type != "cuda":
        raise RuntimeError(f"unified_audio_b200.{face} runs on CUDA only (no CPU fallback)")


class HCodecTokenizerH1(nn.Module):
    """HCodecTokenizer of H-Codec-1.0 (HCodec-1.0/audio_tokenizer.py:18-66) on the device: pad_wav to a multiple of 640 ->
    pad 160/160 + HuBERT-base, mean of the 13 hidden states, sign(x)|x|^0.3 (16 kHz in, no resampling) -> CodecH1.encode.

    codec: CodecH1; feature_extractor: SSLFrontEnd(HUBERT_BASE, in_rate=16000, compress=True)."""

    hop_length = 640                    # audio_tokenizer.py:31 (25 Hz); CodecH1's SEANet strides are fixed

    def __init__(self, codec, feature_extractor: SSLFrontEnd):
        super().__init__()
        if not isinstance(codec, CodecH1) or isinstance(codec, CodecH15):
            raise ValueError(f"HCodecTokenizerH1 needs a CodecH1, got {type(codec).__name__}")
        _check_front_end("HCodecTokenizerH1", codec, feature_extractor, "hubert")
        self.model, self.feature_extractor = codec, feature_extractor

    def pad_wav(self, wav):
        return pad_wav(wav, self.hop_length)

    @torch.no_grad()
    def extract_wav2vec2_features(self, wavs):
        """audio_tokenizer.py:35-49 (HuBERT despite the name): wavs [B, T] -> [B, T/320, 768]"""
        _check_wav("HCodecTokenizerH1", wavs)
        return self.feature_extractor(wavs)

    @torch.no_grad()
    def tokenize(self, wav):
        """audio_tokenizer.py:56-61: wav [B, T] @ 16 kHz -> (acoustic, semantic) int64 [B, nq, ceil(T / 640)]"""
        _check_wav("HCodecTokenizerH1", wav)
        wav = self.pad_wav(wav)
        feats = self.feature_extractor(wav, channel_first=True)        # (b, d, t) written channel-first by the kernel
        return self.model.encode(wav[:, None], feats)

    @torch.no_grad()
    def detokenize(self, acoustic_codes, semantic_codes):
        """audio_tokenizer.py:63-66: -> wav [B, N * 640]"""
        return self.model.decode(acoustic_codes, semantic_codes)


class HCodecTokenizerH15(nn.Module):
    """HCodecTokenizer of H-Codec-1.5 (HCodec-1.5/audio_tokenizer.py:38-86) on the device: pad_wav to a multiple of
    prod(ratios) * 2 -> pad 160/160 + wav2vec2-large-xlsr-53 called bare (no processor normalisation), (hs[11] + hs[14] +
    hs[16]) / 3, sign(x)|x|^0.3 -> the adaptive CodecH15.encode with the codec's own threshold (length-packed codes).

    codec: CodecH15; feature_extractor: SSLFrontEnd(WAV2VEC2_XLSR53_RAW, in_rate=16000, compress=True)."""

    def __init__(self, codec, feature_extractor: SSLFrontEnd):
        super().__init__()
        if not isinstance(codec, CodecH15):
            raise ValueError(f"HCodecTokenizerH15 needs a CodecH15, got {type(codec).__name__}")
        _check_front_end("HCodecTokenizerH15", codec, feature_extractor, "wav2vec2")
        if feature_extractor.cfg.get("do_normalize"):
            raise ValueError("HCodecTokenizerH15: the reference calls wav2vec2 without processor normalisation; build the front end "
                             "from WAV2VEC2_XLSR53_RAW (do_normalize=False)")
        self.model, self.feature_extractor = codec, feature_extractor
        self.hop_length = math.prod(codec.c["ratios"]) * 2             # audio_tokenizer.py:71

    def pad_wav(self, wav):
        return pad_wav(wav, self.hop_length)

    def _features(self, wavs, channel_first):
        T = wavs.shape[-1]
        return self.feature_extractor(ops.pad_wav(wavs, 160, T + 320), channel_first=channel_first)

    @torch.no_grad()
    def extract_wav2vec2_features(self, wavs):
        """audio_tokenizer.py:52-66: wavs [B, T] -> pad 160/160 -> [B, T/320, 1024]"""
        _check_wav("HCodecTokenizerH15", wavs)
        return self._features(wavs, False)

    @torch.no_grad()
    def tokenize(self, wav):
        """audio_tokenizer.py:76-81: wav [B, T] @ 16 kHz -> {'acoustic_codes', 'semantic_codes'} int64 [B, nq, G], token lengths
        packed into the indices as CodecH15.encode returns them"""
        _check_wav("HCodecTokenizerH15", wav)
        wav = self.pad_wav(wav)
        return self.model.encode(wav[:, None], self._features(wav, True))

    @torch.no_grad()
    def detokenize(self, acoustic_codes, semantic_codes, token_lengths=None):
        """audio_tokenizer.py:83-86"""
        return self.model.decode(acoustic_codes, semantic_codes, token_lengths)
