"""H-Codec-2.0 `Codec` with the reference's surface, running on libquark_b200.

Mirrors QuarkAudio-HCodec/HCodec-2.0/vq/codec.py:17-99:
    Codec(encoder_kwargs, decoder_kwargs, quantizer_kwargs, semantic_encoder_kwargs, semantic_decoder_kwargs)
    Codec.encode(x [B,T], feat [B,768,T50]) -> (acoustic_codes, semantic_codes)  int64 [B,nq,N]
    Codec.decode(acoustic_codes, semantic_codes)  -> wav [B, N*3840]
state_dict keys/shapes are the reference's (spec.py); `semantic_decoder.*` keys (training-only module,
codec.py:71) are accepted by load_state_dict and ignored.

Host code is orchestration only: every arithmetic op is a libquark_b200 kernel launched on the current
CUDA stream; activations stay channel-last [B*T, C] end to end (the reference transposes ~120 times per
pass).  There is no PyTorch / CPU fallback.
"""
from __future__ import annotations

import math
import os
from typing import Dict, Optional

import torch
from torch import nn

from . import ops, spec
from .ops import ACT_ELU, ACT_GELU, ACT_NONE, ACT_SWIGLU, Planes, rowmap
from .rvq import ResidualVQ

# GEMM groups -> 3-term split (True) or single-pass fp16 (False).  Evidence: oracle/precision_study.py,
# DESIGN.md "precision policy".
PRECISION_POLICIES = {
    "mixed": dict(convnext=False, lstm_attn=False, mlp=True, mlp_dec=True, conv=True, head=True, dft=True),
    # decoder-side transformer MLP single-pass (it sits behind the RVQ indices, only the waveform budget applies):
    # measured on the shipped config 121.3 vs 125.4 ms per step, waveform error 6.5e-4 vs 2.3e-4 - inside 1e-3 but with
    # 1.5x instead of 4x margin, hence not the default
    "mixed_dec16": dict(convnext=False, lstm_attn=False, mlp=True, mlp_dec=False, conv=True, head=True, dft=True),
    "accurate": dict(convnext=True, lstm_attn=True, mlp=True, mlp_dec=True, conv=True, head=True, dft=True),
    "fast": dict(convnext=False, lstm_attn=False, mlp=False, mlp_dec=False, conv=False, head=False, dft=True),
}


class _Tree(nn.Module):
    """Bare parameter container whose nested attribute names reproduce the reference's module tree."""

    @staticmethod
    def build(specs: Dict[str, tuple]) -> "_Tree":
        root = _Tree()
        for name, shape in specs.items():
            node = root
            parts = name.split(".")
            for p in parts[:-1]:
                if p not in node._modules:
                    node.add_module(p, _Tree())
                node = node._modules[p]
            if name in spec.BUFFERS:
                node.register_buffer(parts[-1], torch.hann_window(shape[0]))
            else:
                node.register_parameter(parts[-1], nn.Parameter(torch.zeros(shape), requires_grad=False))
        return root


def _pad_to(n, m):
    return (n + m - 1) // m * m


class Codec(nn.Module):
    def __init__(self, encoder_kwargs: dict, decoder_kwargs: dict, quantizer_kwargs: dict,
                 semantic_encoder_kwargs: dict, semantic_decoder_kwargs: Optional[dict] = None,
                 precision: str = "mixed"):
        super().__init__()
        self.enc_cfg, self.dec_cfg = dict(encoder_kwargs), dict(decoder_kwargs)
        self.sem_cfg = dict(semantic_encoder_kwargs)
        self.encoder = _Tree.build(spec.encoder_spec(**encoder_kwargs))
        self.decoder = _Tree.build(spec.decoder_spec(**decoder_kwargs))
        self.quantizer = ResidualVQ(**quantizer_kwargs)
        self.semantic_quantizer = ResidualVQ(**quantizer_kwargs)
        self.semantic_encoder = _Tree.build(spec.semantic_encoder_spec(**semantic_encoder_kwargs))
        self.policy = dict(PRECISION_POLICIES[precision])
        self._w = None        # repacked weights (device planes) of the Python-orchestrated path
        self._ws = {}         # workspace cache
        self.precision = precision
        # "c" (default): encode / decode are ONE call each into the handle-level C ABI (csrc/engine.cu owns the weight arena, the
        # workspace and the ~340-kernel orchestration).  "python": the same kernels launched op by op from this file - kept as the
        # cross-check of the engine (tests/test_engine_gpu.py) and as the base CodecH1 builds on.
        self.engine_mode = os.environ.get("QB_CODEC_ENGINE", "c")
        self._engine = None
        self.eval()

    # ------------------------------------------------------------------ state handling
    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        sd = {k: v for k, v in state_dict.items() if not k.startswith("semantic_decoder.")}
        r = super().load_state_dict(sd, strict=strict, assign=assign)
        self._w, self._engine = None, None
        return r

    def _apply(self, fn, *a, **k):
        self._w, self._ws, self._engine = None, {}, None
        return super()._apply(fn, *a, **k)

    def _use_engine(self) -> bool:
        return self.engine_mode == "c" and type(self) is Codec

    def engine(self):
        """The qb_codec handle of this model (built lazily from the current parameters)."""
        if self._engine is None:
            from .engine import CodecEngine
            dev = next(self.parameters()).device
            if dev.type != "cuda":
                raise RuntimeError("unified_audio_b200.Codec runs on CUDA only (no CPU fallback): call .cuda() first")
            self._engine = CodecEngine(dev, self.enc_cfg, self.dec_cfg, dict(num_quantizers=self.quantizer.num_quantizers,
                                                                             codebook_size=self.quantizer.codebook_size),
                                       self.sem_cfg, self.precision, {k: v for k, v in self.state_dict().items()})
        return self._engine

    # ------------------------------------------------------------------ weight repack (load time)
    def _prepare(self):
        if self._w is not None:
            return self._w
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("unified_audio_b200.Codec runs on CUDA only (no CPU fallback): call .cuda() first")
        pol = self.policy
        W: Dict[str, object] = {}

        def conv_w(key, group):
            w = sd[key].float()                                   # [Cout, Cin, k]
            cout, cin, k = w.shape
            cpad = _pad_to(cin, 64)
            wp = torch.zeros(cout, k, cpad, device=dev)
            wp[:, :, :cin] = w.permute(0, 2, 1)
            return Planes.from_f32(wp.reshape(cout, k * cpad), pol[group])

        def lin_w(w, group):
            return Planes.from_f32(w.float().contiguous(), pol[group])

        def f32(key):
            return sd[key].float().contiguous()

        def convnext(prefix, n):
            blocks = []
            for i in range(n):
                p = f"{prefix}{i}."
                blocks.append(dict(
                    dw_w=sd[p + "dwconv.conv.weight"].float().reshape(-1, 7).contiguous(), dw_b=f32(p + "dwconv.conv.bias"),
                    ln_w=f32(p + "norm.weight"), ln_b=f32(p + "norm.bias"),
                    w1=lin_w(sd[p + "pwconv1.linear.weight"], "convnext"), b1=f32(p + "pwconv1.linear.bias"),
                    w2=lin_w(sd[p + "pwconv2.linear.weight"], "convnext"), b2=f32(p + "pwconv2.linear.bias"),
                    gamma=f32(p + "gamma")))
            return blocks

        def transformer(prefix, n, mlp_group="mlp"):
            layers = []
            hdim = sd[f"{prefix}layers.0.self_attn.rnn.weight_hh_l0"].shape[1]
            lstm_u = ops.lstm_tc_units(hdim) if hdim % 256 == 0 else 0
            for i in range(n):
                p = f"{prefix}layers.{i}."
                a = p + "self_attn."
                w13 = torch.stack([sd[p + "mlp.w1.weight"].float(), sd[p + "mlp.w3.weight"].float()], 1)
                layers.append(dict(
                    in_w=f32(p + "input_layernorm.weight"), post_w=f32(p + "post_attention_layernorm.weight"),
                    wih=lin_w(sd[a + "rnn.weight_ih_l0"], "lstm_attn"),
                    b_ih=(sd[a + "rnn.bias_ih_l0"].float() + sd[a + "rnn.bias_hh_l0"].float()).contiguous(),
                    whh=Planes.from_f32(sd[a + "rnn.weight_hh_l0"].float().contiguous(), False),
                    whh_perm=(ops.lstm_tc_permute(sd[a + "rnn.weight_hh_l0"], lstm_u) if lstm_u else None),
                    wqkv=lin_w(torch.cat([sd[a + f"{n_}_proj.weight"].float() for n_ in "qkv"], 0), "lstm_attn"),
                    bqkv=torch.cat([sd[a + f"{n_}_proj.bias"].float() for n_ in "qkv"], 0).contiguous(),
                    wo=lin_w(sd[a + "o_proj.weight"], "lstm_attn"),
                    w13=lin_w(w13.reshape(-1, w13.shape[-1]), mlp_group),      # rows interleaved gate/up
                    w2=lin_w(sd[p + "mlp.w2.weight"], mlp_group)))
            return layers

        e, d = self.enc_cfg, self.dec_cfg
        n_fft, hop = e.get("n_fft", 1920), e.get("hop_length", 960)
        if n_fft != 2 * hop or hop % 64 != 0:
            raise RuntimeError("the STFT/ISTFT kernels assume n_fft == 2*hop and hop % 64 == 0 (shipped config)")
        if d.get("n_fft", 1920) != n_fft or d.get("hop_length", 960) != hop:
            raise RuntimeError("encoder / decoder STFT geometry must match")
        nf = n_fft // 2 + 1
        # forward DFT (window folded in), rows = [re_0..re_nf-1, im_0..im_nf-1], K = n_fft (two hop-block taps)
        s = torch.arange(n_fft, dtype=torch.int64, device=dev)
        k = torch.arange(nf, dtype=torch.int64, device=dev)
        ang = 2.0 * math.pi * (torch.outer(k, s) % n_fft).double() / n_fft      # exact argument reduction
        win = sd["encoder.stft.window"].double()
        fwd = torch.cat([torch.cos(ang) * win, -torch.sin(ang) * win], 0)
        W["dft_fwd"] = _planes_from_f64(fwd, True)
        W["stft2"] = _stft2_weights(n_fft, sd["encoder.stft.window"].float().contiguous(), dev)
        # inverse real DFT (1/N, Hermitian weights c_k, synthesis window folded in), K padded to a multiple of 64
        kin = _pad_to(2 * nf, 64)
        ck = torch.full((nf,), 2.0, dtype=torch.float64, device=dev)
        ck[0] = 1.0
        ck[-1] = 1.0
        wini = sd["decoder.head.istft.window"].double()
        inv = torch.zeros(n_fft, kin, dtype=torch.float64, device=dev)
        angT = ang.t()                                              # [n, k]
        inv[:, :nf] = torch.cos(angT) * ck / n_fft * wini[:, None]
        im = -torch.sin(angT) * ck / n_fft * wini[:, None]
        im[:, 0] = 0.0
        im[:, -1] = 0.0                                             # irfft ignores imag of DC / Nyquist
        inv[:, nf:2 * nf] = im
        W["dft_inv"] = _planes_from_f64(inv, True)
        W["istft_window"] = sd["decoder.head.istft.window"].float().contiguous()
        W["geom"] = dict(n_fft=n_fft, hop=hop, nf=nf, feat_ld=_pad_to(2 * nf, 64), spec_ld=_pad_to(2 * nf, 4), kin=kin)

        W["enc"] = dict(
            embed=conv_w("encoder.embed.conv.weight", "conv"), embed_b=f32("encoder.embed.conv.bias"),
            norm_w=f32("encoder.norm.weight"), norm_b=f32("encoder.norm.bias"),
            convnext=convnext("encoder.prior_net.", e["convnext_layers"]),
            tf=transformer("encoder.post_net.1.", e.get("transformer_layers", 2)),
            fnorm_w=f32("encoder.final_layer_norm.weight"), fnorm_b=f32("encoder.final_layer_norm.bias"),
            out=conv_w("encoder.out.conv.weight", "conv"), out_b=f32("encoder.out.conv.bias"),
            stride=int(50 / e["target_frame_rate"]))
        sem = self.sem_cfg
        blocks = []
        if any(float(r) != 1.0 for r in sem["channel_ratios"]):
            raise RuntimeError("semantic encoder: only channel_ratios == 1 (shipped config) is implemented")
        for i, st in enumerate(sem["strides"]):
            p = f"semantic_encoder.conv_blocks.{i}."
            blocks.append(dict(
                units=[dict(c1=conv_w(p + f"res_units.{u}.conv1.conv.weight", "conv"),
                            c2=conv_w(p + f"res_units.{u}.conv2.weight", "conv")) for u in (0, 1)],
                conv=conv_w(p + "conv.conv.weight", "conv"), conv_b=f32(p + "conv.conv.bias"), stride=st,
                k=3 if st == 1 else 2 * st))
        W["sem"] = dict(conv=conv_w("semantic_encoder.conv.conv.weight", "conv"), blocks=blocks,
                        conv2=conv_w("semantic_encoder.conv2.conv.weight", "conv"))
        res = {}
        for i in (0, 1, 5, 6):
            p = f"decoder.prior_net.{i}."
            res[i] = dict(n1w=f32(p + "norm1.weight"), n1b=f32(p + "norm1.bias"), n2w=f32(p + "norm2.weight"),
                          n2b=f32(p + "norm2.bias"), c1=conv_w(p + "conv1.conv.weight", "conv"),
                          c1b=f32(p + "conv1.conv.bias"), c2=conv_w(p + "conv2.conv.weight", "conv"),
                          c2b=f32(p + "conv2.conv.bias"))
        W["dec"] = dict(
            embed=conv_w("decoder.embed.conv.weight", "conv"), embed_b=f32("decoder.embed.conv.bias"),
            res=res, tf=transformer("decoder.prior_net.3.", d.get("transformer_layers", 2), "mlp_dec"),
            gn_w=f32("decoder.prior_net.7.weight"), gn_b=f32("decoder.prior_net.7.bias"),
            norm_w=f32("decoder.norm.weight"), norm_b=f32("decoder.norm.bias"),
            convnext=convnext("decoder.post_net.", d["convnext_layers"]),
            fnorm_w=f32("decoder.final_layer_norm.weight"), fnorm_b=f32("decoder.final_layer_norm.bias"),
            head=lin_w(sd["decoder.head.out.weight"], "head"), head_b=f32("decoder.head.out.bias"),
            factor=int(50 / d["target_frame_rate"]))
        self._w = W
        return W

    # ------------------------------------------------------------------ workspace
    def _buf(self, name, shape, dtype=torch.float32):
        key = (name, tuple(shape), dtype)
        t = self._ws.get(key)
        if t is None:
            t = torch.zeros(shape, dtype=dtype, device=next(self.parameters()).device)
            self._ws[key] = t
        return t

    def _planes(self, name, shape, split):
        key = ("P", name, tuple(shape), bool(split))
        p = self._ws.get(key)
        if p is None:
            p = Planes.zeros(shape, split, next(self.parameters()).device)
            self._ws[key] = p
        return p

    def _rope(self, T, D=64):
        key = ("rope", T, D)
        r = self._ws.get(key)
        if r is None:
            inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
            fr = torch.arange(T).float()[:, None] * inv[None, :]
            emb = torch.cat((fr, fr), dim=-1)
            dev = next(self.parameters()).device
            r = (emb.cos().to(dev).contiguous(), emb.sin().to(dev).contiguous())
            self._ws[key] = r
        return r

    # ------------------------------------------------------------------ shared blocks
    def _linear(self, a, w, n, M, K, **kw):
        ops.gemm(a, w, n, a_batch=1, a_rows_per_batch=M, a_ld=K, m_per_batch=M, **kw)

    def _convnext(self, blocks, x, B, F, C, I):
        M = B * F
        pol = self.policy["convnext"]
        t1 = self._planes("cnx_t1", (M, C), pol)
        hid = self._planes("cnx_hid", (M, I), pol)
        xm = rowmap(x, C, M, 0)
        for blk in blocks:
            ops.dwconv7_ln(x, blk["dw_w"], blk["dw_b"], blk["ln_w"], blk["ln_b"], B, F, C, t1)
            self._linear(t1, blk["w1"], I, M, C, bias=blk["b1"], act=ACT_GELU, out_planes=hid, out_planes_map=(I, M, 0))
            self._linear(hid, blk["w2"], C, M, I, bias=blk["b2"], gamma=blk["gamma"], residual=xm, out_f32=xm)

    def _transformer(self, layers, x, B, F, C, heads=None, mlp_group="mlp"):
        """encoder_modules/transformer.py:367-393 per layer; x [B*F, C] fp32 updated in place."""
        heads = heads or C // 64
        hd = C // heads
        M, I = B * F, min(4 * C, 4096)
        pa, pm = self.policy["lstm_attn"], self.policy[mlp_group]
        t_a = self._planes("tf_a", (M, C), pa)
        t_b = self._planes("tf_b", (M, C), pa)
        t_m = self._planes("tf_m", (M, C), pm)
        hid = self._planes("tf_hid", (M, I), pm)
        xp = self._buf("tf_xp", (M, 4 * C))
        qkv = self._buf("tf_qkv", (M, 3 * C))
        use_tc = layers[0]["whh_perm"] is not None and B <= 256
        ws = self._buf("lstm_ws", (max(ops.lstm_workspace_bytes(B, C), ops.lstm_tc_workspace_bytes(B, C)),), torch.uint8)
        lstm_u = ops.lstm_tc_units(C) if use_tc else 0
        cos, sin = self._rope(F, hd)
        legacy = os.environ.get("QB_ATTENTION", "umma") == "legacy"
        umma = (not legacy) and hd in (64, 128)          # wgmma attention (csrc/attention_umma.cu), both precision policies
        tc_att = (not umma) and (not pa) and hd == 64
        att_ws = (self._buf("att5_ws", (ops.attention_umma_workspace_bytes(B, F, heads, hd, pa),), torch.uint8) if umma else
                  self._buf("att_ws", (ops.attention_tc_workspace_bytes(B, F, heads),), torch.uint8) if tc_att else None)
        xm = rowmap(x, C, M, 0)
        for L in layers:
            ops.rmsnorm(x, L["in_w"], M, C, t_a)
            self._linear(t_a, L["wih"], 4 * C, M, C, bias=L["b_ih"], out_f32=rowmap(xp, 4 * C, M, 0))
            if use_tc:
                ops.lstm_tc(xp, L["whh_perm"], lstm_u, B, F, C, t_b, ws)
            else:
                ops.lstm(xp, L["whh"], B, F, C, t_b, ws)
            self._linear(t_b, L["wqkv"], 3 * C, M, C, bias=L["bqkv"], out_f32=rowmap(qkv, 3 * C, M, 0))
            if umma:
                ops.attention_umma(qkv, B, F, heads, hd, cos, sin, t_a, att_ws, split=pa)
            elif tc_att:   # legacy: single-pass fp16 policy, head_dim 64: mma.sync flash attention
                ops.attention_tc(qkv, B, F, heads, cos, sin, t_a, att_ws)
            else:        # split-precision policy or head_dim 96: fp32 SIMT attention
                ops.attention_hd(qkv, B, F, heads, hd, cos, sin, t_a)
            self._linear(t_a, L["wo"], C, M, C, residual=xm, out_f32=xm)
            ops.rmsnorm(x, L["post_w"], M, C, t_m)
            self._linear(t_m, L["w13"], 2 * I, M, C, act=ACT_SWIGLU, out_planes=hid, out_planes_map=(I, M, 0))
            self._linear(hid, L["w2"], C, M, I, residual=xm, out_f32=xm)

    # ------------------------------------------------------------------ encoder
    def _encode_emb(self, wav: torch.Tensor, taps=None):
        """vq/codec_encoder.py:62-79 -> emb [B*N, dimension] fp32 (channel-last)."""
        W = self._prepare()
        g, E = W["geom"], W["enc"]
        e = self.enc_cfg
        B, T = wav.shape
        hop, nf, n_fft = g["hop"], g["nf"], g["n_fft"]
        stride = E["stride"]
        if T % (hop * stride) != 0:
            raise ValueError(f"waveform length {T} must be a multiple of {hop * stride} (pad_wav, audio_tokenizer.py:63-66)")
        F = T // hop
        N = F // stride
        C, I, Dq = e["dim"], e["intermediate_dim"], e["dimension"]
        M = B * F
        pc, pd = self.policy["conv"], self.policy["dft"]
        wav = wav.float().contiguous()
        feat = self._planes("enc_feat", (B, F + 2, g["feat_ld"]), pc)
        s2 = W["stft2"]
        if s2 is not None and os.environ.get("QB_STFT", "fft") == "fft":
            # two-stage DFT (csrc/elementwise.cu "two-stage STFT"): MMA chains of 4 / 8 instead of 120 -> fp32-FFT-grade spectrum
            P, Q = s2["P"], s2["Q"]
            ga = self._planes("enc_sg", (M * Q, 64), True)
            ops.stft_gather(wav, hop, n_fft, P, Q, s2["window"], ga)
            Y = self._buf("enc_sy", (M * Q, 2 * P))
            ops.gemm(ga, s2["wA"], 2 * P, a_batch=1, a_rows_per_batch=M * Q, a_ld=64, m_per_batch=M * Q, out_f32=rowmap(Y, 2 * P, M * Q, 0))
            Z = self._planes("enc_sz", (M * P, 128), True)
            ops.stft_twiddle(Y, 2 * P, M, P, Q, s2["tw"], Z)
            X = self._buf("enc_sx", (M * P, s2["ldX"]))
            ops.gemm(Z, s2["wB"], s2["nB"], a_batch=1, a_rows_per_batch=M * P, a_ld=128, m_per_batch=M * P,
                     out_f32=rowmap(X, s2["ldX"], M * P, 0))
            ops.stft_post2(X, s2["ldX"], B, F, nf, P, feat, g["feat_ld"], F + 2, 1)
        else:
            hb = self._planes("enc_hb", (B, F + 1, hop), pd)
            ops.wav_to_hopblocks(wav, hop, hb)
            spec_ = self._buf("enc_spec", (M, g["spec_ld"]))
            ops.gemm(hb, W["dft_fwd"], 2 * nf, a_batch=B, a_rows_per_batch=F + 1, a_ld=hop, m_per_batch=F, taps=2,
                     out_f32=rowmap(spec_, g["spec_ld"], F, 0))
            ops.stft_post(spec_, g["spec_ld"], B, F, nf, feat, g["feat_ld"], F + 2, 1)
        if taps is not None:
            taps["enc.feat"] = feat.float()[:, 1:-1, :2 * nf].transpose(1, 2).clone()
        x0 = self._buf("enc_x0", (M, C))
        ops.gemm(feat, E["embed"], C, a_batch=B, a_rows_per_batch=F + 2, a_ld=g["feat_ld"], m_per_batch=F, taps=3,
                 bias=E["embed_b"], out_f32=rowmap(x0, C, F, 0))
        x = self._buf("enc_x", (M, C))
        ops.layernorm(x0, E["norm_w"], E["norm_b"], B, F, C, out_f32=x)
        if taps is not None:
            taps["enc.embed_norm"] = x.reshape(B, F, C).transpose(1, 2).clone()
        self._convnext(E["convnext"], x, B, F, C, I)
        if taps is not None:
            taps["enc.prior"] = x.reshape(B, F, C).transpose(1, 2).clone()
        self._transformer(E["tf"], x, B, F, C)
        if taps is not None:
            taps["enc.post"] = x.reshape(B, F, C).transpose(1, 2).clone()
        k = 2 * stride + 1
        pad = k // 2
        rpb = _pad_to(F + 2 * pad, stride)
        fin = self._planes("enc_fin", (B, rpb, C), pc)
        ops.layernorm(x, E["fnorm_w"], E["fnorm_b"], B, F, C, out=fin, ld=C, rows_per_batch=rpb, row_off=pad)
        emb = self._buf("enc_emb", (B * N, Dq))
        ops.gemm(fin, E["out"], Dq, a_batch=B, a_rows_per_batch=rpb, a_ld=C, m_per_batch=N, taps=k, stride=stride,
                 bias=E["out_b"], out_f32=rowmap(emb, Dq, N, 0))
        if taps is not None:
            taps["enc.out"] = emb.reshape(B, N, Dq).transpose(1, 2).clone()
        return emb, N

    def _encode_sem(self, feat: torch.Tensor, taps=None):
        """vq/semantic_module.py:196-201 -> [B*N, out_channels] fp32."""
        W = self._prepare()
        S, cfg = W["sem"], self.sem_cfg
        B, Cin, F = feat.shape
        Cs, Co = cfg["encode_channels"], cfg["out_channels"]
        pc = self.policy["conv"]
        cin_pad = _pad_to(Cin, 64)
        fin = self._planes("sem_in", (B, F + 2, cin_pad), pc)
        ops.bct_to_planes(feat.float().contiguous(), fin, cin_pad, F + 2, 1)
        Tc = F
        sx = self._buf(f"sem_x{Tc}", (B * Tc, Cs))
        pe = self._planes(f"sem_pe{Tc}", (B, Tc + 2, Cs), pc)
        ops.gemm(fin, S["conv"], Cs, a_batch=B, a_rows_per_batch=F + 2, a_ld=cin_pad, m_per_batch=F, taps=3,
                 out_f32=rowmap(sx, Cs, Tc, 0), out_planes=pe, out_planes_map=(Cs, Tc + 2, 1), act2=ACT_ELU)
        nb = len(S["blocks"])
        for bi, blk in enumerate(S["blocks"]):
            pu = self._planes(f"sem_pu{Tc}", (B, Tc, Cs), pc)
            for u, un in enumerate(blk["units"]):
                ops.gemm(pe, un["c1"], Cs, a_batch=B, a_rows_per_batch=Tc + 2, a_ld=Cs, m_per_batch=Tc, taps=3,
                         act=ACT_ELU, out_planes=pu, out_planes_map=(Cs, Tc, 0))
                ops.gemm(pu, un["c2"], Cs, a_batch=B, a_rows_per_batch=Tc, a_ld=Cs, m_per_batch=Tc,
                         residual=rowmap(sx, Cs, Tc, 0), out_f32=rowmap(sx, Cs, Tc, 0), out_planes=pe,
                         out_planes_map=(Cs, Tc + 2, 1), act2=ACT_ELU if u == 0 else ACT_NONE)
            st, k = blk["stride"], blk["k"]
            pad = (k - 1) // 2
            if pad != 1 or (Tc + 2) % st != 0:
                raise ValueError(f"semantic encoder: {Tc} frames cannot be strided by {st} with kernel {k} (frame count must be even)")
            Tn = (Tc + 2 * pad - k) // st + 1
            sx2 = self._buf(f"sem_x{Tn}_{bi}", (B * Tn, Cs))
            pe2 = self._planes(f"sem_pe{Tn}_{bi}", (B, Tn + 2, Cs), pc)
            ops.gemm(pe, blk["conv"], Cs, a_batch=B, a_rows_per_batch=Tc + 2, a_ld=Cs, m_per_batch=Tn, taps=k, stride=st,
                     bias=blk["conv_b"], out_f32=rowmap(sx2, Cs, Tn, 0), out_planes=pe2, out_planes_map=(Cs, Tn + 2, 1),
                     act2=ACT_ELU if bi + 1 < nb else ACT_NONE)
            sx, pe, Tc = sx2, pe2, Tn
            if taps is not None:
                taps[f"sem.block{bi}"] = sx.reshape(B, Tc, Cs).transpose(1, 2).clone()
        out = self._buf("sem_out", (B * Tc, Co))
        ops.gemm(pe, S["conv2"], Co, a_batch=B, a_rows_per_batch=Tc + 2, a_ld=Cs, m_per_batch=Tc, taps=3,
                 out_f32=rowmap(out, Co, Tc, 0))
        if taps is not None:
            taps["sem.out"] = out.reshape(B, Tc, Co).transpose(1, 2).clone()
        return out, Tc

    # ------------------------------------------------------------------ decoder
    def _resnet(self, R, x, B, F, C):
        """vq/conv.py:286-303."""
        M = B * F
        pc = self.policy["conv"]
        stats = self._buf("gn_stats", (B, 32, 2))
        pr = self._planes("res_pr", (B, F + 2, C), pc)
        h = self._buf("res_h", (M, C))
        ops.groupnorm_stats(x, B, F, C, stats)
        ops.groupnorm_apply(x, stats, R["n1w"], R["n1b"], B, F, C, True, out=pr, ld=C, rows_per_batch=F + 2, row_off=1)
        ops.gemm(pr, R["c1"], C, a_batch=B, a_rows_per_batch=F + 2, a_ld=C, m_per_batch=F, taps=3, bias=R["c1b"],
                 out_f32=rowmap(h, C, F, 0))
        ops.groupnorm_stats(h, B, F, C, stats)
        ops.groupnorm_apply(h, stats, R["n2w"], R["n2b"], B, F, C, True, out=pr, ld=C, rows_per_batch=F + 2, row_off=1)
        ops.gemm(pr, R["c2"], C, a_batch=B, a_rows_per_batch=F + 2, a_ld=C, m_per_batch=F, taps=3, bias=R["c2b"],
                 residual=rowmap(x, C, F, 0), out_f32=rowmap(x, C, F, 0))

    def _decode_z(self, z: torch.Tensor, B: int, N: int, taps=None):
        """vq/codec_decoder.py:62-72.  z [B*N, input_channels] fp32 channel-last -> wav [B, N*factor*hop]."""
        W = self._prepare()
        g, D = W["geom"], W["dec"]
        d = self.dec_cfg
        Cin, C, I = d["input_channels"], d["dim"], d["intermediate_dim"]
        f = D["factor"]
        F = N * f
        M = B * F
        hop, nf, n_fft = g["hop"], g["nf"], g["n_fft"]
        pc, ph, pd = self.policy["conv"], self.policy["head"], self.policy["dft"]
        k = f + 1
        pad = k // 2
        zin = self._planes("dec_zin", (B, F + 2 * pad, Cin), pc)
        ops.rows_to_planes(z, B, N, Cin, zin, Cin, F + 2 * pad, pad, repeat=f)
        x = self._buf("dec_x", (M, C))
        ops.gemm(zin, D["embed"], C, a_batch=B, a_rows_per_batch=F + 2 * pad, a_ld=Cin, m_per_batch=F, taps=k,
                 bias=D["embed_b"], out_f32=rowmap(x, C, F, 0))
        if taps is not None:
            taps["dec.embed"] = x.reshape(B, F, C).transpose(1, 2).clone()
        self._resnet(D["res"][0], x, B, F, C)
        if taps is not None:
            taps["dec.res0"] = x.reshape(B, F, C).transpose(1, 2).clone()
        self._resnet(D["res"][1], x, B, F, C)
        self._transformer(D["tf"], x, B, F, C, mlp_group="mlp_dec")
        if taps is not None:
            taps["dec.tf"] = x.reshape(B, F, C).transpose(1, 2).clone()
        self._resnet(D["res"][5], x, B, F, C)
        self._resnet(D["res"][6], x, B, F, C)
        stats = self._buf("gn_stats", (B, 32, 2))
        h = self._buf("res_h", (M, C))
        ops.groupnorm_stats(x, B, F, C, stats)
        ops.groupnorm_apply(x, stats, D["gn_w"], D["gn_b"], B, F, C, False, out_f32=h)
        if taps is not None:
            taps["dec.prior"] = h.reshape(B, F, C).transpose(1, 2).clone()
        ops.layernorm(h, D["norm_w"], D["norm_b"], B, F, C, out_f32=x)
        self._convnext(D["convnext"], x, B, F, C, I)
        if taps is not None:
            taps["dec.post"] = x.reshape(B, F, C).transpose(1, 2).clone()
        t1 = self._planes("dec_fn", (M, C), ph)
        ops.layernorm(x, D["fnorm_w"], D["fnorm_b"], B, F, C, out=t1)
        if taps is not None:
            taps["dec.final_norm"] = t1.float().reshape(B, F, C).clone()
        head = self._buf("dec_head", (M, g["spec_ld"]))
        self._linear(t1, D["head"], 2 * nf, M, C, bias=D["head_b"], out_f32=rowmap(head, g["spec_ld"], M, 0))
        sp = self._planes("dec_sp", (M, g["kin"]), pd)
        ops.istft_pre(head, g["spec_ld"], M, nf, sp, g["kin"])
        frames = self._buf("dec_frames", (M, n_fft))
        self._linear(sp, W["dft_inv"], n_fft, M, g["kin"], out_f32=rowmap(frames, n_fft, M, 0))
        wav = torch.empty(B, F * hop, device=z.device)
        ops.istft_ola(frames, W["istft_window"], B, F, n_fft, wav, hop)
        return wav

    # ------------------------------------------------------------------ public surface
    @torch.no_grad()
    def encode(self, x, feat, taps=None):
        """vq/codec.py:75-87: x [B,T] fp32, feat [B,768,T/960] fp32 -> (acoustic, semantic) int64 [B,nq,N]."""
        if self._use_engine():
            eng = self.engine()
            if taps is None:
                return eng.encode(x, feat)
            eng.set_taps(taps)
            try:
                return eng.encode(x, feat)
            finally:
                eng.set_taps(None)
        emb, N = self._encode_emb(x, taps)
        sem, Ns = self._encode_sem(feat, taps)
        if Ns != N:
            raise ValueError(f"semantic stream has {Ns} frames but the acoustic stream has {N}")
        B = x.shape[0]
        ia, _ = self.quantizer.encode_rows(emb, want_quantized=False)
        isem, _ = self.semantic_quantizer.encode_rows(sem, want_quantized=False)
        return (ia.reshape(B, N, -1).transpose(1, 2).contiguous(), isem.reshape(B, N, -1).transpose(1, 2).contiguous())

    @torch.no_grad()
    def decode(self, acoustic_codes, semantic_codes, taps=None):
        """vq/codec.py:89-99: int64 [B,nq,N] x2 -> wav [B, N*3840]."""
        if self._use_engine():
            eng = self.engine()
            if taps is None:
                return eng.decode(acoustic_codes, semantic_codes)
            eng.set_taps(taps)
            try:
                return eng.decode(acoustic_codes, semantic_codes)
            finally:
                eng.set_taps(None)
        B, nq, N = acoustic_codes.shape
        Dq = self.quantizer.dim
        z = self._buf("dec_z", (B * N, 2 * Dq))
        ia = acoustic_codes.transpose(1, 2).reshape(B * N, nq).long().contiguous()
        isem = semantic_codes.transpose(1, 2).reshape(B * N, nq).long().contiguous()
        self.quantizer.decode_rows(ia, z, 2 * Dq, 0)
        self.semantic_quantizer.decode_rows(isem, z, 2 * Dq, Dq)
        return self._decode_z(z, B, N, taps)

    # ------------------------------------------------------------------ CUDA-graph replay of a fixed-shape call
    def graphed(self, fn_name: str, *example_inputs, warmup: int = 2) -> "GraphedCall":
        """Capture `encode`, `decode` or `roundtrip` (encode -> decode) for the shapes of `example_inputs` into ONE CUDA
        graph: a step is ~340 kernel launches, a third of them a few microseconds long (RVQ layers, norms, small GEMMs) -
        replaying the graph removes the host launch gaps.  Returns a callable taking tensors of the same shapes (device or
        pinned host; they are copied into the graph's static inputs) and returning the static output tensors."""
        fn = dict(encode=self.encode, decode=self.decode, roundtrip=self.roundtrip)[fn_name]
        return GraphedCall(fn, example_inputs, warmup)

    @torch.no_grad()
    def roundtrip(self, x, feat):
        """encode -> decode: (acoustic, semantic, reconstructed wav)."""
        ac, sc = self.encode(x, feat)
        return ac, sc, self.decode(ac, sc)

    def forward(self, x, feat):
        raise RuntimeError("unified_audio_b200.Codec implements the inference path only (encode / decode); "
                           "training forward (codec.py:51-72) is out of scope")


class GraphedCall:
    """A fixed-shape call captured in a CUDA graph (static input / output buffers, `torch.cuda.graphs`)."""

    def __init__(self, fn, example_inputs, warmup: int = 2):
        self.inputs = [t.detach().to("cuda", copy=True) for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):              # warm-up off the capture: lazy weight preparation, workspaces, attributes
            for _ in range(max(warmup, 1)):
                fn(*self.inputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        n0 = ops.launch_count()
        with torch.cuda.graph(self.graph):
            self.outputs = fn(*self.inputs)
        self.launches_per_replay = ops.launch_count() - n0      # library kernels recorded in the graph

    def __call__(self, *inputs):
        if inputs:
            if len(inputs) != len(self.inputs):
                raise ValueError("graphed call: wrong number of inputs")
            for dst, src in zip(self.inputs, inputs):
                if src.shape != dst.shape or src.dtype != dst.dtype:
                    raise ValueError(f"graphed call captured for {tuple(dst.shape)} {dst.dtype}, got {tuple(src.shape)} {src.dtype}")
                if src.data_ptr() != dst.data_ptr():
                    dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.outputs

    # ------------------------------------------------------------------ streaming host I/O
    def stream(self, host_inputs, host_outputs):
        """One step of a serving loop with HOST tensors on both sides, copies overlapped with compute: the H2D copy of this step's
        (pinned) inputs runs on a copy stream into a staging buffer while the previous step still computes; the step itself is a
        device-to-device move into the graph's static inputs + the replay + a device-to-device move of its outputs into a second
        staging buffer, from which the copy stream drains them into `host_outputs` (pinned) under the next step.  Call
        `finish()` (or torch.cuda.synchronize()) before reading `host_outputs` of the last step."""
        cur = torch.cuda.current_stream()
        if getattr(self, "_io", None) is None:
            outs = self.outputs if isinstance(self.outputs, (tuple, list)) else (self.outputs,)
            # two copy streams: on one, the H2D of step i + 1 would queue behind the D2H of step i, which waits for step i's compute
            self._io = dict(stream=torch.cuda.Stream(), d2h_stream=torch.cuda.Stream(), in_stage=[torch.empty_like(t) for t in self.inputs],
                            out_stage=[torch.empty_like(t) for t in outs], h2d=torch.cuda.Event(), staged=torch.cuda.Event(),
                            consumed=torch.cuda.Event(), drained=torch.cuda.Event())
            self._io["consumed"].record(cur)
            self._io["drained"].record(cur)
        io = self._io
        with torch.cuda.stream(io["stream"]):
            io["stream"].wait_event(io["consumed"])            # the previous step has moved its inputs out of the staging buffer
            for dst, src in zip(io["in_stage"], host_inputs):
                dst.copy_(src, non_blocking=True)
            io["h2d"].record(io["stream"])
        cur.wait_event(io["h2d"])
        for dst, src in zip(self.inputs, io["in_stage"]):
            dst.copy_(src, non_blocking=True)
        io["consumed"].record(cur)
        self.graph.replay()
        outs = self.outputs if isinstance(self.outputs, (tuple, list)) else (self.outputs,)
        cur.wait_event(io["drained"])                           # the previous step's outputs have left the staging buffer
        for dst, src in zip(io["out_stage"], outs):
            dst.copy_(src, non_blocking=True)
        io["staged"].record(cur)
        with torch.cuda.stream(io["d2h_stream"]):
            io["d2h_stream"].wait_event(io["staged"])
            for dst, src in zip(host_outputs, io["out_stage"]):
                dst.copy_(src, non_blocking=True)
            io["drained"].record(io["d2h_stream"])

    def finish(self):
        if getattr(self, "_io", None) is not None:
            torch.cuda.current_stream().wait_event(self._io["drained"])


def stft2_factors(n_fft: int):
    """n_fft = P * Q with P <= 64 and Q <= 64 (P as large as possible): 1920 -> (48, 40), 1280 -> (40, 32); None if impossible"""
    for P in range(64, 0, -1):
        if n_fft % P == 0 and n_fft // P <= 64:
            return P, n_fft // P
    return None


def _stft2_weights(n_fft: int, window: torch.Tensor, dev):
    """DFT matrices of the two-stage STFT in fp64 (exact argument reduction): W_A [2P, 64], W_B [2*K2, 128], twiddle [Q*P, 2]"""
    pq = stft2_factors(n_fft)
    if pq is None:
        return None
    P, Q = pq
    nf = n_fft // 2 + 1
    K2 = (nf - 1) // P + 1
    two_pi = 2.0 * math.pi
    k1 = torch.arange(P, dtype=torch.int64)
    a = torch.arange(P, dtype=torch.int64)
    angA = two_pi * (torch.outer(k1, a) % P).double() / P
    wA = torch.zeros(2 * P, 64, dtype=torch.float64)
    wA[0::2, :P] = torch.cos(angA)
    wA[1::2, :P] = -torch.sin(angA)
    k2 = torch.arange(K2, dtype=torch.int64)
    b = torch.arange(Q, dtype=torch.int64)
    angB = two_pi * (torch.outer(k2, b) % Q).double() / Q
    wB = torch.zeros(2 * K2, 128, dtype=torch.float64)
    wB[0::2, :Q] = torch.cos(angB)
    wB[0::2, Q:2 * Q] = torch.sin(angB)
    wB[1::2, :Q] = -torch.sin(angB)
    wB[1::2, Q:2 * Q] = torch.cos(angB)
    angT = two_pi * (torch.outer(b, k1) % n_fft).double() / n_fft          # [b, k1]
    tw = torch.stack([torch.cos(angT), -torch.sin(angT)], -1).float().reshape(Q * P, 2).contiguous()
    return dict(P=P, Q=Q, wA=_planes_from_f64(wA.to(dev), True), wB=_planes_from_f64(wB.to(dev), True), tw=tw.to(dev), nB=2 * K2,
                ldX=_pad_to(2 * K2, 4), window=window)


def _planes_from_f64(w: torch.Tensor, split: bool) -> Planes:
    hi = w.clamp(-65504.0, 65504.0).half()
    lo = (w - hi.double()).half() if split else None
    return Planes(hi.contiguous(), lo.contiguous() if lo is not None else None)
