"""H-Codec-1.0 `Codec` (BASELINE.json configs[0]) with the reference's surface, running on libquark_b200.

Mirrors QuarkAudio-HCodec/HCodec-1.0/vq/codec.py:21-188: `Codec(encoder_kwargs, decoder_kwargs, quantizer_kwargs)`
(all three ignored - the reference hard-codes its hyper-parameters at codec.py:30-136),
`.encode(x [B,1,T] @16 kHz, feat [B,768,T/320]) -> (int64 [B,4,N], int64 [B,4,N])`, `.decode(...) -> f32 [B, N*640]`.
state_dict keys are the reference's, including the old-style weight-norm pairs `...conv.conv.weight_g / weight_v`
(HCodec-1.0/vq/encoder_modules/conv.py:25-28), folded into plain weights at load.

SEANet encoder = strided / reflect-padded conv stack (encoder_modules/seanet.py:121-208): every conv runs as a
TMA-im2col GEMM over a reflect-filled channel-last plane buffer; decoder = sub-pixel x2 up-sampler (vq/conv.py:60-93)
+ the H-Codec-2.0 block set at width 768 (8 heads of 96) + ISTFT(1280, hop 320).

This face is orchestrated from Python: `encode` / `decode` launch the libquark_b200 kernels op by op on the current CUDA
stream, from weights repacked here at first use.  `CodecH15` (codec_h15.py) builds on it.  The H-Codec-2.0 `Codec`
(codec.py) is backed by the C engine instead.  There is no PyTorch / CPU fallback.
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from . import ops
from .codec import _CodecFace, _Tree, _pad_to, PRECISION_POLICIES
from .ops import ACT_ELU, ACT_GELU, ACT_NONE, ACT_SWIGLU, Planes, rowmap
from .rvq import ResidualVQ

RATIOS = [2, 4, 5, 8]          # SEANetEncoder reverses ratios=[8,5,4,2] (seanet.py:111)
H1 = dict(n_filters=32, dimension=512, dec_dim=768, dec_inter=2304, dec_layers=12, n_fft=1280, hop=320, nq=4,
          codebook_size=1024, sem_in=768, sem_ch=768, sem_strides=[2, 1], tf_layers=2, heads=8)


def _tf_spec(out, prefix, dim, inter, layers):
    for i in range(layers):
        p = f"{prefix}layers.{i}."
        for n in ("weight_ih_l0", "weight_hh_l0"):
            out[p + "self_attn.rnn." + n] = (4 * dim, dim)
        for n in ("bias_ih_l0", "bias_hh_l0"):
            out[p + "self_attn.rnn." + n] = (4 * dim,)
        for n in "qkv":
            out[p + f"self_attn.{n}_proj.weight"] = (dim, dim)
            out[p + f"self_attn.{n}_proj.bias"] = (dim,)
        out[p + "self_attn.o_proj.weight"] = (dim, dim)
        out[p + "mlp.w1.weight"] = (inter, dim)
        out[p + "mlp.w2.weight"] = (dim, inter)
        out[p + "mlp.w3.weight"] = (inter, dim)
        out[p + "input_layernorm.weight"] = (dim,)
        out[p + "post_attention_layernorm.weight"] = (dim,)


def h1_spec(c) -> Dict[str, Dict[str, tuple]]:
    enc, dec, sem = {}, {}, {}

    def wn(p, cout, cin, k):
        enc[p + "conv.conv.bias"] = (cout,)
        enc[p + "conv.conv.weight_g"] = (cout, 1, 1)
        enc[p + "conv.conv.weight_v"] = (cout, cin, k)

    nf, dim = c["n_filters"], c["dimension"]
    wn("model.0.", nf, 1, 7)
    mult, idx = 1, 1
    for r in c.get("ratios", RATIOS):
        ch = mult * nf
        wn(f"model.{idx}.block.1.", ch // 2, ch, 3)
        wn(f"model.{idx}.block.3.", ch, ch // 2, 1)
        wn(f"model.{idx}.shortcut.", ch, ch, 1)
        wn(f"model.{idx + 2}.", ch * 2, ch, 2 * r)
        mult *= 2
        idx += 3
    _tf_spec(enc, f"model.{idx + 1}.", dim, dim * 4, c["tf_layers"])
    wn(f"model.{idx + 4}.", dim, dim, 4)
    dd, di = c["dec_dim"], c["dec_inter"]
    dec["embed.up.weight"] = (dd * 2, 2 * dim, 1)
    dec["embed.up.bias"] = (dd * 2,)
    dec["embed.dw.weight"] = (dd, 1, 5)
    dec["embed.dw.bias"] = (dd,)
    dec["norm.weight"] = (dd,)
    dec["norm.bias"] = (dd,)
    for i in range(c["dec_layers"]):
        p = f"post_net.{i}."
        dec[p + "gamma"] = (dd,)
        dec[p + "dwconv.conv.weight"] = (dd, 1, 7)
        dec[p + "dwconv.conv.bias"] = (dd,)
        dec[p + "norm.weight"] = (dd,)
        dec[p + "norm.bias"] = (dd,)
        dec[p + "pwconv1.linear.weight"] = (di, dd)
        dec[p + "pwconv1.linear.bias"] = (di,)
        dec[p + "pwconv2.linear.weight"] = (dd, di)
        dec[p + "pwconv2.linear.bias"] = (dd,)
    dec["final_layer_norm.weight"] = (dd,)
    dec["final_layer_norm.bias"] = (dd,)
    for i in (0, 1, 5, 6):
        p = f"prior_net.{i}."
        for j in (1, 2):
            dec[p + f"norm{j}.weight"] = (dd,)
            dec[p + f"norm{j}.bias"] = (dd,)
            dec[p + f"conv{j}.conv.weight"] = (dd, dd, 3)
            dec[p + f"conv{j}.conv.bias"] = (dd,)
    _tf_spec(dec, "prior_net.3.", dd, dd * 4, c["tf_layers"])
    dec["prior_net.7.weight"] = (dd,)
    dec["prior_net.7.bias"] = (dd,)
    dec["head.out.weight"] = (c["n_fft"] + 2, dd)
    dec["head.out.bias"] = (c["n_fft"] + 2,)
    dec["head.istft.window"] = (c["n_fft"],)
    sc = c["sem_ch"]
    sem["conv.conv.weight"] = (sc, c["sem_in"], 3)
    for i, st in enumerate(c["sem_strides"]):
        p = f"conv_blocks.{i}."
        for u in (0, 1):
            sem[p + f"res_units.{u}.conv1.conv.weight"] = (sc, sc, 3)
            sem[p + f"res_units.{u}.conv2.weight"] = (sc, sc, 1)
        k = 3 if st == 1 else 2 * st
        sem[p + "conv.conv.weight"] = (sc, sc, k)
        sem[p + "conv.conv.bias"] = (sc,)
    sem["conv2.conv.weight"] = (dim, sc, 3)
    return dict(encoder=enc, decoder=dec, semantic_encoder=sem)


def semantic_decoder_config(c) -> dict:
    """Decoder kwargs of the semantic decoder: the config's own `sem_dec` (H-Codec-1.5's decoder_kwargs["semantic_decoder"]), else
    the sizes H-Codec-1.0 hard-codes (vq/codec.py:130-136: code_dim -> semantic encoder width -> SSL width, its strides)."""
    if c.get("sem_dec") is not None:
        return dict(c["sem_dec"])
    return dict(code_dim=c["dimension"], output_channels=c["sem_in"], decode_channels=c["sem_ch"],
                channel_ratios=[1] * len(c["sem_strides"]), strides=list(c["sem_strides"]))


class CodecH1(_CodecFace):
    def __init__(self, encoder_kwargs: dict = None, decoder_kwargs: dict = None, quantizer_kwargs: dict = None,
                 precision: str = "mixed", _cfg: dict = None, semantic_decoder: bool = False):
        super().__init__()
        c = dict(_cfg or H1)
        self.c = c
        sp = h1_spec(c)
        self.encoder = _Tree.build(sp["encoder"])
        self.decoder = _Tree.build(sp["decoder"])
        q = dict(dim=c["dimension"], codebook_size=c["codebook_size"], num_quantizers=c["nq"])
        self.quantizer = ResidualVQ(**q)
        self.semantic_quantizer = ResidualVQ(**q)
        self.semantic_encoder = _Tree.build(sp["semantic_encoder"])
        self._add_semantic_decoder(semantic_decoder, semantic_decoder_config(c))
        self.sem_cfg = dict(encode_channels=c["sem_ch"], out_channels=c["dimension"], strides=c["sem_strides"],
                            channel_ratios=[1] * len(c["sem_strides"]))
        self.dec_cfg = dict(dim=c["dec_dim"], intermediate_dim=c["dec_inter"])
        self.policy = dict(PRECISION_POLICIES[precision])
        self.precision = precision
        self.eval()

    # ------------------------------------------------------------------ weight repack
    def _prepare(self):
        if self._w is not None:
            return self._w
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        dev = self._require_cuda()
        pol, c = self.policy, self.c
        W: Dict[str, object] = {}

        def pack(w, group):
            return ops.conv_planes(w.float(), pol[group])

        def wn(p):     # fold old-style weight norm: w = g * v / ||v||  (encoder_modules/conv.py:25-28)
            v = sd[p + "conv.conv.weight_v"].double()
            w = sd[p + "conv.conv.weight_g"].double() * v / v.flatten(1).norm(dim=1)[:, None, None]
            return dict(w=pack(w.float(), "conv"), b=sd[p + "conv.conv.bias"].float().contiguous(), k=v.shape[-1],
                        cout=v.shape[0], cin=v.shape[1])

        f32 = lambda k: sd[k].float().contiguous()
        stages = []
        idx = 1
        for r in c.get("ratios", RATIOS):
            stages.append(dict(b1=wn(f"encoder.model.{idx}.block.1."), b3=wn(f"encoder.model.{idx}.block.3."),
                               sc=wn(f"encoder.model.{idx}.shortcut."), down=wn(f"encoder.model.{idx + 2}."), r=r))
            idx += 3
        W["enc"] = dict(conv0=wn("encoder.model.0."), stages=stages,
                        tf=self._pack_tf(sd, f"encoder.model.{idx + 1}.", c["tf_layers"]),
                        final=wn(f"encoder.model.{idx + 4}."))
        blocks = []
        for i, st in enumerate(c["sem_strides"]):
            p = f"semantic_encoder.conv_blocks.{i}."
            blocks.append(dict(units=[dict(c1=pack(sd[p + f"res_units.{u}.conv1.conv.weight"], "conv"),
                                           c2=pack(sd[p + f"res_units.{u}.conv2.weight"], "conv")) for u in (0, 1)],
                               conv=pack(sd[p + "conv.conv.weight"], "conv"), conv_b=f32(p + "conv.conv.bias"), stride=st,
                               k=3 if st == 1 else 2 * st))
        W["sem"] = dict(conv=pack(sd["semantic_encoder.conv.conv.weight"], "conv"), blocks=blocks,
                        conv2=pack(sd["semantic_encoder.conv2.conv.weight"], "conv"))
        res = {}
        for i in (0, 1, 5, 6):
            p = f"decoder.prior_net.{i}."
            res[i] = dict(n1w=f32(p + "norm1.weight"), n1b=f32(p + "norm1.bias"), n2w=f32(p + "norm2.weight"),
                          n2b=f32(p + "norm2.bias"), c1=pack(sd[p + "conv1.conv.weight"], "conv"), c1b=f32(p + "conv1.conv.bias"),
                          c2=pack(sd[p + "conv2.conv.weight"], "conv"), c2b=f32(p + "conv2.conv.bias"))
        cn = []
        for i in range(c["dec_layers"]):
            p = f"decoder.post_net.{i}."
            cn.append(dict(dw_w=sd[p + "dwconv.conv.weight"].float().reshape(-1, 7).contiguous(), dw_b=f32(p + "dwconv.conv.bias"),
                           ln_w=f32(p + "norm.weight"), ln_b=f32(p + "norm.bias"),
                           w1=Planes.from_f32(sd[p + "pwconv1.linear.weight"].float().contiguous(), pol["convnext"]),
                           b1=f32(p + "pwconv1.linear.bias"),
                           w2=Planes.from_f32(sd[p + "pwconv2.linear.weight"].float().contiguous(), pol["convnext"]),
                           b2=f32(p + "pwconv2.linear.bias"), gamma=f32(p + "gamma")))
        n_fft, hop = c["n_fft"], c["hop"]
        nf = n_fft // 2 + 1
        kin = _pad_to(2 * nf, 64)
        s = torch.arange(n_fft, dtype=torch.int64, device=dev)
        k = torch.arange(nf, dtype=torch.int64, device=dev)
        angT = (2.0 * math.pi * (torch.outer(k, s) % n_fft).double() / n_fft).t()
        ck = torch.full((nf,), 2.0, dtype=torch.float64, device=dev)
        ck[0] = 1.0
        ck[-1] = 1.0
        win = sd["decoder.head.istft.window"].double()
        inv = torch.zeros(n_fft, kin, dtype=torch.float64, device=dev)
        inv[:, :nf] = torch.cos(angT) * ck / n_fft * win[:, None]
        im = -torch.sin(angT) * ck / n_fft * win[:, None]
        im[:, 0] = 0.0
        im[:, -1] = 0.0
        inv[:, nf:2 * nf] = im
        W["dec"] = dict(up=pack(sd["decoder.embed.up.weight"], "conv"), up_b=f32("decoder.embed.up.bias"),
                        dw_w=sd["decoder.embed.dw.weight"].float().reshape(-1, 5).contiguous(), dw_b=f32("decoder.embed.dw.bias"),
                        res=res, tf=self._pack_tf(sd, "decoder.prior_net.3.", c["tf_layers"]),
                        gn_w=f32("decoder.prior_net.7.weight"), gn_b=f32("decoder.prior_net.7.bias"),
                        norm_w=f32("decoder.norm.weight"), norm_b=f32("decoder.norm.bias"), convnext=cn,
                        fnorm_w=f32("decoder.final_layer_norm.weight"), fnorm_b=f32("decoder.final_layer_norm.bias"),
                        head=Planes.from_f32(sd["decoder.head.out.weight"].float().contiguous(), pol["head"]),
                        head_b=f32("decoder.head.out.bias"), dft_inv=_planes_from_f64(inv, True),
                        window=sd["decoder.head.istft.window"].float().contiguous(), nf=nf, kin=kin, spec_ld=_pad_to(2 * nf, 4))
        if self.sem_dec_cfg is not None:
            W["sem_dec"] = self._pack_semantic_decoder(sd)
        self._w = W
        return W

    def _pack_semantic_decoder(self, sd):
        """semantic_decoder.* -> GEMM weights at the semantic encoder's precision: k3 convs as tap-major planes, each
        ConvTranspose1d(2s, s) as the phase weight of ops.convt_planes with its bias repeated per phase."""
        split, p = self.policy["conv"], "semantic_decoder."
        blocks = []
        for i, st in enumerate(self.sem_dec_cfg["strides"]):
            b = f"{p}conv_blocks.{i}."
            units = [dict(c1=ops.conv_planes(sd[b + f"res_units.{u}.conv1.conv.weight"].float(), split),
                          c2=ops.conv_planes(sd[b + f"res_units.{u}.conv2.weight"].float(), split)) for u in (0, 1)]
            if st == 1:
                w = sd[b + "conv.conv.weight"].float()
                blocks.append(dict(stride=1, w=ops.conv_planes(w, split), b=sd[b + "conv.conv.bias"].float().contiguous(),
                                   cin=w.shape[1], cout=w.shape[0], units=units))
            else:
                w = sd[b + "conv.deconv.weight"].float()
                wt, J = ops.convt_planes(w, st, split)
                blocks.append(dict(stride=st, w=wt, J=J, b=sd[b + "conv.deconv.bias"].float().repeat(st).contiguous(),
                                   cin=w.shape[0], cout=w.shape[1], units=units))
        w1, w2 = sd[p + "conv1.conv.weight"].float(), sd[p + "conv2.conv.weight"].float()
        return dict(conv1=ops.conv_planes(w1, split), code_dim=w1.shape[1], c0=w1.shape[0], blocks=blocks,
                    conv2=ops.conv_planes(w2, split), cout=w2.shape[0])

    def _semantic_decode_rows(self, z, B, N):
        """vq/semantic_module.py:294-299 (Decoder), :245-249 (DecoderBlock), :78-81 (ResidualUnit) on quantised rows
        z [B*N, code_dim] fp32 -> pred_feat fp32 [B, C_ssl, T].  Channel-last planes end to end: every conv input sits in a
        buffer zero-padded by one frame on each side, the fp32 trunk of a block is updated in place by the 1x1 convs' residual
        epilogues, and each epilogue writes the planes (ELU'd where the next conv wants it) its consumer reads."""
        D = self._prepare()["sem_dec"]
        split = self.policy["conv"]
        cd = _pad_to(D["code_dim"], 64)
        zp = self._planes(f"sd_z{N}", (B, N + 2, cd), split)
        ops.rows_to_planes(z, B, N, D["code_dim"], zp, cd, N + 2, 1)
        cp = _pad_to(D["c0"], 64)
        xin = self._planes("sd_in0", (B, N + 2, cp), split)
        ops.gemm(zp, D["conv1"], D["c0"], a_batch=B, a_rows_per_batch=N + 2, a_ld=cd, m_per_batch=N, taps=3, out_planes=xin,
                 out_planes_map=(cp, N + 2, 1))
        T = N
        for bi, blk in enumerate(D["blocks"]):
            st, co = blk["stride"], blk["cout"]
            cpi, cpo = cp, _pad_to(co, 64)
            pe = None
            if st == 1:
                Tn = T
                trunk = self._buf(f"sd_x{bi}", (B * T, co))
                tr = rowmap(trunk, co, T, 0)
                pe = self._planes(f"sd_pe{bi}", (B, T + 2, cpo), split)
                ops.gemm(xin, blk["w"], co, a_batch=B, a_rows_per_batch=T + 2, a_ld=cpi, m_per_batch=T, taps=3, bias=blk["b"],
                         out_f32=tr, out_planes=pe, out_planes_map=(cpo, T + 2, 1), act2=ACT_ELU)
            else:
                # ConvTranspose1d(2s, s, padding (s+1)//2, output_padding s%2) as a J-tap GEMM (the input buffer's one-frame pads are
                # the J - 1 = 1 zero rows it needs): row q holds the s phases of uncropped frames q*s.., and the output clip is
                # frames [pad, pad + T*s) of those rows read as [(T + 1) * s, co]
                J, pad, Tn = blk["J"], (st + 1) // 2, T * st
                if J != 2:
                    raise ValueError(f"semantic decoder block {bi}: a {J}-tap transposed conv is not built (kernel 2 * stride has 2)")
                up = self._buf(f"sd_up{bi}", (B, T + 1, st * co))
                ops.gemm(xin, blk["w"], st * co, a_batch=B, a_rows_per_batch=T + 2, a_ld=cpi, m_per_batch=T + 1, taps=J,
                         bias=blk["b"], out_f32=rowmap(up, st * co, T + 1, 0))
                tr = rowmap(up, co, (T + 1) * st, pad)
                pe = self._planes(f"sd_pe{bi}", (B, Tn + 2, cpo), split)
                ops.elu_planes(up.view(-1)[pad * co:], (T + 1) * st * co, B, Tn, co, pe, cpo, Tn + 2, 1)
            T = Tn
            pu = self._planes(f"sd_pu{bi}", (B * T, cpo), split)
            nxt = self._planes(f"sd_in{bi + 1}", (B, T + 2, cpo), split)
            for u, un in enumerate(blk["units"]):
                ops.gemm(pe, un["c1"], co, a_batch=B, a_rows_per_batch=T + 2, a_ld=cpo, m_per_batch=T, taps=3, act=ACT_ELU,
                         out_planes=pu, out_planes_map=(cpo, T, 0))
                last = u == len(blk["units"]) - 1
                ops.gemm(pu, un["c2"], co, a_batch=B, a_rows_per_batch=T, a_ld=cpo, m_per_batch=T, residual=tr,
                         out_f32=None if last else tr, out_planes=nxt if last else pe, out_planes_map=(cpo, T + 2, 1),
                         act2=ACT_NONE if last else ACT_ELU)
            xin, cp = nxt, cpo
        Co = D["cout"]
        rows = self._buf("sd_out", (B * T, Co))
        ops.gemm(xin, D["conv2"], Co, a_batch=B, a_rows_per_batch=T + 2, a_ld=cp, m_per_batch=T, taps=3,
                 out_f32=rowmap(rows, Co, T, 0))
        pred = torch.empty(B, Co, T, device=z.device)
        ops.ssl_compress(rows, B, T, Co, 0.0, True, pred)          # power 0: the plain [B, T, C] -> [B, C, T] copy
        return pred

    def _pack_tf(self, sd, prefix, n):
        pol = self.policy
        layers = []
        hdim = sd[f"{prefix}layers.0.self_attn.rnn.weight_hh_l0"].shape[1]
        lstm_u = ops.lstm_tc_units(hdim) if hdim % 256 == 0 else 0
        if not lstm_u:
            raise ValueError(f"{prefix}: LSTM width {hdim} unsupported by the wgmma recurrence "
                             f"(needs H % 256 == 0, and H / U CTAs of U = 4, 8 or 12 units fitting on the SMs)")
        for i in range(n):
            p = f"{prefix}layers.{i}."
            a = p + "self_attn."
            w13 = torch.stack([sd[p + "mlp.w1.weight"].float(), sd[p + "mlp.w3.weight"].float()], 1)
            lw = lambda w, g: Planes.from_f32(w.float().contiguous(), pol[g])
            layers.append(dict(
                in_w=sd[p + "input_layernorm.weight"].float().contiguous(), post_w=sd[p + "post_attention_layernorm.weight"].float().contiguous(),
                wih=lw(sd[a + "rnn.weight_ih_l0"], "lstm_attn"),
                b_ih=(sd[a + "rnn.bias_ih_l0"].float() + sd[a + "rnn.bias_hh_l0"].float()).contiguous(),
                whh_perm=ops.lstm_tc_permute(sd[a + "rnn.weight_hh_l0"], lstm_u), lstm_u=lstm_u,
                wqkv=lw(torch.cat([sd[a + f"{n_}_proj.weight"].float() for n_ in "qkv"], 0), "lstm_attn"),
                bqkv=torch.cat([sd[a + f"{n_}_proj.bias"].float() for n_ in "qkv"], 0).contiguous(),
                wo=lw(sd[a + "o_proj.weight"], "lstm_attn"), w13=lw(w13.reshape(-1, w13.shape[-1]), "mlp"),
                w2=lw(sd[p + "mlp.w2.weight"], "mlp")))
        return layers

    # ------------------------------------------------------------------ blocks
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

    def _transformer(self, layers, x, B, F, C, heads=None):
        """encoder_modules/transformer.py:367-393 per layer; x [B*F, C] fp32 updated in place."""
        heads = heads or C // 64
        hd = C // heads
        M, I = B * F, min(4 * C, 4096)
        pa, pm = self.policy["lstm_attn"], self.policy["mlp"]
        t_a = self._planes("tf_a", (M, C), pa)
        t_b = self._planes("tf_b", (M, C), pa)
        t_m = self._planes("tf_m", (M, C), pm)
        hid = self._planes("tf_hid", (M, I), pm)
        xp = self._buf("tf_xp", (M, 4 * C))
        qkv = self._buf("tf_qkv", (M, 3 * C))
        ws = self._buf("lstm_ws", (ops.lstm_tc_workspace_bytes(B, C),), torch.uint8)
        cos, sin = self._cached(("rope", F, hd), lambda: ops.rope_tables(F, hd, self._dev()))
        att_ws = self._buf("att5_ws", (ops.self_attention_workspace_bytes(B, F, heads, hd, pa),), torch.uint8)
        xm = rowmap(x, C, M, 0)
        for L in layers:
            ops.rmsnorm(x, L["in_w"], M, C, t_a)
            self._linear(t_a, L["wih"], 4 * C, M, C, bias=L["b_ih"], out_f32=rowmap(xp, 4 * C, M, 0))
            ops.lstm_tc(xp, L["whh_perm"], L["lstm_u"], B, F, C, t_b, ws)
            self._linear(t_b, L["wqkv"], 3 * C, M, C, bias=L["bqkv"], out_f32=rowmap(qkv, 3 * C, M, 0))
            ops.self_attention(qkv, B, F, heads, hd, cos, sin, t_a, att_ws, pa)
            self._linear(t_a, L["wo"], C, M, C, residual=xm, out_f32=xm)
            ops.rmsnorm(x, L["post_w"], M, C, t_m)
            self._linear(t_m, L["w13"], 2 * I, M, C, act=ACT_SWIGLU, out_planes=hid, out_planes_map=(I, M, 0))
            self._linear(hid, L["w2"], C, M, I, residual=xm, out_f32=xm)

    # ------------------------------------------------------------------ SEANet encoder
    def _sconv(self, src: Planes, cw, B, T_in, stride, *, src_rpb, bias=True, residual=None, out_f32=None, out=None,
               out_map=(0, 0, 0), act2=ACT_NONE):
        """strided conv over a (reflect-filled) plane buffer; T_out = T_in / stride."""
        k, cin_pad = cw["k"], _pad_to(cw["cin"], 64)
        T_out = T_in // stride
        ops.gemm(src, cw["w"], cw["cout"], a_batch=B, a_rows_per_batch=src_rpb, a_ld=cin_pad, m_per_batch=T_out, taps=k,
                 stride=stride, bias=cw["b"] if bias else None, residual=residual, out_f32=out_f32, out_planes=out,
                 out_planes_map=out_map, act2=act2)
        return T_out

    def _encode_emb(self, x: torch.Tensor, taps=None):
        """encoder_modules/seanet.py:121-208 as built at vq/codec.py:30-35.  x [B,1,T] -> emb [B*N, 512]."""
        W = self._prepare()
        E, c = W["enc"], self.c
        pc = self.policy["conv"]
        B, one, T = x.shape
        if one != 1:
            raise ValueError(f"expected a mono waveform [B, 1, T], got {tuple(x.shape)}")
        if T % 640 != 0:
            raise ValueError(f"waveform length {T} must be a multiple of 640 (hop 320 x final stride 2)")
        x = x.float().reshape(B, T, 1).contiguous()
        p0 = self._planes("h1_p0", (B, T + 6, 64), pc)
        ops.rows_to_planes(x, B, T, 1, p0, 64, T + 6, 3)
        ops.reflect_pad_rows(p0, B, T + 6, 64, T, 3, 3, 3)
        ch = c["n_filters"]
        cp = _pad_to(ch, 64)
        y = self._buf(f"h1_y{T}", (B * T, ch))
        pe = self._planes(f"h1_pe{T}", (B, T + 2, cp), pc)
        self._sconv(p0, E["conv0"], B, T, 1, src_rpb=T + 6, out_f32=rowmap(y, ch, T, 0), out=pe, out_map=(cp, T + 2, 1),
                    act2=ACT_ELU)
        ops.reflect_pad_rows(pe, B, T + 2, cp, T, 1, 1, 1)
        Tc = T
        for st in E["stages"]:
            r = st["r"]
            cp, ch2, cph = _pad_to(ch, 64), ch // 2, _pad_to(ch // 2, 64)
            px = self._planes(f"h1_px{Tc}", (B, Tc, cp), pc)
            ops.rows_to_planes(y, B, Tc, ch, px, cp, Tc, 0)
            pu = self._planes(f"h1_pu{Tc}", (B, Tc, cph), pc)
            self._sconv(pe, st["b1"], B, Tc, 1, src_rpb=Tc + 2, out=pu, out_map=(cph, Tc, 0), act2=ACT_ELU)
            s = self._buf(f"h1_s{Tc}", (B * Tc, ch))
            self._sconv(px, st["sc"], B, Tc, 1, src_rpb=Tc, out_f32=rowmap(s, ch, Tc, 0))
            left = r - r // 2
            pd = self._planes(f"h1_pd{Tc}", (B, Tc + r, cp), pc)
            self._sconv(pu, st["b3"], B, Tc, 1, src_rpb=Tc, residual=rowmap(s, ch, Tc, 0), out=pd, out_map=(cp, Tc + r, left),
                        act2=ACT_ELU)
            ops.reflect_pad_rows(pd, B, Tc + r, cp, Tc, left, left, r // 2)
            Tn, chn = Tc // r, ch * 2
            cpn = _pad_to(chn, 64)
            y = self._buf(f"h1_y{Tn}", (B * Tn, chn))
            last = st is E["stages"][-1]
            pe = None if last else self._planes(f"h1_pe{Tn}", (B, Tn + 2, cpn), pc)
            self._sconv(pd, st["down"], B, Tc, r, src_rpb=Tc + r, out_f32=rowmap(y, chn, Tn, 0), out=pe,
                        out_map=(cpn, Tn + 2, 1), act2=ACT_ELU)
            if pe is not None:
                ops.reflect_pad_rows(pe, B, Tn + 2, cpn, Tn, 1, 1, 1)
            Tc, ch = Tn, chn
            if taps is not None:
                taps[f"enc.down{r}"] = y.reshape(B, Tc, ch).transpose(1, 2).clone()
        F = Tc
        self._transformer(E["tf"], y, B, F, ch, heads=c["heads"])
        if taps is not None:
            taps["enc.tf"] = y.reshape(B, F, ch).transpose(1, 2).clone()
        pf = self._planes("h1_pf", (B, F + 2, ch), pc)
        ops.rows_to_planes(y, B, F, ch, pf, ch, F + 2, 1, act=ACT_ELU)
        ops.reflect_pad_rows(pf, B, F + 2, ch, F, 1, 1, 1)
        N = F // 2
        emb = self._buf("h1_emb", (B * N, ch))
        self._sconv(pf, E["final"], B, F, 2, src_rpb=F + 2, out_f32=rowmap(emb, ch, N, 0))
        if taps is not None:
            taps["enc.out"] = emb.reshape(B, N, ch).transpose(1, 2).clone()
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
        """vq/codec_decoder.py:54-66 -> wav [B, N*640]."""
        W = self._prepare()
        D, c = W["dec"], self.c
        C, I, Cin = c["dec_dim"], c["dec_inter"], 2 * c["dimension"]
        pc, ph = self.policy["conv"], self.policy["head"]
        zp = self._planes("h1_zp", (B * N, Cin), pc)
        ops.rows_to_planes(z, 1, B * N, Cin, zp, Cin, B * N, 0)
        up = self._buf("h1_up", (B * N, 2 * C))
        ops.gemm(zp, D["up"], 2 * C, a_batch=1, a_rows_per_batch=B * N, a_ld=Cin, m_per_batch=B * N, bias=D["up_b"],
                 out_f32=rowmap(up, 2 * C, B * N, 0))
        F = 2 * N                                   # [B*N, 2*C] == [B, 2N, C]: the sub-pixel shuffle is a view
        M = B * F
        x = self._buf("dec_x", (M, C))
        ops.dwconv(up, D["dw_w"], D["dw_b"], B, F, C, 5, x)
        if taps is not None:
            taps["dec.embed"] = x.reshape(B, F, C).transpose(1, 2).clone()
        self._resnet(D["res"][0], x, B, F, C)
        self._resnet(D["res"][1], x, B, F, C)
        self._transformer(D["tf"], x, B, F, C, heads=c["heads"])
        if taps is not None:
            taps["dec.tf"] = x.reshape(B, F, C).transpose(1, 2).clone()
        self._resnet(D["res"][5], x, B, F, C)
        self._resnet(D["res"][6], x, B, F, C)
        stats = self._buf("gn_stats", (B, 32, 2))
        h = self._buf("res_h", (M, C))
        ops.groupnorm_stats(x, B, F, C, stats)
        ops.groupnorm_apply(x, stats, D["gn_w"], D["gn_b"], B, F, C, False, out_f32=h)
        ops.layernorm(h, D["norm_w"], D["norm_b"], B, F, C, out_f32=x)
        self._convnext(D["convnext"], x, B, F, C, I)
        if taps is not None:
            taps["dec.post"] = x.reshape(B, F, C).transpose(1, 2).clone()
        t1 = self._planes("dec_fn", (M, C), ph)
        ops.layernorm(x, D["fnorm_w"], D["fnorm_b"], B, F, C, out=t1)
        n_fft, hop, nf = c["n_fft"], c["hop"], D["nf"]
        head = self._buf("dec_head", (M, D["spec_ld"]))
        self._linear(t1, D["head"], 2 * nf, M, C, bias=D["head_b"], out_f32=rowmap(head, D["spec_ld"], M, 0))
        sp = self._planes("dec_sp", (M, D["kin"]), True)
        ops.istft_pre(head, D["spec_ld"], M, nf, sp, D["kin"])
        frames = self._buf("dec_frames", (M, n_fft))
        self._linear(sp, D["dft_inv"], n_fft, M, D["kin"], out_f32=rowmap(frames, n_fft, M, 0))
        wav = torch.empty(B, F * hop, device=z.device)
        ops.istft_ola(frames, D["window"], B, F, n_fft, wav, hop)
        return wav

    # ------------------------------------------------------------------ public surface
    @torch.no_grad()
    def encode(self, x, feat, taps=None):
        """vq/codec.py:165-174: x [B,1,T] fp32, feat [B,768,T/320] fp32 -> (acoustic, semantic) int64 [B,nq,N]."""
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
        """vq/codec.py:177-186: int64 [B,nq,N] x2 -> wav [B, N*640]."""
        B, nq, N = acoustic_codes.shape
        Dq = self.quantizer.dim
        z = self._buf("dec_z", (B * N, 2 * Dq))
        ia = acoustic_codes.transpose(1, 2).reshape(B * N, nq).long().contiguous()
        isem = semantic_codes.transpose(1, 2).reshape(B * N, nq).long().contiguous()
        self.quantizer.decode_rows(ia, z, 2 * Dq, 0)
        self.semantic_quantizer.decode_rows(isem, z, 2 * Dq, Dq)
        return self._decode_z(z, B, N, taps)

    def _require_semantic_decoder(self):
        if self.sem_dec_cfg is None:
            raise RuntimeError(f"{type(self).__name__}.semantic_decode needs the semantic decoder: construct the face with "
                               "semantic_decoder=True")

    @torch.no_grad()
    def semantic_decode(self, semantic_codes):
        """vq/codec.py:161 on the codes' quantised rows: int64 [B,nq,N] -> pred_feat fp32 [B, 768, N*prod(strides)]."""
        self._require_semantic_decoder()
        B, nq, N = semantic_codes.shape
        z = self._buf("sd_zrows", (B * N, self.semantic_quantizer.dim))
        self.semantic_quantizer.decode_rows(semantic_codes.transpose(1, 2).reshape(B * N, nq).long().contiguous(), z,
                                            self.semantic_quantizer.dim, 0)
        return self._semantic_decode_rows(z, B, N)

    def forward(self, x, feat, use_mask=False, domain_split=None):
        """vq/codec.py:138-163 in evaluation mode: (recon [B, T], pred_feat fp32 [B, 768, T_feat], commit_loss 0-d fp32), recon =
        decode(*encode(x, feat)).  use_mask / domain_split are unused by the reference's forward too."""
        self._check_forward()
        with torch.no_grad():
            ac, sc = self.encode(x, feat)
            return self.decode(ac, sc), self.semantic_decode(sc), self._commit_loss()


def _planes_from_f64(w: torch.Tensor, split: bool) -> Planes:
    hi = w.clamp(-65504.0, 65504.0).half()
    lo = (w - hi.double()).half() if split else None
    return Planes(hi.contiguous(), lo.contiguous() if lo is not None else None)
