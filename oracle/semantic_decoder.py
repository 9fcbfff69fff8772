"""CPU restatement of the codecs' semantic decoder and of `Codec.forward` in evaluation mode.

TEST INFRASTRUCTURE - see oracle/__init__.py.  Functional PyTorch-CPU code over flat state-dicts with the reference's keys; fp32 or
fp64 (the dtype follows the state-dict).  vq/semantic_module.py is byte-identical in HCodec-1.0, 1.5 and 2.0, so one restatement
serves the three codecs.  tests/test_codec_forward_host.py pins it against the reference's own `semantic_module.Decoder`.

Paths are relative to /root/reference/QuarkAudio-HCodec/HCodec-2.0/ unless stated.
"""
from __future__ import annotations

from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import adaptive as ad
from . import hcodec1 as h1
from . import hcodec15 as h15
from . import hcodec2 as h2
from .weights import make_tensor


def semantic_decoder_forward(sd, cfg, z, prefix="semantic_decoder."):
    """vq/semantic_module.py:294-299 (Decoder), :245-249 (DecoderBlock), :78-81 (ResidualUnit, ELU, bias-free convs), :84-120
    (ConvTranspose1d with padding (s+1)//2, output_padding s%2).  z [B, code_dim, N] -> [B, output_channels, N * prod(strides)]."""
    p = prefix
    h = F.conv1d(z, sd[p + "conv1.conv.weight"], None, padding=1)
    for i, st in enumerate(cfg["strides"]):
        b = f"{p}conv_blocks.{i}."
        if st == 1:
            h = F.conv1d(h, sd[b + "conv.conv.weight"], sd[b + "conv.conv.bias"], padding=1)
        else:
            h = F.conv_transpose1d(h, sd[b + "conv.deconv.weight"], sd[b + "conv.deconv.bias"], stride=st, padding=(st + 1) // 2,
                                   output_padding=st % 2)
        for u in (0, 1):
            y = F.conv1d(F.elu(h), sd[b + f"res_units.{u}.conv1.conv.weight"], None, padding=1)
            y = F.conv1d(F.elu(y), sd[b + f"res_units.{u}.conv2.weight"], None)
            h = h + y
    return F.conv1d(h, sd[p + "conv2.conv.weight"], None, padding=1)


def param_specs(cfg, prefix="semantic_decoder."):
    """name -> (shape, kind, fan) of Decoder(**cfg) (vq/semantic_module.py:252-292), the kinds of oracle/weights.py"""
    out: OrderedDict = OrderedDict()
    dc, ratios = cfg["decode_channels"], cfg.get("channel_ratios", [1] * len(cfg["strides"]))
    c0 = int(dc * ratios[0])
    out[prefix + "conv1.conv.weight"] = ((c0, cfg["code_dim"], 3), "w", cfg["code_dim"] * 3)
    cout = dc
    for i, st in enumerate(cfg["strides"]):
        cin = int(dc * ratios[i])
        cout = int(dc * ratios[i + 1]) if i + 1 < len(cfg["strides"]) else dc
        b = f"{prefix}conv_blocks.{i}."
        if st == 1:
            out[b + "conv.conv.weight"] = ((cout, cin, 3), "w", cin * 3)
            out[b + "conv.conv.bias"] = ((cout,), "b", cin * 3)
        else:       # each output frame of ConvTranspose1d(2s, s) sums 2 taps of every input channel
            out[b + "conv.deconv.weight"] = ((cin, cout, 2 * st), "w", cin * 2)
            out[b + "conv.deconv.bias"] = ((cout,), "b", cin * 2)
        for u in (0, 1):
            out[b + f"res_units.{u}.conv1.conv.weight"] = ((cout, cout, 3), "w", cout * 3)
            out[b + f"res_units.{u}.conv2.weight"] = ((cout, cout, 1), "w", cout)
    out[prefix + "conv2.conv.weight"] = ((cfg["output_channels"], cout, 3), "w", cout * 3)
    return out


def make_state_dict(cfg, seed=0):
    """seeded semantic_decoder.* tensors (oracle/weights.py's per-name generators, so they add to any codec's seeded state-dict)"""
    return OrderedDict((k, make_tensor(k, shape, kind, fan, seed)) for k, (shape, kind, fan) in param_specs(cfg).items())


def h1_config(c):
    """H-Codec-1.0 hard-codes Decoder(code_dim=512, output_channels=768, decode_channels=768, strides=(2, 1)) (HCodec-1.0/vq/
    codec.py:130-136): the quantiser width, the SSL width and the semantic encoder's width and strides of the flat config"""
    return c.get("sem_dec") or dict(code_dim=c["dimension"], output_channels=c["sem_in"], decode_channels=c["sem_ch"],
                                    channel_ratios=[1] * len(c["sem_strides"]), strides=list(c["sem_strides"]))


def _dequantize(sd, name, codes):
    B, nq, N = codes.shape
    cb = h2._codebooks(sd, name)
    return h2.rvq_decode(codes.transpose(1, 2).reshape(B * N, nq), cb).reshape(B, N, -1).transpose(1, 2)


@torch.no_grad()
def h2_forward(sd, cfg, x, feat, aten_lstm=True):
    """HCodec-2.0/vq/codec.py:54-72 in eval mode -> (recon, pred_feat, commit_loss 0)"""
    ac, sc = h2.codec_encode(sd, cfg, x, feat, aten_lstm=aten_lstm)
    recon = h2.codec_decode(sd, cfg, ac, sc, aten_lstm=aten_lstm)
    pred = semantic_decoder_forward(sd, cfg["semantic_decoder_config"], _dequantize(sd, "semantic_quantizer", sc))
    return recon, pred, torch.zeros((), dtype=recon.dtype)


@torch.no_grad()
def h1_forward(sd, c, x, feat):
    """HCodec-1.0/vq/codec.py:138-163 in eval mode -> (recon, pred_feat, commit_loss 0)"""
    ac, sc = h1.codec_encode(sd, c, x, feat)
    recon = h1.codec_decode(sd, c, ac, sc)
    pred = semantic_decoder_forward(sd, h1_config(c), _dequantize(sd, "semantic_quantizer", sc))
    return recon, pred, torch.zeros((), dtype=recon.dtype)


@torch.no_grad()
def h15_forward(sd, c, x, feat):
    """HCodec-1.5/vq/codec_adaptive.py:100-147 in eval mode -> {recon, pred_feat, commit_loss 0, token_lengths [B, G]}: the semantic
    decoder reads the de-aggregated semantic stream (:132, :139)"""
    ac, sc = h15.codec_encode(sd, c, x, feat)
    recon = h15.codec_decode(sd, c, ac, sc)
    plain, lens = ad.extract_lengths(sc, c["codebook_size"])
    pred = semantic_decoder_forward(sd, h1_config(c), _dequantize(sd, "semantic_quantizer", ad.deaggregate_by_lengths(plain, lens)))
    return dict(recon=recon, pred_feat=pred, commit_loss=torch.zeros((), dtype=recon.dtype), token_lengths=lens.long())
