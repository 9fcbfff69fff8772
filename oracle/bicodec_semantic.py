"""CPU restatement of BiCodec `get_semantic_tokens` - the semantic half of BiCodec tokenize (SURVEY.md 8f.1).

TEST INFRASTRUCTURE - see oracle/__init__.py.  Paths relative to QuarkAudio-UniSE/model/bicodec/.

    BiCodec.get_semantic_tokens(batch) -> int64 [B, T]                                                 bicodec.py:167-172
      z      = Encoder(feat^T): VocosBackbone(input_channels -> dim, no condition) -> 2 x [SamplingBlock(ratio 1) = 3 x,
               VocosBackbone(dim -> dim, 2 layers)] -> Linear(dim -> out_channels)
               (modules/encoder_decoder/feat_encoder.py:29-90, modules/blocks/vocos.py:273-335, modules/blocks/samper.py:79-100)
      tokens = FactorizedVectorQuantize.tokenize: z_e = weight-normed 1x1 conv (in_project), F.normalize of z_e and of the
               codebook, argmax of -dist     (modules/vq/factorized_vector_quantize.py:59-61,148-152,169-187)

Everything here runs in the dtype of its inputs (the tests use float64).  The reference ships no config.yaml; ENCODER_PARAMS
restates the published Spark-TTS-0.5B `encoder` section, which cannot be checked offline.  Pinning:
oracle/make_golden_bicodec_semantic.py runs the reference's own Encoder, FactorizedVectorQuantize and BiCodecTokenizer on the seeded
weights below.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import bicodec as ob
from .weights import _gen

ENCODER_PARAMS = dict(input_channels=1024, vocos_dim=384, vocos_intermediate_dim=2048, vocos_num_layers=12, out_channels=1024,
                      sample_ratios=[1, 1])
BICODEC_SEMANTIC_FULL = dict(ob.BICODEC_FULL, encoder=ENCODER_PARAMS)


def bicodec_semantic_small():
    """the small detokenize config (quantizer 128 -> 256 x 8) with an encoder over the small wav2vec2 width (64 channels)"""
    return dict(ob.bicodec_small(), encoder=dict(input_channels=64, vocos_dim=64, vocos_intermediate_dim=192, vocos_num_layers=3,
                                                 out_channels=128, sample_ratios=[1, 1]))


# --------------------------------------------------------------------------- parameter layout
def semantic_param_specs(c):
    """reference state-dict keys of the semantic-token path without the codebook (shared with detokenize) -> (shape, kind)"""
    out = OrderedDict()
    e, q = c["encoder"], c["quantizer"]
    dim, inter = e["vocos_dim"], e["vocos_intermediate_dim"]

    def backbone(prefix, cin, layers):
        out[prefix + "embed.weight"] = ((dim, cin, 7), "w"); out[prefix + "embed.bias"] = ((dim,), "b")
        out[prefix + "norm.weight"] = ((dim,), "nw"); out[prefix + "norm.bias"] = ((dim,), "nb")
        for i in range(layers):
            b = f"{prefix}convnext.{i}."
            out[b + "gamma"] = ((dim,), ("gamma", layers))
            out[b + "dwconv.weight"] = ((dim, 1, 7), "w"); out[b + "dwconv.bias"] = ((dim,), "b")
            out[b + "norm.weight"] = ((dim,), "nw"); out[b + "norm.bias"] = ((dim,), "nb")
            out[b + "pwconv1.weight"] = ((inter, dim), "w"); out[b + "pwconv1.bias"] = ((inter,), "b")
            out[b + "pwconv2.weight"] = ((dim, inter), "w"); out[b + "pwconv2.bias"] = ((dim,), "b")
        out[prefix + "final_layer_norm.weight"] = ((dim,), "nw"); out[prefix + "final_layer_norm.bias"] = ((dim,), "nb")

    backbone("encoder.encoder.", e["input_channels"], e["vocos_num_layers"])
    for i, r in enumerate(e["sample_ratios"]):
        if r != 1:
            raise NotImplementedError("SamplingBlock ratios other than 1 (the shipped encoder uses [1, 1])")
        backbone(f"encoder.downsample.{i}.1.", dim, 2)
    out["encoder.project.weight"] = ((e["out_channels"], dim), "w"); out["encoder.project.bias"] = ((e["out_channels"],), "b")
    out["quantizer.in_project.bias"] = ((q["codebook_dim"],), "b")
    out["quantizer.in_project.weight_g"] = ((q["codebook_dim"], 1, 1), "g")
    out["quantizer.in_project.weight_v"] = ((q["codebook_dim"], q["input_dim"], 1), "w")
    return out


def make_semantic_state_dict(c, seed=0):
    """Seeded weights of the encoder and in_project, scaled as oracle.bicodec scales the prenet (fan-in weights, layer scale
    1 / layers, norm affines near the identity); in_project's gain is its |v| perturbed by 10 %."""
    sd = OrderedDict()
    for name, (shape, kind) in semantic_param_specs(c).items():
        g = _gen(seed, name)
        fan = None
        if isinstance(kind, tuple):
            kind, fan = kind
        if kind == "w":
            t = torch.randn(shape, generator=g) * (1.0 / math.prod(shape[1:])) ** 0.5
        elif kind == "b":
            t = 0.05 * torch.randn(shape, generator=g)
        elif kind == "nw":
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif kind == "nb":
            t = 0.05 * torch.randn(shape, generator=g)
        elif kind == "gamma":
            t = (1.0 / fan) * (1.0 + 0.2 * torch.randn(shape, generator=g))
        elif kind == "g":
            t = torch.zeros(shape)
        else:
            raise ValueError(kind)
        sd[name] = t
    v = sd["quantizer.in_project.weight_v"]
    nrm = v.reshape(v.shape[0], -1).norm(dim=1).reshape(v.shape[0], 1, 1)
    sd["quantizer.in_project.weight_g"] = nrm * (1.0 + 0.1 * torch.randn(nrm.shape, generator=_gen(seed, "quantizer.in_project.weight_g")))
    return sd


def synth_feat(B, T, C, seed):
    """wav2vec2-like features: unit-scale noise with a per-clip offset and a slow drift over time"""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float64)[None, :, None] / max(T, 1)
    x = torch.randn(B, T, C, generator=g, dtype=torch.float64) + 0.5 * torch.randn(B, 1, C, generator=g, dtype=torch.float64)
    return (x + torch.sin(6.0 * t + torch.randn(B, 1, C, generator=g, dtype=torch.float64))).float()


# --------------------------------------------------------------------------- forward
def encoder(sd, c, feat):
    """feat_encoder.py:79-90 on channel-last features: feat [B, T, input_channels] -> [B, T, out_channels]"""
    e = c["encoder"]
    dim = e["vocos_dim"]
    x = ob.vocos_backbone(sd, "encoder.encoder.", feat.transpose(1, 2), e["vocos_num_layers"], dim)       # [B, T, dim]
    for i, _ in enumerate(e["sample_ratios"]):
        x = ob.vocos_backbone(sd, f"encoder.downsample.{i}.1.", (x + x + x).transpose(1, 2), 2, dim)    # SamplingBlock(1) = 3 x
    return F.linear(x, sd["encoder.project.weight"], sd["encoder.project.bias"])


def fvq_scores(sd, z):
    """z [B, T, input_dim] -> (scores [B, T, K] = 2 e.c - |c|^2 with e, c L2-normalised, z_e [B, T, codebook_dim]): the
    reference's -dist (factorized_vector_quantize.py:169-187) without the row constant |e|^2"""
    w = ob.wn_weight(sd, "quantizer.in_project.")[:, :, 0]
    z_e = F.linear(z, w, sd["quantizer.in_project.bias"])
    e = F.normalize(z_e, dim=-1)
    cb = F.normalize(sd["quantizer.codebook.weight"], dim=1)
    return 2 * e @ cb.t() - cb.pow(2).sum(1), z_e


def fvq_tokenize(sd, z):
    """FactorizedVectorQuantize.tokenize: z [B, T, input_dim] -> (int64 [B, T], z_e [B, T, codebook_dim]); the first index wins
    exact ties, as torch.max"""
    s, z_e = fvq_scores(sd, z)
    return s.max(-1)[1], z_e


def fvq_margins(sd, z):
    """best score minus the second best, per token [B, T]"""
    s, _ = fvq_scores(sd, z)
    top = s.topk(2, dim=-1).values
    return top[..., 0] - top[..., 1]


@torch.no_grad()
def get_semantic_tokens(sd, c, feat, taps=None):
    """bicodec.py:167-172: feat [B, T, input_channels] -> int64 [B, T]"""
    z = encoder(sd, c, feat)
    tokens, z_e = fvq_tokenize(sd, z)
    if taps is not None:
        taps.update(encoder=z, z_e=z_e)
    return tokens
