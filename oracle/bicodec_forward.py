"""CPU restatement of BiCodec `forward` in evaluation mode (SURVEY.md 8f.1).

TEST INFRASTRUCTURE - see oracle/__init__.py.  Paths relative to QuarkAudio-UniSE/model/bicodec/.

    BiCodec.forward(batch) -> dict                                                                       bicodec.py:113-149
      tokens     = get_semantic_tokens / get_global_tokens (oracle.bicodec_semantic, oracle.bicodec_global)
      z_q        = out_project(z_e + (q - z_e)) with q the codebook row of the token (factorized_vector_quantize.py:70-140);
                   in exact arithmetic the detokenize gather out_project(q) (oracle.bicodec.fvq_detokenize)
      d_vector   = project(ResidualFSQ(perceiver(latent))) (speaker_encoder.py:85-101); in exact arithmetic the detokenize of the
                   global tokens (oracle.bicodec.speaker_detokenize, restated here in the dtype of the weights)
      x_vector   = linear(bn(ASTP(latent))), ASTP with global context (ecapa_tdnn.py:195-210, pooling_layers.py:119-144)
      x          = prenet(z_q, d_vector); pred_feat = postnet(x) (feat_decoder.Decoder without a condition, feat_decoder.py:81-97)
      recons     = WaveGenerator(x + d_vector)
      perplexity = exp(-sum p log(p + 1e-10)), p = per-code count / (B T); cluster_size = number of codes used (:97-103)
      vq_loss    = mean of two empty tensors in eval mode = NaN (:121-131)

Everything here runs in the dtype of its inputs.  The reference ships no config.yaml; POSTNET_PARAMS restates the published
Spark-TTS-0.5B `postnet` section, which cannot be checked offline.  Pinning: oracle/make_golden_bicodec_forward.py runs the reference's
own BiCodec, built with all its submodules, on the seeded weights below.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import bicodec as ob
from . import bicodec_global as og
from . import bicodec_semantic as osm
from .weights import _gen

POSTNET_PARAMS = dict(input_channels=1024, vocos_dim=384, vocos_intermediate_dim=2048, vocos_num_layers=6, out_channels=1024,
                      sample_ratios=[1, 1], use_tanh_at_final=False)
BICODEC_FORWARD_FULL = dict(osm.BICODEC_SEMANTIC_FULL, mel_params=og.MEL_PARAMS, postnet=POSTNET_PARAMS)
ASTP_BOTTLENECK = 128


def bicodec_forward_small(base):
    """`base` (the small semantic + global config) with a postnet from the prenet's width back to the encoder's input width"""
    return dict(base, postnet=dict(input_channels=base["prenet"]["out_channels"], vocos_dim=64, vocos_intermediate_dim=192,
                                   vocos_num_layers=2, out_channels=base["encoder"]["input_channels"], sample_ratios=[1, 1],
                                   use_tanh_at_final=False))


# --------------------------------------------------------------------------- parameter layout
def forward_param_specs(c):
    """reference state-dict keys of what only forward runs (the postnet and the x-vector branch, without num_batches_tracked) ->
    (shape, kind)"""
    out = OrderedDict()
    p = c["postnet"]
    dim, inter = p["vocos_dim"], p["vocos_intermediate_dim"]

    def backbone(prefix, layers):
        out[prefix + "embed.weight"] = ((dim, dim, 7), "w"); out[prefix + "embed.bias"] = ((dim,), "b")
        out[prefix + "norm.weight"] = ((dim,), "nw"); out[prefix + "norm.bias"] = ((dim,), "nb")
        for i in range(layers):
            b = f"{prefix}convnext.{i}."
            out[b + "gamma"] = ((dim,), ("gamma", layers))
            out[b + "dwconv.weight"] = ((dim, 1, 7), "w"); out[b + "dwconv.bias"] = ((dim,), "b")
            out[b + "norm.weight"] = ((dim,), "nw"); out[b + "norm.bias"] = ((dim,), "nb")
            out[b + "pwconv1.weight"] = ((inter, dim), "w"); out[b + "pwconv1.bias"] = ((inter,), "b")
            out[b + "pwconv2.weight"] = ((dim, inter), "w"); out[b + "pwconv2.bias"] = ((dim,), "b")
        out[prefix + "final_layer_norm.weight"] = ((dim,), "nw"); out[prefix + "final_layer_norm.bias"] = ((dim,), "nb")

    out["postnet.linear_pre.weight"] = ((dim, p["input_channels"]), "w"); out["postnet.linear_pre.bias"] = ((dim,), "b")
    for i, r in enumerate(p["sample_ratios"]):
        if r != 1:
            raise NotImplementedError("SamplingBlock ratios other than 1 (the shipped postnet uses [1, 1])")
        backbone(f"postnet.downsample.{i}.1.", 2)
    backbone("postnet.vocos_backbone.", p["vocos_num_layers"])
    out["postnet.linear.weight"] = ((p["out_channels"], dim), "w"); out["postnet.linear.bias"] = ((p["out_channels"],), "b")
    E, C = "speaker_encoder.speaker_encoder.", og.ECAPA_OUT
    out[E + "pool.linear1.weight"] = ((ASTP_BOTTLENECK, 3 * C, 1), "w"); out[E + "pool.linear1.bias"] = ((ASTP_BOTTLENECK,), "b")
    out[E + "pool.linear2.weight"] = ((C, ASTP_BOTTLENECK, 1), "w_att"); out[E + "pool.linear2.bias"] = ((C,), "b")
    out[E + "bn.weight"] = ((2 * C,), "bn_w"); out[E + "bn.bias"] = ((2 * C,), "bn_b")
    out[E + "bn.running_mean"] = ((2 * C,), "bn_m"); out[E + "bn.running_var"] = ((2 * C,), "bn_v")
    out[E + "linear.weight"] = ((c["speaker"]["out_dim"], 2 * C), "w"); out[E + "linear.bias"] = ((c["speaker"]["out_dim"],), "b")
    return out


def make_forward_state_dict(c, seed=0):
    """Seeded weights of the postnet (scaled as oracle.bicodec scales the prenet) and the x-vector branch: attention logits 3x the
    fan-in scale, so that the softmax over frames is far from uniform; BatchNorm statistics far from the identity."""
    sd = OrderedDict()
    for name, (shape, kind) in forward_param_specs(c).items():
        g = _gen(seed, name)
        fan = None
        if isinstance(kind, tuple):
            kind, fan = kind
        if kind == "w":
            t = torch.randn(shape, generator=g) * (1.0 / math.prod(shape[1:])) ** 0.5
        elif kind == "w_att":
            t = torch.randn(shape, generator=g) * 3.0 / math.prod(shape[1:]) ** 0.5
        elif kind == "b":
            t = 0.05 * torch.randn(shape, generator=g)
        elif kind in ("nw", "bn_w"):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif kind in ("nb", "bn_b"):
            t = 0.05 * torch.randn(shape, generator=g)
        elif kind == "gamma":
            t = (1.0 / fan) * (1.0 + 0.2 * torch.randn(shape, generator=g))
        elif kind == "bn_m":
            t = 0.2 + 0.4 * torch.rand(shape, generator=g)
        elif kind == "bn_v":
            t = 0.5 + 2.0 * torch.rand(shape, generator=g)
        else:
            raise ValueError(kind)
        sd[name] = t
    return sd


# --------------------------------------------------------------------------- forward
def postnet(sd, c, x):
    """feat_decoder.py:81-97 without a condition: x [B, input_channels, T] -> [B, out_channels, T]"""
    p = c["postnet"]
    dim = p["vocos_dim"]
    y = F.linear(x.transpose(1, 2), sd["postnet.linear_pre.weight"], sd["postnet.linear_pre.bias"])
    for i, _ in enumerate(p["sample_ratios"]):
        y = ob.vocos_backbone(sd, f"postnet.downsample.{i}.1.", (y + y + y).transpose(1, 2), 2, dim)     # SamplingBlock(1) = 3 x
    y = ob.vocos_backbone(sd, "postnet.vocos_backbone.", y.transpose(1, 2), p["vocos_num_layers"], dim)
    return F.linear(y, sd["postnet.linear.weight"], sd["postnet.linear.bias"]).transpose(1, 2)


def astp_context(latent):
    """[mean | sqrt(unbiased var + 1e-7)] over T: latent [B, C, T] -> [B, 2C]"""
    return torch.cat([latent.mean(-1), torch.sqrt(latent.var(-1) + 1e-7)], 1)


def astp_pool(latent, logits):
    """attentive [mean | sqrt(max(var, 1e-7))] with alpha = softmax over T of logits [B, C, T] -> [B, 2C]"""
    a = torch.softmax(logits, dim=2)
    mean = (a * latent).sum(2)
    var = (a * latent ** 2).sum(2) - mean ** 2
    return torch.cat([mean, torch.sqrt(var.clamp(min=1e-7))], 1)


def x_vector(sd, latent):
    """ECAPA_TDNN's linear(bn(ASTP(latent))) (ecapa_tdnn.py:206-208): latent [B, 1536, T] -> [B, out_dim]"""
    E = "speaker_encoder.speaker_encoder."
    ctx = astp_context(latent)
    C = latent.shape[1]
    x_in = torch.cat([latent, ctx[:, :C, None].expand_as(latent), ctx[:, C:, None].expand_as(latent)], 1)
    h = torch.tanh(F.conv1d(x_in, sd[E + "pool.linear1.weight"], sd[E + "pool.linear1.bias"]))
    logits = F.conv1d(h, sd[E + "pool.linear2.weight"], sd[E + "pool.linear2.bias"])
    pooled = astp_pool(latent, logits)
    y = F.batch_norm(pooled, sd[E + "bn.running_mean"], sd[E + "bn.running_var"], sd[E + "bn.weight"], sd[E + "bn.bias"], False, 0.0, 1e-5)
    return F.linear(y, sd[E + "linear.weight"], sd[E + "linear.bias"])


def fvq_usage(indices, K):
    """(perplexity, number of codes used) of indices [B, T] over K codes, in float64 (factorized_vector_quantize.py:97-103)"""
    counts = torch.bincount(indices.reshape(-1), minlength=K).double()
    p = counts / indices.numel()
    return torch.exp(-(p * torch.log(p + 1e-10)).sum()), int((counts > 0).sum())


def d_vector(sd, c, glob):
    """oracle.bicodec.speaker_detokenize in the dtype of sd (one quantizer): [B, 1, N] -> [B, out_dim]"""
    w = sd["speaker_encoder.quantizer.project_out.weight"]
    codes = ob.fsq_codes(c["speaker"]["fsq_levels"], glob[:, 0]).to(w.dtype)
    zq = F.linear(codes, w, sd["speaker_encoder.quantizer.project_out.bias"])
    return F.linear(zq.transpose(1, 2).reshape(zq.shape[0], -1), sd["speaker_encoder.project.weight"], sd["speaker_encoder.project.bias"])


@torch.no_grad()
def forward(sd, c, batch, taps=None):
    """bicodec.py:113-149 in evaluation mode on the oracle's restatements; the float outputs in the dtype of sd and the inputs"""
    sem_taps, glob_taps = {}, {}
    sem = osm.get_semantic_tokens(sd, c, batch["feat"], sem_taps)
    glob = og.get_global_tokens(sd, c, batch["ref_wav"], glob_taps)
    z_q = ob.fvq_detokenize(sd, sem)
    dvec = d_vector(sd, c, glob)
    x = ob.prenet_forward(sd, c, z_q, dvec)
    pred_feat = postnet(sd, c, x)
    recons = ob.wave_generator(sd, c, x + dvec.unsqueeze(-1))
    perplexity, active = fvq_usage(sem, c["quantizer"]["codebook_size"])
    if taps is not None:
        taps.update(semantic=sem, global_tokens=glob, latent=glob_taps["latent"], encoder=sem_taps["encoder"], prenet_out=x)
    return {"vq_loss": torch.full((), float("nan")), "perplexity": perplexity, "cluster_size": float(active), "recons": recons,
            "pred_feat": pred_feat, "x_vector": x_vector(sd, glob_taps["latent"]), "d_vector": dvec,
            "audios": batch["wav"].unsqueeze(1), "with_speaker_loss": False}
