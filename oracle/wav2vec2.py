"""CPU restatement of the wav2vec2 feature front end of BiCodec's tokenizer.

TEST INFRASTRUCTURE - see oracle/__init__.py.

    BiCodecTokenizer.extract_wav2vec2_features (QuarkAudio-UniSE/model/bicodec/audio_tokenizer.py:74-90):
        wav [B, L] @ 16 kHz -> Wav2Vec2FeatureExtractor (do_normalize=True: per utterance (x - mean) / sqrt(var + 1e-7),
        population variance) -> Wav2Vec2Model "wav2vec2-large-xlsr-53" (output_hidden_states) ->
        (hidden_states[11] + hidden_states[14] + hidden_states[16]) / 3                        [B, T', 1024]

wav2vec2-large-xlsr-53 is `transformers.Wav2Vec2Model` (third-party; the architecture is reproduced here from its published
definition and configuration): 7 strided convs WITH bias (k 10,3,3,3,3,2,2 / s 5,2,2,2,2,2,2), each followed by LayerNorm over
channels and GELU (feat_extract_norm="layer") -> LayerNorm -> Linear 512 -> 1024 -> + GELU(weight-normed grouped conv k=128,
16 groups, trailing sample removed) -> 24 pre-LN layers (do_stable_layer_norm: x += attn(LN(x)); x += FF(LN(x))) -> LayerNorm.
hidden_states[0] is the positional-conv output, hidden_states[k] (k < 24) the residual stream after layer k; only the last
carries `encoder.layer_norm`.  So states 11 / 14 / 16 need layers 1-16 only.  No 160/160 padding (unlike HuBERT / WavLM).
Pinning: oracle/make_golden_wav2vec2.py compares against `transformers.Wav2Vec2FeatureExtractor` and `Wav2Vec2Model` built from a
config (random weights of the same seed: the checkpoint is not available offline).
"""
from __future__ import annotations

from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import hubert as oh

WAV2VEC2_XLSR53 = dict(oh.HUBERT_BASE, hidden=1024, layers=24, heads=16, ffn=4096, hidden_state_ids=(11, 14, 16))


def wav2vec2_small():
    """reduced widths, full depth past the last averaged state (layer 17 and encoder.layer_norm stay dead)"""
    return dict(oh.hubert_small(), layers=17, hidden_state_ids=(11, 14, 16))


def param_specs(c):
    """transformers.Wav2Vec2Model state-dict keys (without masked_spec_embed) -> (shape, kind)"""
    out = OrderedDict()
    cin = 1
    for i, (co, k) in enumerate(zip(c["conv_dim"], c["conv_kernel"])):
        p = f"feature_extractor.conv_layers.{i}."
        out[p + "conv.weight"] = ((co, cin, k), "w"); out[p + "conv.bias"] = ((co,), "b")
        out[p + "layer_norm.weight"] = ((co,), "nw"); out[p + "layer_norm.bias"] = ((co,), "nb")
        cin = co
    for k, v in oh.param_specs(c).items():
        if not k.startswith("feature_extractor."):
            out[k] = v
    return out


def make_state_dict(c, seed=0):
    sd = OrderedDict()
    for name, (shape, kind) in param_specs(c).items():
        g = oh._gen(seed, name)
        if kind == "w":
            fan = 1
            for v in shape[1:]:
                fan *= v
            sd[name] = torch.randn(shape, generator=g) * (1.5 / fan) ** 0.5
        elif kind in ("b", "nb"):
            sd[name] = 0.05 * torch.randn(shape, generator=g)
        elif kind == "nw":
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif kind == "g":
            sd[name] = torch.zeros(shape)
    v = sd["encoder.pos_conv_embed.conv.parametrizations.weight.original1"]
    sd["encoder.pos_conv_embed.conv.parametrizations.weight.original0"] = v.pow(2).sum((0, 1), keepdim=True).sqrt() * 0.5
    return sd


def normalize(wav, eps=1e-7):
    """Wav2Vec2FeatureExtractor.zero_mean_unit_var_norm per utterance, statistics in fp64"""
    x = wav.double()
    m = x.mean(-1, keepdim=True)
    v = (x - m).pow(2).mean(-1, keepdim=True)
    return ((x - m) / torch.sqrt(v + eps)).float()


def feature_encoder(sd, c, wav):
    """Wav2Vec2FeatureEncoder with Wav2Vec2LayerNormConvLayer: [B, T] -> [B, C, T']"""
    x = wav[:, None]
    for i, s in enumerate(c["conv_stride"]):
        p = f"feature_extractor.conv_layers.{i}."
        x = F.conv1d(x, sd[p + "conv.weight"], sd[p + "conv.bias"], stride=s)
        x = F.layer_norm(x.transpose(1, 2), (x.shape[1],), sd[p + "layer_norm.weight"], sd[p + "layer_norm.bias"], 1e-5)
        x = F.gelu(x).transpose(1, 2)
    return x


def encoder_layer(sd, p, c, x):
    """Wav2Vec2EncoderLayerStableLayerNorm (pre-LN): x [B,T,H]"""
    B, T, H = x.shape
    h, d = c["heads"], H // c["heads"]
    lin = lambda n, t: F.linear(t, sd[p + f"{n}.weight"], sd[p + f"{n}.bias"])
    y = F.layer_norm(x, (H,), sd[p + "layer_norm.weight"], sd[p + "layer_norm.bias"], c["eps"])
    q = lin("attention.q_proj", y).view(B, T, h, d).transpose(1, 2)
    k = lin("attention.k_proj", y).view(B, T, h, d).transpose(1, 2)
    v = lin("attention.v_proj", y).view(B, T, h, d).transpose(1, 2)
    a = torch.softmax((q @ k.transpose(-1, -2)) * d ** -0.5, -1) @ v
    x = x + lin("attention.out_proj", a.transpose(1, 2).reshape(B, T, H))
    y = F.layer_norm(x, (H,), sd[p + "final_layer_norm.weight"], sd[p + "final_layer_norm.bias"], c["eps"])
    return x + lin("feed_forward.output_dense", F.gelu(lin("feed_forward.intermediate_dense", y)))


@torch.no_grad()
def hidden_states(sd, c, wav, layers=None):
    """Wav2Vec2Model(wav, output_hidden_states=True).hidden_states[: layers + 1] (all 1 + c["layers"] by default)"""
    feats = feature_encoder(sd, c, wav).transpose(1, 2)
    Cc = feats.shape[-1]
    x = F.layer_norm(feats, (Cc,), sd["feature_projection.layer_norm.weight"], sd["feature_projection.layer_norm.bias"], c["eps"])
    x = F.linear(x, sd["feature_projection.projection.weight"], sd["feature_projection.projection.bias"])
    pos = F.conv1d(x.transpose(1, 2), oh.pos_conv_weight(sd), sd["encoder.pos_conv_embed.conv.bias"], padding=c["pos_k"] // 2,
                   groups=c["pos_groups"])
    if c["pos_k"] % 2 == 0:
        pos = pos[:, :, :-1]                                # Wav2Vec2SamePadLayer
    x = x + F.gelu(pos).transpose(1, 2)
    H = x.shape[-1]
    n = c["layers"] if layers is None else layers
    hs = [x]
    for i in range(n):
        x = encoder_layer(sd, f"encoder.layers.{i}.", c, x)
        hs.append(x)
    if n == c["layers"]:
        hs[-1] = F.layer_norm(x, (H,), sd["encoder.layer_norm.weight"], sd["encoder.layer_norm.bias"], c["eps"])
    return hs


@torch.no_grad()
def extract_wav2vec2_features(sd, c, wav16k):
    """audio_tokenizer.py:74-90: normalise, run the layers the averaged states need, (hs[11] + hs[14] + hs[16]) / 3"""
    ids = c["hidden_state_ids"]
    hs = hidden_states(sd, c, normalize(wav16k), layers=max(ids))
    return sum(hs[i] for i in ids) / len(ids)
