"""CPU restatement of BiCodec `get_global_tokens` - the speaker half of BiCodec tokenize (SURVEY.md 8f.1).

TEST INFRASTRUCTURE - see oracle/__init__.py.  Paths relative to QuarkAudio-UniSE/model/bicodec/.

    BiCodec.get_global_tokens(batch) -> int32 [B, 1, token_num]                                          bicodec.py:174-178
      mel    = torchaudio MelSpectrogram(power 1, slaney norm and scale, center / reflect, periodic Hann)   bicodec.py:201-221
      latent = ECAPA_TDNN_GLOB_c512 up to relu(conv(cat(out2, out3, out4)))        modules/speaker/ecapa_tdnn.py:153-212
      x      = PerceiverResampler(latent): proj_context, 2 x [cross attention over cat(latents, x), GEGLU feed-forward], RMSNorm
                                                                                   modules/speaker/perceiver_encoder.py:297-350
      tokens = ResidualFSQ (one quantizer): project_in -> bound -> round -> codes_to_indices
                                                                modules/fsq/residual_fsq.py:158-252, finite_scalar_quantization.py

Everything here runs in the dtype of its inputs (the tests use float64).  The mel filter bank and window are restated from
torchaudio's formulas (slaney mel scale and area normalisation) rather than taken from torchaudio.  The reference ships no
config.yaml; MEL_PARAMS restates the published Spark-TTS-0.5B `mel_params`, which cannot be checked offline.  Pinning:
oracle/make_golden_bicodec_global.py runs the reference's own SpeakerEncoder and mel transformer on the seeded weights below.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

from . import bicodec as ob
from .weights import _gen

MEL_PARAMS = dict(sample_rate=16000, n_fft=1024, win_length=640, hop_length=320, mel_fmin=10, mel_fmax=None, num_mels=128)
REF_SEGMENT_DURATION, LATENT_HOP_LENGTH = 6, 320          # audio_tokenizer.py:60-64: 96000 samples, 301 mel frames

BICODEC_GLOBAL_FULL = dict(ob.BICODEC_FULL, mel_params=MEL_PARAMS)
ECAPA_C, ECAPA_SCALE, ECAPA_SE, ECAPA_OUT = 512, 8, 128, 1536   # ECAPA_TDNN_GLOB_c512 and dim_context = 512 * 3 are fixed
HEADS, DIM_HEAD, DEPTH = 8, 64, 2


def bicodec_global_small():
    """short clips, 80 mel bands, the small detokenize config's speaker (latent 16, 8 tokens); ECAPA keeps its 512 channels"""
    return dict(ob.bicodec_small(), mel_params=dict(MEL_PARAMS, num_mels=80))


def ff_inner(dim):
    return int(dim * 4 * 2 / 3)                 # FeedForward(dim, mult=4): perceiver_encoder.py:238-251


# --------------------------------------------------------------------------- parameter layout
def speaker_param_specs(c):
    """reference state-dict keys of the global-token path -> (shape, kind); the x-vector branch (pool, bn, linear) and
    BatchNorm's num_batches_tracked are not part of it"""
    out = OrderedDict()
    s, nm = c["speaker"], c["mel_params"]["num_mels"]
    E = "speaker_encoder.speaker_encoder."

    def crb(p, cin, cout, k):
        out[p + "conv.weight"] = ((cout, cin, k), "w"); out[p + "conv.bias"] = ((cout,), "b")
        bn(p + "bn.", cout)

    def bn(p, ch):
        out[p + "weight"] = ((ch,), "bn_w"); out[p + "bias"] = ((ch,), "bn_b")
        out[p + "running_mean"] = ((ch,), "bn_m"); out[p + "running_var"] = ((ch,), "bn_v")

    crb(E + "layer1.", nm, ECAPA_C, 5)
    w = ECAPA_C // ECAPA_SCALE
    for k in (2, 3, 4):
        p = f"{E}layer{k}.se_res2block."
        crb(p + "0.", ECAPA_C, ECAPA_C, 1)
        for i in range(ECAPA_SCALE - 1):
            out[f"{p}1.convs.{i}.weight"] = ((w, w, 3), "w"); out[f"{p}1.convs.{i}.bias"] = ((w,), "b")
            bn(f"{p}1.bns.{i}.", w)
        crb(p + "2.", ECAPA_C, ECAPA_C, 1)
        out[p + "3.linear1.weight"] = ((ECAPA_SE, ECAPA_C), "w"); out[p + "3.linear1.bias"] = ((ECAPA_SE,), "b")
        out[p + "3.linear2.weight"] = ((ECAPA_C, ECAPA_SE), "w"); out[p + "3.linear2.bias"] = ((ECAPA_C,), "b")
    out[E + "conv.weight"] = ((ECAPA_OUT, 3 * ECAPA_C, 1), "w"); out[E + "conv.bias"] = ((ECAPA_OUT,), "b")
    P, dim, inner = "speaker_encoder.perceiver_sampler.", s["latent_dim"], ff_inner(s["latent_dim"])
    if dim != ECAPA_OUT:
        out[P + "proj_context.weight"] = ((dim, ECAPA_OUT), "w"); out[P + "proj_context.bias"] = ((dim,), "b")
    out[P + "latents"] = ((s["token_num"], dim), "latents")
    for layer in range(DEPTH):
        q = f"{P}layers.{layer}."
        out[q + "0.to_q.weight"] = ((HEADS * DIM_HEAD, dim), "w_q")
        out[q + "0.to_kv.weight"] = ((2 * HEADS * DIM_HEAD, dim), "w")
        out[q + "0.to_out.weight"] = ((dim, HEADS * DIM_HEAD), "w")
        out[q + "1.0.weight"] = ((2 * inner, dim), "w"); out[q + "1.0.bias"] = ((2 * inner,), "b")
        out[q + "1.2.weight"] = ((dim, inner), "w"); out[q + "1.2.bias"] = ((dim,), "b")
    out[P + "norm.gamma"] = ((dim,), "bn_w")
    out["speaker_encoder.quantizer.project_in.weight"] = ((len(s["fsq_levels"]), dim), "proj_in")
    out["speaker_encoder.quantizer.project_in.bias"] = ((len(s["fsq_levels"]),), "b")
    return out


def make_speaker_state_dict(c, seed=0):
    """Seeded weights that make a test bite: BatchNorm statistics far from the identity (means 0.2-0.6, variances 1-3),
    latents with the reference's std 0.02 read through to_q weights 30x the fan-in scale (so that the tokens differ), and project_in wide enough that every FSQ dimension visits all its levels."""
    sd = OrderedDict()
    for name, (shape, kind) in speaker_param_specs(c).items():
        g = _gen(seed, name)
        if kind == "w":
            fan_in = math.prod(shape[1:])
            t = torch.randn(shape, generator=g) * (1.0 / fan_in) ** 0.5
        elif kind == "b":
            t = 0.05 * torch.randn(shape, generator=g)
        elif kind == "bn_w":
            t = 1.0 + 0.2 * torch.randn(shape, generator=g)
        elif kind == "bn_b":
            t = 0.1 * torch.randn(shape, generator=g)
        elif kind == "bn_m":
            t = 0.2 + 0.4 * torch.rand(shape, generator=g)
        elif kind == "bn_v":            # > the variance of a post-ReLU unit-scale conv output: the sequential Res2 chain stays O(1)
            t = 1.0 + 2.0 * torch.rand(shape, generator=g)
        elif kind == "w_q":             # queries of O(1) from latents of std 0.02: each token attends to its own keys
            t = torch.randn(shape, generator=g) * 30.0 / shape[1] ** 0.5
        elif kind == "latents":
            t = 0.02 * torch.randn(shape, generator=g)
        elif kind == "proj_in":
            t = torch.randn(shape, generator=g) * 3.0 / shape[1] ** 0.5
        else:
            raise ValueError(kind)
        sd[name] = t
    return sd


# --------------------------------------------------------------------------- mel front end
def hann_window(mp, dtype=torch.float64):
    """torch.hann_window(win_length) (periodic), zero-padded to the middle of n_fft as torch.stft pads it"""
    n, win = mp["n_fft"], mp["win_length"]
    k = torch.arange(win, dtype=torch.float64)
    w = 0.5 - 0.5 * torch.cos(2 * math.pi * k / win)
    out = torch.zeros(n, dtype=torch.float64)
    left = (n - win) // 2
    out[left:left + win] = w
    return out.to(dtype)


def _hz_to_mel(f):
    f = torch.as_tensor(f, dtype=torch.float64)
    logstep = math.log(6.4) / 27.0
    return torch.where(f >= 1000.0, 15.0 + torch.log(f.clamp_min(1e-10) / 1000.0) / logstep, 3.0 * f / 200.0)


def _mel_to_hz(m):
    logstep = math.log(6.4) / 27.0
    return torch.where(m >= 15.0, 1000.0 * torch.exp(logstep * (m - 15.0)), 200.0 * m / 3.0)


def mel_filterbank(mp, dtype=torch.float64):
    """torchaudio.functional.melscale_fbanks(norm="slaney", mel_scale="slaney") -> [n_fft // 2 + 1, num_mels]"""
    sr, n_fft, n_mels = mp["sample_rate"], mp["n_fft"], mp["num_mels"]
    f_min, f_max = float(mp["mel_fmin"]), float(mp["mel_fmax"] if mp["mel_fmax"] is not None else sr / 2)
    all_freqs = torch.linspace(0, sr // 2, n_fft // 2 + 1, dtype=torch.float64)
    m_pts = torch.linspace(float(_hz_to_mel(f_min)), float(_hz_to_mel(f_max)), n_mels + 2, dtype=torch.float64)
    f_pts = _mel_to_hz(m_pts)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    down = -slopes[:, :-2] / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    fb = torch.clamp(torch.minimum(down, up), min=0.0)
    fb = fb * (2.0 / (f_pts[2:n_mels + 2] - f_pts[:n_mels]))[None, :]
    return fb.to(dtype)


def mel_spectrogram(wav, mp):
    """[B, L] -> magnitude mel [B, num_mels, 1 + L // hop]"""
    dt = wav.dtype
    spec = torch.stft(wav, mp["n_fft"], mp["hop_length"], window=hann_window(mp, dt), center=True, pad_mode="reflect",
                      return_complex=True).abs()
    return torch.einsum("bft,fm->bmt", spec, mel_filterbank(mp, dt))


# --------------------------------------------------------------------------- ECAPA-TDNN / perceiver / FSQ
def _conv_relu_bn(sd, p, x, padding=0, dilation=1):
    """Conv1dReluBn (ecapa_tdnn.py:90-109), BatchNorm in eval mode (eps 1e-5)"""
    y = F.relu(F.conv1d(x, sd[p + "conv.weight"], sd[p + "conv.bias"], padding=padding, dilation=dilation))
    return F.batch_norm(y, sd[p + "bn.running_mean"], sd[p + "bn.running_var"], sd[p + "bn.weight"], sd[p + "bn.bias"], False, 0.0, 1e-5)


def _se_res2block(sd, p, x, dilation):
    """SE_Res2Block (ecapa_tdnn.py:136-150): 1x1 -> Res2 (7 sequential k3 convs) -> 1x1 -> SE -> + x"""
    y = _conv_relu_bn(sd, p + "0.", x)
    w = ECAPA_C // ECAPA_SCALE
    spx = torch.split(y, w, 1)
    outs, sp = [], None
    for i in range(ECAPA_SCALE - 1):
        sp = spx[i] if i == 0 else sp + spx[i]
        sp = F.relu(F.conv1d(sp, sd[f"{p}1.convs.{i}.weight"], sd[f"{p}1.convs.{i}.bias"], padding=dilation, dilation=dilation))
        b = f"{p}1.bns.{i}."
        sp = F.batch_norm(sp, sd[b + "running_mean"], sd[b + "running_var"], sd[b + "weight"], sd[b + "bias"], False, 0.0, 1e-5)
        outs.append(sp)
    outs.append(spx[ECAPA_SCALE - 1])
    y = _conv_relu_bn(sd, p + "2.", torch.cat(outs, 1))
    s = F.relu(F.linear(y.mean(dim=2), sd[p + "3.linear1.weight"], sd[p + "3.linear1.bias"]))
    s = torch.sigmoid(F.linear(s, sd[p + "3.linear2.weight"], sd[p + "3.linear2.bias"]))
    return x + y * s.unsqueeze(2)


def ecapa_latent(sd, mel):
    """mel [B, num_mels, T] -> latent [B, 1536, T]"""
    E = "speaker_encoder.speaker_encoder."
    o1 = _conv_relu_bn(sd, E + "layer1.", mel, padding=2)
    o2 = _se_res2block(sd, E + "layer2.se_res2block.", o1, 2)
    o3 = _se_res2block(sd, E + "layer3.se_res2block.", o2, 3)
    o4 = _se_res2block(sd, E + "layer4.se_res2block.", o3, 4)
    return F.relu(F.conv1d(torch.cat([o2, o3, o4], 1), sd[E + "conv.weight"], sd[E + "conv.bias"]))


def perceiver(sd, c, latent):
    """latent [B, 1536, T] -> [B, token_num, latent_dim] (after the final RMSNorm)"""
    P, dim = "speaker_encoder.perceiver_sampler.", c["speaker"]["latent_dim"]
    x = latent.transpose(1, 2)
    if dim != ECAPA_OUT:
        x = F.linear(x, sd[P + "proj_context.weight"], sd[P + "proj_context.bias"])
    B = x.shape[0]
    lat = sd[P + "latents"][None].expand(B, -1, -1)
    for layer in range(DEPTH):
        q_ = f"{P}layers.{layer}."
        ctx = torch.cat([lat, x], 1)
        q = F.linear(lat, sd[q_ + "0.to_q.weight"]).reshape(B, -1, HEADS, DIM_HEAD).transpose(1, 2)
        k, v = F.linear(ctx, sd[q_ + "0.to_kv.weight"]).chunk(2, dim=-1)
        k = k.reshape(B, -1, HEADS, DIM_HEAD).transpose(1, 2)
        v = v.reshape(B, -1, HEADS, DIM_HEAD).transpose(1, 2)
        att = (torch.einsum("bhid,bhjd->bhij", q, k) * DIM_HEAD ** -0.5).softmax(dim=-1)
        o = torch.einsum("bhij,bhjd->bhid", att, v).transpose(1, 2).reshape(B, -1, HEADS * DIM_HEAD)
        lat = F.linear(o, sd[q_ + "0.to_out.weight"]) + lat
        h, gate = F.linear(lat, sd[q_ + "1.0.weight"], sd[q_ + "1.0.bias"]).chunk(2, dim=-1)
        lat = F.linear(F.gelu(gate) * h, sd[q_ + "1.2.weight"], sd[q_ + "1.2.bias"]) + lat
    return F.normalize(lat, dim=-1) * dim ** 0.5 * sd[P + "norm.gamma"]


def fsq_bound(z, levels):
    """finite_scalar_quantization.py:126-131"""
    lv = torch.tensor(levels, dtype=z.dtype)
    half_l = (lv - 1) * (1 + 1e-3) / 2
    offset = torch.where(torch.tensor(levels) % 2 == 0, 0.5, 0.0).to(z.dtype)
    return (z + (offset / half_l).atanh()).tanh() * half_l - offset


def fsq_tokenize(sd, c, x):
    """x [B, N, latent_dim] -> (tokens int32 [B, 1, N], z [B, N, len(levels)] = project_in(x), the input of bound)"""
    s = c["speaker"]
    if s["fsq_num_quantizers"] != 1:
        raise NotImplementedError("residual FSQ with more than one quantizer")
    z = F.linear(x, sd["speaker_encoder.quantizer.project_in.weight"], sd["speaker_encoder.quantizer.project_in.bias"])
    q = torch.round(fsq_bound(z, s["fsq_levels"])).long()
    lv = torch.tensor(s["fsq_levels"], dtype=torch.int64)
    basis = torch.cumprod(torch.tensor([1] + list(s["fsq_levels"][:-1]), dtype=torch.int64), 0)
    idx = ((q + lv // 2) * basis).sum(-1).to(torch.int32)
    return idx[:, None, :], z


def fsq_margins(z, levels):
    """fp64 distance of bound(z) to the nearest rounding boundary (a half-integer), per decision: [..., len(levels)]"""
    b = fsq_bound(z.double(), levels)
    return ((b - torch.floor(b)) - 0.5).abs()


@torch.no_grad()
def get_global_tokens(sd, c, ref_wav, taps=None):
    """bicodec.py:174-178: ref_wav [B, L] -> int32 [B, 1, token_num]"""
    mel = mel_spectrogram(ref_wav, c["mel_params"])
    latent = ecapa_latent(sd, mel)
    x = perceiver(sd, c, latent)
    tokens, z = fsq_tokenize(sd, c, x)
    if taps is not None:
        taps.update(mel=mel, latent=latent, perceiver=x, z=z)
    return tokens


def get_ref_clip(wav, ref_segment_length):
    """audio_tokenizer.py:54-72"""
    if ref_segment_length > wav.shape[-1]:
        wav = torch.tile(wav, (1, ref_segment_length // wav.shape[-1] + 1))
    return wav[:, :ref_segment_length]
