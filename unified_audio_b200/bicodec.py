"""BiCodec `detokenize` (the decoder UniSE feeds its AR-LM tokens to) on libquark_b200 - SURVEY.md 8(f).1.

Mirrors QuarkAudio-UniSE/model/bicodec/bicodec.py:182-199:
    BiCodec(config).detokenize(semantic_tokens [B,T] int64, global_tokens [B,1,32] int64) -> wav [B,1,T*320] fp32
state_dict keys are the reference's (`quantizer.*`, `speaker_encoder.*`, `prenet.*`, `decoder.*`, old-style weight-norm
`weight_g / weight_v` pairs); by default the keys of the tokenize side (`encoder.*`, `postnet.*`, ECAPA / perceiver,
`mel_transformer.*`, `quantizer.in_project.*`) are accepted at load and ignored.  The reference ships no `config.yaml` (it comes with the
Spark-TTS-0.5B checkpoint, U/README.md:57-74); BICODEC_CONFIG and MEL_PARAMS restate that published configuration.

With `global_tokens=True` the module also holds the global-token path, bicodec.py:174-178:
    BiCodec.get_global_tokens({"ref_wav": [B, L]}) -> int32 [B, 1, token_num]
and a strict load requires its keys (`speaker_encoder.speaker_encoder.{layer1..layer4,conv}.*` with BatchNorm running statistics,
`speaker_encoder.perceiver_sampler.*`, `speaker_encoder.quantizer.project_in.*`).  Still ignored: the x-vector branch the reference
computes and discards (`speaker_encoder.speaker_encoder.{pool,bn,linear}.*`), BatchNorm's `num_batches_tracked` and
`mel_transformer.*` (window and filter bank are rebuilt from MEL_PARAMS).  Mapping: MelSpectrogram =
centred reflect framing + two-stage DFT GEMMs + |X| + the slaney filter bank as a GEMM; Conv1dReluBn = one GEMM with a ReLU
epilogue and the eval BatchNorm folded into gamma + a broadcast residual row; squeeze-excitation, the perceiver's cross attention
RMSNorm + FSQ and the feed-forward's GEGLU are kernels of csrc/speaker.cu.  Every contraction is a 3-term split.

With `semantic_tokens=True` the module also holds the semantic-token path, bicodec.py:167-172:
    BiCodec.get_semantic_tokens({"feat": [B, T, input_channels]}) -> int64 [B, T]
and a strict load requires `encoder.*` (feat_encoder.py:29-90) and `quantizer.in_project.*`.  The Encoder's three Vocos backbones
run on the same GEMM / ConvNeXt kernels as the prenet, SamplingBlock(1)'s 3 x folded into the downsample backbones' embed convs, and
`project` is one GEMM; `qb_fvq_tokenize` (csrc/rvq.cu) does in_project, the normalisation and the codebook arg-max in fp64.  Every
encoder contraction is a 3-term split whatever `precision` says (the tokens are discrete; `precision` governs detokenize).  With
both flags, `tokenize(batch)` returns (semantic_tokens, global_tokens).  `postnet.*` and `quantizer.cluster_size` are ignored.
ENCODER_PARAMS restates the published encoder section for a config without an "encoder" entry.

With `full=True` (both token paths implied) the module is the reference's whole BiCodec and runs its eval-mode forward,
bicodec.py:113-149:
    BiCodec.forward({"feat", "ref_wav", "wav"}) -> {"recons", "pred_feat", "x_vector", "d_vector", "perplexity", "cluster_size",
                                                    "vq_loss", "audios", "with_speaker_loss"}
and a strict load also requires `postnet.*` (POSTNET_PARAMS restates the published section) and the x-vector branch
`speaker_encoder.speaker_encoder.{pool,bn,linear}.*`; only `mel_transformer.*`, `quantizer.cluster_size` and BatchNorm's
`num_batches_tracked` stay ignored.  The postnet runs on the prenet's kernels; ASTP pooling and the codebook usage statistics are
kernels of csrc/speaker.cu and csrc/rvq.cu around 3-term GEMMs.

How the path maps onto the library (every arithmetic op is a libquark_b200 kernel; channel-last activations):
  * FactorizedVectorQuantize.detokenize (modules/vq/factorized_vector_quantize.py:154-167) and the residual-FSQ de-quantiser
    (modules/fsq/residual_fsq.py:112-156) are index -> row gathers from tables prepared at load
    (codebook @ out_project, implicit FSQ codebook @ project_out);
  * prenet (modules/encoder_decoder/feat_decoder.py:81-97) = Vocos ConvNeXt stacks: the H-Codec ConvNeXt kernels, with
    AdaLayerNorm (modules/blocks/vocos.py:88-111) as a per-clip scale / shift row produced by ONE GEMM for all 13 norms;
  * WaveGenerator (modules/encoder_decoder/wave_generator.py:32-91): Snake -> fp16 planes (`qb_snake_planes`), dilated k=7
    convs as TMA-im2col GEMMs with a tap spacing (`qb_gemm_desc.dilation`), and every weight-normed ConvTranspose1d
    (k, stride s) as a ceil(k/s)-tap GEMM that produces all s output phases as s*Cout columns - its row-major output IS the
    up-sampled channel-last signal, shifted by the transposed conv's padding (no col2im, no zero insertion).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import ops
from .codec import _Face, _Tree, _pad_to
from .ops import ACT_GELU, ACT_RELU, ACT_SNAKE, ACT_TANH, Planes, rowmap

BICODEC_CONFIG = dict(
    sample_rate=16000, hop=320,
    quantizer=dict(input_dim=1024, codebook_size=8192, codebook_dim=8),
    speaker=dict(out_dim=1024, latent_dim=128, token_num=32, fsq_levels=[4, 4, 4, 4, 4, 4], fsq_num_quantizers=1),
    prenet=dict(input_channels=1024, vocos_dim=384, vocos_intermediate_dim=2048, vocos_num_layers=12, out_channels=1024,
                condition_dim=1024, sample_ratios=[1, 1], use_tanh_at_final=False),
    decoder=dict(input_channel=1024, channels=1536, rates=[8, 5, 4, 2], kernel_sizes=[16, 11, 8, 4]),
)

# BiCodec's `mel_params` (bicodec.py:201-221): the published Spark-TTS-0.5B values, restated like BICODEC_CONFIG and likewise not
# verifiable offline.  A config without a "mel_params" entry uses these.
MEL_PARAMS = dict(sample_rate=16000, n_fft=1024, win_length=640, hop_length=320, mel_fmin=10, mel_fmax=None, num_mels=128)
# BiCodec's `encoder` section (the feature Encoder, feat_encoder.py:29-90): the published Spark-TTS-0.5B values, restated like
# MEL_PARAMS and likewise not verifiable offline.  A config without an "encoder" entry uses these.
ENCODER_PARAMS = dict(input_channels=1024, vocos_dim=384, vocos_intermediate_dim=2048, vocos_num_layers=12, out_channels=1024,
                      sample_ratios=[1, 1])
# BiCodec's `postnet` section (feat_decoder.Decoder without a condition, which only forward runs): restated from the published
# Spark-TTS-0.5B configuration as well as it can be recalled - it is not in the reference tree and cannot be checked offline.  A
# config with a "postnet" entry overrides it.
POSTNET_PARAMS = dict(input_channels=1024, vocos_dim=384, vocos_intermediate_dim=2048, vocos_num_layers=6, out_channels=1024,
                      sample_ratios=[1, 1], use_tanh_at_final=False)
ECAPA_C, ECAPA_SCALE, ECAPA_OUT, HEADS = 512, 8, 1536, 8   # ECAPA_TDNN_GLOB_c512, dim_context = 512 * 3, 8 heads x 64 (fixed)
ASTP_BOTTLENECK = 128                                      # ASTP's bottleneck_dim (pooling_layers.py:119), fixed

# 3-term split (True) or single-pass fp16 (False) per GEMM group; "accurate" is the default until the error budget of the
# 26-conv generator is mapped (DESIGN.md)
PRECISION = {
    "accurate": dict(prenet=True, gen=True),
    "mixed": dict(prenet=False, gen=True),
    "fast": dict(prenet=False, gen=False),
}


def _wn_spec(out, prefix, shape, n_out=None):
    """old-style weight norm (layers.py:24-29): bias, weight_g [out, 1, ...], weight_v"""
    out[prefix + "bias"] = (shape[0] if n_out is None else n_out,)
    out[prefix + "weight_g"] = (shape[0],) + (1,) * (len(shape) - 1)
    out[prefix + "weight_v"] = tuple(shape)


def _backbone_spec(out, prefix, cin, dim, inter, layers, cond):
    """VocosBackbone(input_channels=cin, dim, intermediate_dim=inter, num_layers=layers, condition_dim=cond) (vocos.py:273-335)"""
    def norm(pp):
        if cond:
            out[pp + "scale.weight"] = (dim, cond); out[pp + "scale.bias"] = (dim,)
            out[pp + "shift.weight"] = (dim, cond); out[pp + "shift.bias"] = (dim,)
        else:
            out[pp + "weight"] = (dim,); out[pp + "bias"] = (dim,)

    out[prefix + "embed.weight"] = (dim, cin, 7)
    out[prefix + "embed.bias"] = (dim,)
    norm(prefix + "norm.")
    for i in range(layers):
        b = f"{prefix}convnext.{i}."
        out[b + "gamma"] = (dim,)
        out[b + "dwconv.weight"] = (dim, 1, 7); out[b + "dwconv.bias"] = (dim,)
        norm(b + "norm.")
        out[b + "pwconv1.weight"] = (inter, dim); out[b + "pwconv1.bias"] = (inter,)
        out[b + "pwconv2.weight"] = (dim, inter); out[b + "pwconv2.bias"] = (dim,)
    out[prefix + "final_layer_norm.weight"] = (dim,); out[prefix + "final_layer_norm.bias"] = (dim,)


def _feat_decoder_spec(out, prefix, p, cond):
    """feat_decoder.Decoder (feat_decoder.py:29-79) under `prefix`: linear_pre, the SamplingBlock(1) + 2-layer backbones, the main
    backbone (AdaLayerNorm on a `cond`-wide condition, or LayerNorm when cond is None) and linear"""
    dim, inter = p["vocos_dim"], p["vocos_intermediate_dim"]
    name = prefix.rstrip(".")
    out[prefix + "linear_pre.weight"] = (dim, p["input_channels"]); out[prefix + "linear_pre.bias"] = (dim,)
    for i, r in enumerate(p["sample_ratios"]):
        if r != 1:
            raise NotImplementedError(f"{name} SamplingBlock ratios other than 1 (the shipped configuration uses [1, 1])")
        _backbone_spec(out, f"{prefix}downsample.{i}.1.", dim, dim, inter, 2, None)
    _backbone_spec(out, prefix + "vocos_backbone.", dim, dim, inter, p["vocos_num_layers"], cond)
    out[prefix + "linear.weight"] = (p["out_channels"], dim); out[prefix + "linear.bias"] = (p["out_channels"],)


def bicodec_spec(c) -> Dict[str, tuple]:
    """Reference state-dict keys -> shapes of the detokenize path."""
    out: Dict[str, tuple] = {}
    q, s, p, d = c["quantizer"], c["speaker"], c["prenet"], c["decoder"]
    wn = lambda prefix, shape, n_out=None: _wn_spec(out, prefix, shape, n_out)

    out["quantizer.codebook.weight"] = (q["codebook_size"], q["codebook_dim"])
    wn("quantizer.out_project.", (q["input_dim"], q["codebook_dim"], 1))
    out["speaker_encoder.quantizer.project_out.weight"] = (s["latent_dim"], len(s["fsq_levels"]))
    out["speaker_encoder.quantizer.project_out.bias"] = (s["latent_dim"],)
    out["speaker_encoder.project.weight"] = (s["out_dim"], s["latent_dim"] * s["token_num"])
    out["speaker_encoder.project.bias"] = (s["out_dim"],)
    _feat_decoder_spec(out, "prenet.", p, p["condition_dim"])
    ch = d["channels"]
    wn("decoder.model.0.", (ch, d["input_channel"], 7))
    for i, (k, r) in enumerate(zip(d["kernel_sizes"], d["rates"])):
        cin, cout = ch // 2 ** i, ch // 2 ** (i + 1)
        b = f"decoder.model.{i + 1}.block."
        out[b + "0.alpha"] = (1, cin, 1)
        wn(b + "1.", (cin, cout, k), cout)
        for j in range(3):
            u = f"{b}{j + 2}.block."
            out[u + "0.alpha"] = (1, cout, 1)
            wn(u + "1.", (cout, cout, 7))
            out[u + "2.alpha"] = (1, cout, 1)
            wn(u + "3.", (cout, cout, 1))
    n = len(d["rates"])
    out[f"decoder.model.{n + 1}.alpha"] = (1, ch // 2 ** n, 1)
    wn(f"decoder.model.{n + 2}.", (1, ch // 2 ** n, 7))
    return out


def speaker_spec(c) -> Dict[str, tuple]:
    """Reference state-dict keys -> shapes of the global-token path (SpeakerEncoder.tokenize, speaker_encoder.py:104-109)
    without the x-vector branch it discards (pool / bn / linear) and without BatchNorm's num_batches_tracked."""
    out: Dict[str, tuple] = {}
    s, nm, w = c["speaker"], c.get("mel_params", MEL_PARAMS)["num_mels"], ECAPA_C // ECAPA_SCALE
    E = "speaker_encoder.speaker_encoder."

    def bn(p, ch):
        for k in ("weight", "bias", "running_mean", "running_var"):
            out[p + k] = (ch,)

    def crb(p, cin, cout, k):
        out[p + "conv.weight"], out[p + "conv.bias"] = (cout, cin, k), (cout,)
        bn(p + "bn.", cout)

    crb(E + "layer1.", nm, ECAPA_C, 5)
    for k in (2, 3, 4):
        p = f"{E}layer{k}.se_res2block."
        crb(p + "0.", ECAPA_C, ECAPA_C, 1)
        for i in range(ECAPA_SCALE - 1):
            out[f"{p}1.convs.{i}.weight"], out[f"{p}1.convs.{i}.bias"] = (w, w, 3), (w,)
            bn(f"{p}1.bns.{i}.", w)
        crb(p + "2.", ECAPA_C, ECAPA_C, 1)
        out[p + "3.linear1.weight"], out[p + "3.linear1.bias"] = (128, ECAPA_C), (128,)
        out[p + "3.linear2.weight"], out[p + "3.linear2.bias"] = (ECAPA_C, 128), (ECAPA_C,)
    out[E + "conv.weight"], out[E + "conv.bias"] = (ECAPA_OUT, 3 * ECAPA_C, 1), (ECAPA_OUT,)
    P, dim, inner = "speaker_encoder.perceiver_sampler.", s["latent_dim"], int(s["latent_dim"] * 4 * 2 / 3)
    if dim != ECAPA_OUT:
        out[P + "proj_context.weight"], out[P + "proj_context.bias"] = (dim, ECAPA_OUT), (dim,)
    out[P + "latents"] = (s["token_num"], dim)
    for layer in range(2):
        q = f"{P}layers.{layer}."
        out[q + "0.to_q.weight"], out[q + "0.to_kv.weight"] = (HEADS * 64, dim), (2 * HEADS * 64, dim)
        out[q + "0.to_out.weight"] = (dim, HEADS * 64)
        out[q + "1.0.weight"], out[q + "1.0.bias"] = (2 * inner, dim), (2 * inner,)
        out[q + "1.2.weight"], out[q + "1.2.bias"] = (dim, inner), (dim,)
    out[P + "norm.gamma"] = (dim,)
    out["speaker_encoder.quantizer.project_in.weight"] = (len(s["fsq_levels"]), dim)
    out["speaker_encoder.quantizer.project_in.bias"] = (len(s["fsq_levels"]),)
    return out


def encoder_spec(c) -> Dict[str, tuple]:
    """Reference state-dict keys -> shapes of the semantic-token path: the feature Encoder (feat_encoder.py:29-90) and the
    quantiser's in_project (factorized_vector_quantize.py:59-61)"""
    out: Dict[str, tuple] = {}
    e, q = c.get("encoder", ENCODER_PARAMS), c["quantizer"]
    dim, inter = e["vocos_dim"], e["vocos_intermediate_dim"]
    _backbone_spec(out, "encoder.encoder.", e["input_channels"], dim, inter, e["vocos_num_layers"], None)
    for i, r in enumerate(e["sample_ratios"]):
        if r != 1:
            raise NotImplementedError("encoder SamplingBlock ratios other than 1 (the shipped configuration uses [1, 1])")
        _backbone_spec(out, f"encoder.downsample.{i}.1.", dim, dim, inter, 2, None)
    out["encoder.project.weight"] = (e["out_channels"], dim); out["encoder.project.bias"] = (e["out_channels"],)
    _wn_spec(out, "quantizer.in_project.", (q["codebook_dim"], q["input_dim"], 1))
    return out


def postnet_spec(c) -> Dict[str, tuple]:
    """Reference state-dict keys -> shapes of the postnet (feat_decoder.Decoder without a condition, bicodec.py:86,135), from the
    config's "postnet" entry or POSTNET_PARAMS"""
    p = c.get("postnet", POSTNET_PARAMS)
    if p.get("use_tanh_at_final", False):
        raise NotImplementedError("postnet use_tanh_at_final (False in the shipped configuration)")
    if p.get("condition_dim") is not None:
        raise NotImplementedError("a conditioned postnet (BiCodec.forward calls it without a condition, bicodec.py:135)")
    out: Dict[str, tuple] = {}
    _feat_decoder_spec(out, "postnet.", p, None)
    return out


def xvector_spec(c) -> Dict[str, tuple]:
    """Reference state-dict keys -> shapes of ECAPA_TDNN's x-vector branch (ecapa_tdnn.py:186-192,206-208): ASTP with global context
    (pooling_layers.py:119-132), BatchNorm1d over [mean | std] and the final Linear, without num_batches_tracked"""
    E = "speaker_encoder.speaker_encoder."
    out: Dict[str, tuple] = {E + "pool.linear1.weight": (ASTP_BOTTLENECK, 3 * ECAPA_OUT, 1), E + "pool.linear1.bias": (ASTP_BOTTLENECK,),
                             E + "pool.linear2.weight": (ECAPA_OUT, ASTP_BOTTLENECK, 1), E + "pool.linear2.bias": (ECAPA_OUT,)}
    for k in ("weight", "bias", "running_mean", "running_var"):
        out[E + "bn." + k] = (2 * ECAPA_OUT,)
    out[E + "linear.weight"], out[E + "linear.bias"] = (c["speaker"]["out_dim"], 2 * ECAPA_OUT), (c["speaker"]["out_dim"],)
    return out


def _ignored_prefixes(global_tokens: bool, semantic_tokens: bool, full: bool = False) -> tuple:
    """Checkpoint keys a BiCodec face accepts at load and does not hold: the postnet (forward only), the mel transformer's buffers
    (rebuilt from mel_params), the FVQ usage statistics, the side of tokenize that is not built, and with the global-token path
    the x-vector branch the reference computes and discards (speaker_encoder.py:104-109).  The whole module (`full`) holds the
    postnet and the x-vector branch; the cluster_size EMA is training state and stays ignored."""
    if full:
        return ("mel_transformer.", "quantizer.cluster_size")
    out = ("postnet.", "mel_transformer.", "quantizer.cluster_size")
    if not semantic_tokens:
        out += ("encoder.", "quantizer.in_project.")
    if global_tokens:
        out += ("speaker_encoder.speaker_encoder.pool.", "speaker_encoder.speaker_encoder.bn.", "speaker_encoder.speaker_encoder.linear.")
    else:
        out += ("speaker_encoder.speaker_encoder.", "speaker_encoder.perceiver_sampler.", "speaker_encoder.quantizer.project_in.")
    return out


def hann_window(mp) -> torch.Tensor:
    """torch.hann_window(win_length) (periodic) zero-padded to the middle of n_fft, as torch.stft applies it; fp64"""
    n, win = mp["n_fft"], mp["win_length"]
    k = torch.arange(win, dtype=torch.float64)
    out = torch.zeros(n, dtype=torch.float64)
    out[(n - win) // 2:(n - win) // 2 + win] = 0.5 - 0.5 * torch.cos(2 * math.pi * k / win)
    return out


def mel_filterbank(mp) -> torch.Tensor:
    """Slaney-scale, slaney-normalised triangular filters (torchaudio melscale_fbanks) [n_fft // 2 + 1, num_mels]; fp64"""
    def hz_to_mel(f):
        return 15.0 + math.log(f / 1000.0) / (math.log(6.4) / 27.0) if f >= 1000.0 else 3.0 * f / 200.0

    sr, n_fft, n_mels = mp["sample_rate"], mp["n_fft"], mp["num_mels"]
    f_max = float(mp["mel_fmax"]) if mp["mel_fmax"] is not None else sr / 2
    freqs = torch.linspace(0, sr // 2, n_fft // 2 + 1, dtype=torch.float64)
    m = torch.linspace(hz_to_mel(float(mp["mel_fmin"])), hz_to_mel(f_max), n_mels + 2, dtype=torch.float64)
    f = torch.where(m >= 15.0, 1000.0 * torch.exp(math.log(6.4) / 27.0 * (m - 15.0)), 200.0 * m / 3.0)
    slopes = f[None, :] - freqs[:, None]
    fb = torch.clamp(torch.minimum(-slopes[:, :-2] / (f[1:-1] - f[:-2]), slopes[:, 2:] / (f[2:] - f[1:-1])), min=0.0)
    return fb * (2.0 / (f[2:] - f[:-2]))[None, :]


def _backbone_weights(sd, prefix, layers, cond, in_scale, split):
    """A VocosBackbone's prepared weights: the embed conv as conv planes (times in_scale), the pointwise convs as planes, and the
    fp32 vectors of the depthwise convs and norms (no norm affine when the backbone is conditioned)."""
    dim = sd[prefix + "embed.bias"].shape[0]
    blocks = []
    for i in range(layers):
        b = f"{prefix}convnext.{i}."
        blk = dict(dw_w=sd[b + "dwconv.weight"].reshape(dim, 7).contiguous(), dw_b=sd[b + "dwconv.bias"].contiguous(),
                   w1=Planes.from_f32(sd[b + "pwconv1.weight"], split), b1=sd[b + "pwconv1.bias"].contiguous(),
                   w2=Planes.from_f32(sd[b + "pwconv2.weight"], split), b2=sd[b + "pwconv2.bias"].contiguous(),
                   gamma=sd[b + "gamma"].contiguous())
        if not cond:
            blk.update(ln_w=sd[b + "norm.weight"].contiguous(), ln_b=sd[b + "norm.bias"].contiguous())
        blocks.append(blk)
    out = dict(embed=ops.conv_planes(sd[prefix + "embed.weight"] * in_scale, split), embed_b=sd[prefix + "embed.bias"].contiguous(),
               blocks=blocks, fn_w=sd[prefix + "final_layer_norm.weight"].contiguous(),
               fn_b=sd[prefix + "final_layer_norm.bias"].contiguous(), layers=layers)
    if not cond:
        out.update(n_w=sd[prefix + "norm.weight"].contiguous(), n_b=sd[prefix + "norm.bias"].contiguous())
    return out


class BiCodec(_Face):
    """`global_tokens=True` adds the global-token path (`mel_spectrogram`, `get_global_tokens`) and `semantic_tokens=True` the
    semantic-token path (`get_semantic_tokens`); with both, `tokenize` returns the pair.  `full=True` is the whole reference module:
    both token paths plus the postnet and ECAPA's x-vector branch, which only `forward` runs.  Each flag makes its reference keys part
    of the module, required by a strict load.  The default object is the detokenize path alone."""

    def __init__(self, config: dict = None, precision: str = "accurate", global_tokens: Optional[bool] = None,
                 semantic_tokens: Optional[bool] = None, full: bool = False):
        super().__init__()
        self.cfg = dict(config or BICODEC_CONFIG)
        self.policy = PRECISION[precision]
        self.full = bool(full)
        if self.full and False in (global_tokens, semantic_tokens):
            raise ValueError("BiCodec(full=True) holds both token paths: global_tokens and semantic_tokens cannot be False")
        self.global_tokens, self.semantic_tokens = self.full or bool(global_tokens), self.full or bool(semantic_tokens)
        spec = bicodec_spec(self.cfg)
        if self.global_tokens:
            spec.update(speaker_spec(self.cfg))
        if self.semantic_tokens:
            spec.update(encoder_spec(self.cfg))
        if self.full:
            spec.update(postnet_spec(self.cfg))
            spec.update(xvector_spec(self.cfg))
        tree = _Tree.build(spec)
        for name, child in tree.named_children():
            self.add_module(name, child)
        self._ignored = _ignored_prefixes(self.global_tokens, self.semantic_tokens, self.full)
        self._wg = None                 # prepared weights of the global-token path
        self._we = None                 # prepared weights of the semantic-token path
        self._wf = None                 # prepared weights of what only forward runs (postnet, x-vector)
        self.eval()

    # ------------------------------------------------------------------ state
    def _ignored_key(self, key: str) -> bool:
        return key.startswith(self._ignored) or (self.global_tokens and key.endswith(".num_batches_tracked"))

    def _drop_prepared(self):
        super()._drop_prepared()
        self._wg = self._we = self._wf = None

    # ------------------------------------------------------------------ load-time weight preparation
    def _prepare(self):
        if self._w is not None:
            return self._w
        dev = self._require_cuda()
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        c = self.cfg
        q, s, p, d = c["quantizer"], c["speaker"], c["prenet"], c["decoder"]
        sp_pre, sp_gen = self.policy["prenet"], self.policy["gen"]

        def wnw(prefix):      # fold torch.nn.utils.weight_norm (dim 0): w = g * v / ||v||   (layers.py:24-29)
            v, g = sd[prefix + "weight_v"], sd[prefix + "weight_g"]
            return v * (g / v.reshape(v.shape[0], -1).norm(dim=1).reshape(g.shape))

        W = {}
        # ---- gathers
        W["zq_table"] = (sd["quantizer.codebook.weight"] @ wnw("quantizer.out_project.")[:, :, 0].t()
                         + sd["quantizer.out_project.bias"])[None].contiguous()           # [1, K, input_dim]
        levels = torch.tensor(s["fsq_levels"], dtype=torch.int64, device=dev)
        basis = torch.cumprod(torch.tensor([1] + list(s["fsq_levels"][:-1]), dtype=torch.int64, device=dev), 0)
        half = (levels // 2).float()
        ids = torch.arange(int(torch.prod(levels)), device=dev)
        implicit = (((ids[:, None] // basis) % levels).float() - half) / half             # finite_scalar_quantization.py:139-162
        if s["fsq_num_quantizers"] != 1:
            raise NotImplementedError("residual FSQ with more than one quantizer (the shipped speaker encoder uses one)")
        W["fsq_table"] = (implicit @ sd["speaker_encoder.quantizer.project_out.weight"].t()
                          + sd["speaker_encoder.quantizer.project_out.bias"])[None].contiguous()   # [1, 4096, latent]
        L, N = s["latent_dim"], s["token_num"]
        pw = sd["speaker_encoder.project.weight"].reshape(s["out_dim"], L, N).permute(0, 2, 1).reshape(s["out_dim"], N * L)
        W["spk_w"] = Planes.from_f32(pw.contiguous(), True)       # flatten order (d, n) -> gather order (n, d)
        W["spk_b"] = sd["speaker_encoder.project.bias"].contiguous()

        # ---- prenet
        W["lin_pre"] = Planes.from_f32(sd["prenet.linear_pre.weight"], sp_pre)
        W["lin_pre_b"] = sd["prenet.linear_pre.bias"].contiguous()
        # SamplingBlock(up = down = 1) returns conv_res + skip1 + skip2 = 3 x (samper.py:75-100): folded into the embed conv
        W["down"] = [_backbone_weights(sd, f"prenet.downsample.{i}.1.", 2, None, 3.0, sp_pre) for i in range(len(p["sample_ratios"]))]
        W["bb"] = _backbone_weights(sd, "prenet.vocos_backbone.", p["vocos_num_layers"], p["condition_dim"], 1.0, sp_pre)
        # all AdaLayerNorm scale / shift projections of the conditioned backbone as one [2 (L+1) dim, cond] matrix
        names = ["prenet.vocos_backbone.norm."] + [f"prenet.vocos_backbone.convnext.{i}.norm." for i in range(p["vocos_num_layers"])]
        W["cond_w"] = Planes.from_f32(torch.cat([torch.cat([sd[n + "scale.weight"], sd[n + "shift.weight"]], 0) for n in names], 0), True)
        W["cond_b"] = torch.cat([torch.cat([sd[n + "scale.bias"], sd[n + "shift.bias"]], 0) for n in names], 0).contiguous()
        W["lin"] = Planes.from_f32(sd["prenet.linear.weight"], sp_pre)
        W["lin_b"] = sd["prenet.linear.bias"].contiguous()

        # ---- WaveGenerator
        G = dict(conv0=ops.conv_planes(wnw("decoder.model.0."), sp_gen), conv0_b=sd["decoder.model.0.bias"].contiguous(), stages=[])
        ch = d["channels"]
        for i, (k, r) in enumerate(zip(d["kernel_sizes"], d["rates"])):
            cin, cout = ch // 2 ** i, ch // 2 ** (i + 1)
            b = f"decoder.model.{i + 1}.block."
            wt, J = ops.convt_planes(wnw(b + "1."), r, sp_gen)
            st = dict(alpha=sd[b + "0.alpha"].reshape(-1).contiguous(), wt=wt, J=J, k=k, s=r, cin=cin, cout=cout,
                      bt=sd[b + "1.bias"].repeat(r).contiguous(), units=[])
            for j, dil in enumerate((1, 3, 9)):
                u = f"{b}{j + 2}.block."
                st["units"].append(dict(dil=dil, a1=sd[u + "0.alpha"].reshape(-1).contiguous(), w1=ops.conv_planes(wnw(u + "1."), sp_gen),
                                        b1=sd[u + "1.bias"].contiguous(), a2=sd[u + "2.alpha"].reshape(-1).contiguous(),
                                        w2=ops.conv_planes(wnw(u + "3."), sp_gen), b2=sd[u + "3.bias"].contiguous()))
            G["stages"].append(st)
        n = len(d["rates"])
        G["alpha_f"] = sd[f"decoder.model.{n + 1}.alpha"].reshape(-1).contiguous()
        G["conv_f"] = ops.conv_planes(wnw(f"decoder.model.{n + 2}."), sp_gen)
        G["conv_f_b"] = sd[f"decoder.model.{n + 2}.bias"].contiguous()
        W["gen"] = G
        self._w = W
        return W

    # ------------------------------------------------------------------ blocks
    def _conv(self, a: Planes, w: Planes, n, B, rows_in, ld, m, taps, **kw):
        ops.gemm(a, w, n, a_batch=B, a_rows_per_batch=rows_in, a_ld=ld, m_per_batch=m, taps=taps, **kw)

    def _backbone(self, bw, x, B, T, dim, inter, cond=None, cond_stride=0, tag="", cin=None, split=None, scope=""):
        """VocosBackbone (vocos.py:273-335) on the fp32 trunk x [B*T, cin] (cin defaults to dim); returns a new fp32 [B*T, dim].
        `split` defaults to the prenet's precision; `scope` prefixes every scratch name."""
        M = B * T
        sp = self.policy["prenet"] if split is None else split
        cin = dim if cin is None else cin
        cp = _pad_to(cin, 64)
        pad = self._planes(scope + "bb_pad", (B, T + 6, cp), sp)
        ops.rows_to_planes(x, B, T, cin, pad, cp, T + 6, 3)
        y = self._buf(scope + "bb_y", (M, dim))
        self._conv(pad, bw["embed"], dim, B, T + 6, cp, T, 7, bias=bw["embed_b"], out_f32=rowmap(y, dim, T, 0))
        h = self._buf(scope + "bb_h" + tag, (M, dim))
        if cond is None:
            ops.layernorm(y, bw["n_w"], bw["n_b"], B, T, dim, out_f32=h)
        else:
            ops.adalayernorm(y, cond[0], cond[0][dim:], cond_stride, B, T, dim, out_f32=h)
        t1 = self._planes(scope + "bb_t1", (M, dim), sp)
        hid = self._planes(scope + "bb_hid", (M, inter), sp)
        hm = rowmap(h, dim, M, 0)
        for i, blk in enumerate(bw["blocks"]):
            if cond is None:
                ops.dwconv7_ln(h, blk["dw_w"], blk["dw_b"], blk["ln_w"], blk["ln_b"], B, T, dim, t1)
            else:
                cs = cond[i + 1]
                ops.dwconv7_adaln(h, blk["dw_w"], blk["dw_b"], cs, cs[dim:], cond_stride, B, T, dim, t1)
            ops.gemm(t1, blk["w1"], inter, a_batch=1, a_rows_per_batch=M, a_ld=dim, m_per_batch=M, bias=blk["b1"], act=ACT_GELU,
                     out_planes=hid, out_planes_map=(inter, M, 0))
            ops.gemm(hid, blk["w2"], dim, a_batch=1, a_rows_per_batch=M, a_ld=inter, m_per_batch=M, bias=blk["b2"],
                     gamma=blk["gamma"], residual=hm, out_f32=hm)
        out = self._buf(scope + "bb_out" + tag, (M, dim))
        ops.layernorm(h, bw["fn_w"], bw["fn_b"], B, T, dim, out_f32=out)
        return out

    # ------------------------------------------------------------------ public surface
    @torch.no_grad()
    def detokenize(self, semantic_tokens: torch.Tensor, global_tokens: torch.Tensor, taps=None) -> torch.Tensor:
        """bicodec.py:182-199"""
        pre, dvec = self._prenet(semantic_tokens, global_tokens, taps)
        return self._wave(pre, dvec, *semantic_tokens.shape, taps)

    def _prenet(self, semantic_tokens, global_tokens, taps=None):
        """the gathers (z_q, d_vector) and prenet(z_q, d_vector) of bicodec.py:193-195 -> (prenet output [B*T, out_channels], d_vector
        [B, out_dim]), both fp32 scratch"""
        W = self._prepare()
        c = self.cfg
        q, s, p = c["quantizer"], c["speaker"], c["prenet"]
        B, T = semantic_tokens.shape
        M = B * T
        D_in, dim, inter = q["input_dim"], p["vocos_dim"], p["vocos_intermediate_dim"]
        if dim % 64 or inter % 64 or D_in % 64 or p["out_channels"] % 64 or p["condition_dim"] % 64:
            raise ValueError("BiCodec widths must be multiples of 64")
        sp_pre = self.policy["prenet"]
        # ---- z_q: codebook row @ out_project, gathered  (factorized_vector_quantize.py:154-167)
        zq = self._buf("zq", (M, D_in))
        ops.rvq_decode(semantic_tokens.reshape(M, 1).long().contiguous(), W["zq_table"], M, D_in, q["codebook_size"], 1, zq, D_in, 0)
        # ---- d_vector (speaker_encoder.py:111-116)
        N, L = s["token_num"], s["latent_dim"]
        if tuple(global_tokens.shape) != (B, s["fsq_num_quantizers"], N):
            raise ValueError(f"global_tokens must be [B, {s['fsq_num_quantizers']}, {N}]")
        codes = self._buf("spk_codes", (B * N, L))
        ops.rvq_decode(global_tokens.reshape(B * N, 1).long().contiguous(), W["fsq_table"], B * N, L, W["fsq_table"].shape[1], 1,
                       codes, L, 0)
        cpl = self._planes("spk_codes_p", (B, N * L), True)
        ops.split_f16(codes, cpl)
        dvec = self._buf("dvec", (B, s["out_dim"]))
        ops.gemm(cpl, W["spk_w"], s["out_dim"], a_batch=1, a_rows_per_batch=B, a_ld=N * L, m_per_batch=B, bias=W["spk_b"],
                 out_f32=rowmap(dvec, s["out_dim"], B, 0))
        # ---- AdaLayerNorm rows for all 13 norms: [B, (layers + 1) * 2 * dim]
        n_norm = p["vocos_num_layers"] + 1
        dpl = self._planes("dvec_p", (B, s["out_dim"]), True)
        ops.split_f16(dvec, dpl)
        cond = self._buf("cond", (B, n_norm * 2 * dim))
        ops.gemm(dpl, W["cond_w"], n_norm * 2 * dim, a_batch=1, a_rows_per_batch=B, a_ld=p["condition_dim"], m_per_batch=B,
                 bias=W["cond_b"], out_f32=rowmap(cond, n_norm * 2 * dim, B, 0))
        cond_rows = [cond.view(-1)[j * 2 * dim:] for j in range(n_norm)]        # scale at +0, shift at +dim, stride = row
        # ---- prenet (feat_decoder.py:81-97)
        zpl = self._planes("zq_p", (M, D_in), sp_pre)
        ops.split_f16(zq, zpl) if sp_pre else ops.rows_to_planes(zq, 1, M, D_in, zpl, D_in, M, 0)
        x = self._buf("pre_x", (M, dim))
        ops.gemm(zpl, W["lin_pre"], dim, a_batch=1, a_rows_per_batch=M, a_ld=D_in, m_per_batch=M, bias=W["lin_pre_b"],
                 out_f32=rowmap(x, dim, M, 0))
        for i, bw in enumerate(W["down"]):
            x = self._backbone(bw, x, B, T, dim, inter, tag=f"_d{i}")
        x = self._backbone(W["bb"], x, B, T, dim, inter, cond_rows, n_norm * 2 * dim, tag="_c")
        xpl = self._planes("pre_out_p", (M, dim), sp_pre)
        ops.split_f16(x, xpl) if sp_pre else ops.rows_to_planes(x, 1, M, dim, xpl, dim, M, 0)
        C0 = p["out_channels"]
        pre = self._buf("pre_out", (M, C0))
        ops.gemm(xpl, W["lin"], C0, a_batch=1, a_rows_per_batch=M, a_ld=dim, m_per_batch=M, bias=W["lin_b"],
                 out_f32=rowmap(pre, C0, M, 0))
        if p["use_tanh_at_final"]:
            raise NotImplementedError("prenet use_tanh_at_final (False in the shipped configuration)")
        if taps is not None:
            taps["z_q"], taps["d_vector"], taps["prenet.out"] = zq.clone(), dvec.clone(), pre.clone()
        return pre, dvec

    def _wave(self, pre, dvec, B, T, taps=None):
        """WaveGenerator(prenet output + d_vector) (bicodec.py:196-197) -> fresh wav [B, 1, T * hop]"""
        W = self._prepare()
        C0, d = self.cfg["prenet"]["out_channels"], self.cfg["decoder"]
        dev = self._dev()
        sp_gen = self.policy["gen"]
        # ---- WaveGenerator (wave_generator.py:59-91)
        # Every Snake but one per stage rides in a GEMM epilogue: a conv's fp32 output is the residual trunk, its fp16-plane
        # output is Snake_alpha(trunk) written straight into the interior of the NEXT convolution's zero-padded buffer
        # (qb_gemm_desc.act2 / act2_param); the dilated conv's own Snake is `act`.  Only the transposed conv's output - all
        # s phases of a frame in one row, shifted by the padding - needs the stand-alone Snake kernel.
        G = W["gen"]
        a0 = self._planes("gen_in", (B, T + 6, C0), sp_gen)
        ops.addvec_planes(pre, dvec, B, T, C0, a0, C0, T + 6, 3)                    # x + d_vector[:, :, None]  (bicodec.py:197)
        ch = d["channels"]
        stages = G["stages"]

        def up_in(si, Tc):      # padded input buffer of stage si's transposed conv
            st = stages[si]
            cpi = _pad_to(st["cin"], 64)
            return self._planes(f"gen_up_in{si}", (B, Tc + 2 * (st["J"] - 1), cpi), sp_gen), cpi, Tc + 2 * (st["J"] - 1), st["J"] - 1

        Tc = T
        nxt_pl, nxt_ld, nxt_rpb, nxt_off = up_in(0, Tc)
        self._conv(a0, G["conv0"], ch, B, T + 6, C0, T, 7, bias=G["conv0_b"], act2=ACT_SNAKE, act2_param=stages[0]["alpha"],
                   out_planes=nxt_pl, out_planes_map=(nxt_ld, nxt_rpb, nxt_off))
        cl = ch // 2 ** len(d["rates"])
        for si, st in enumerate(stages):
            cin, cout, J, sdn, k = st["cin"], st["cout"], st["J"], st["s"], st["k"]
            cpo = _pad_to(cout, 64)
            a, cpi, rows_in, _ = up_in(si, Tc)
            # transposed conv as a J-tap GEMM producing all `s` phases of every input frame
            up = self._buf(f"gen_up{si}", (B, Tc + J - 1, sdn * cout))
            self._conv(a, st["wt"], sdn * cout, B, rows_in, cpi, Tc + J - 1, J, bias=st["bt"],
                       out_f32=rowmap(up, sdn * cout, Tc + J - 1, 0))
            pad_t = (k - sdn) // 2
            Tn = Tc * sdn
            # the up-sampled clip b is rows [pad_t, pad_t + Tn) of up[b] viewed as [(Tc + J - 1) * s, cout]
            res = rowmap(up, cout, (Tc + J - 1) * sdn, pad_t)
            units = st["units"]
            bufs = [self._planes(f"gen_u{si}_{u['dil']}", (B, Tn + 6 * u["dil"], cpo), sp_gen) for u in units]
            ops.snake_planes(up.view(-1)[pad_t * cout:], (Tc + J - 1) * sdn * cout, units[0]["a1"], B, Tn, cout, bufs[0], cpo,
                             Tn + 6 * units[0]["dil"], 3 * units[0]["dil"])
            a2 = self._planes(f"gen_v{si}", (B * Tn, cpo), sp_gen)
            dense = [self._buf(f"gen_x{si}a", (B * Tn, cout)), self._buf(f"gen_x{si}b", (B * Tn, cout))]
            for ui, un in enumerate(units):
                dil = un["dil"]
                # Snake -> dilated k7 conv -> Snake (epilogue) -> planes
                self._conv(bufs[ui], un["w1"], cout, B, Tn + 6 * dil, cpo, Tn, 7, dilation=dil, bias=un["b1"], act=ACT_SNAKE,
                           act_param=un["a2"], out_planes=a2, out_planes_map=(cpo, Tn, 0))
                # 1x1 conv + residual -> fp32 trunk, and Snake(trunk) planes for whoever consumes it next
                last = ui == len(units) - 1
                if not last:
                    nd = units[ui + 1]["dil"]
                    n_pl, n_ld, n_rpb, n_off, n_alpha = bufs[ui + 1], cpo, Tn + 6 * nd, 3 * nd, units[ui + 1]["a1"]
                elif si + 1 < len(stages):
                    n_pl, n_ld, n_rpb, n_off = up_in(si + 1, Tn)
                    n_alpha = stages[si + 1]["alpha"]
                else:
                    cpf = _pad_to(cl, 64)
                    n_pl, n_ld, n_rpb, n_off, n_alpha = self._planes("gen_f", (B, Tn + 6, cpf), sp_gen), cpf, Tn + 6, 3, G["alpha_f"]
                nxt = dense[ui & 1]
                need_f32 = (not last) or taps is not None
                ops.gemm(a2, un["w2"], cout, a_batch=B, a_rows_per_batch=Tn, a_ld=cpo, m_per_batch=Tn, bias=un["b2"], residual=res,
                         out_f32=rowmap(nxt, cout, Tn, 0) if need_f32 else None, act2=ACT_SNAKE, act2_param=n_alpha,
                         out_planes=n_pl, out_planes_map=(n_ld, n_rpb, n_off))
                res = rowmap(nxt, cout, Tn, 0)
            Tc = Tn
            if taps is not None:
                taps[f"dec.stage{si}"] = dense[(len(units) - 1) & 1].clone().reshape(B, Tc, cout)
        cpf = _pad_to(cl, 64)
        af = self._planes("gen_f", (B, Tc + 6, cpf), sp_gen)
        wav = torch.empty(B, 1, Tc, device=dev)
        self._conv(af, G["conv_f"], 1, B, Tc + 6, cpf, Tc, 7, bias=G["conv_f_b"], act=ACT_TANH, out_f32=rowmap(wav, 1, Tc, 0))
        return wav

    # ------------------------------------------------------------------ global (speaker) tokens
    def _mel_params(self):
        return self.cfg.get("mel_params", MEL_PARAMS)

    def _prepare_global(self):
        if self._wg is not None:
            return self._wg
        if not self.global_tokens:
            raise RuntimeError("this BiCodec was built without the global-token path: construct it with BiCodec(..., global_tokens=True)")
        dev = self._require_cuda()
        keys = speaker_spec(self.cfg)
        sd = {k: v.detach().double().cpu() for k, v in self.state_dict().items() if k in keys}
        mp, s = self._mel_params(), self.cfg["speaker"]
        n_fft, nf = mp["n_fft"], mp["n_fft"] // 2 + 1
        if n_fft % 64 or n_fft > 4096 or mp["win_length"] > n_fft:
            raise ValueError("mel_params: the two-stage DFT needs n_fft a multiple of 64, at most 4096, and win_length <= n_fft")
        if s["fsq_num_quantizers"] != 1:
            raise NotImplementedError("residual FSQ with more than one quantizer (the shipped speaker encoder uses one)")

        def f32(t):
            return t.float().contiguous().to(dev)

        def pl(w):
            return Planes.from_f32(f32(w), True)

        def crb(p, w, b):          # Conv1dReluBn: conv -> ReLU -> eval BatchNorm as the GEMM's gamma and broadcast residual row
            g = sd[p + "bn.weight"] / torch.sqrt(sd[p + "bn.running_var"] + 1e-5)
            return dict(w=w, b=f32(b), g=f32(g), t=f32(sd[p + "bn.bias"] - sd[p + "bn.running_mean"] * g))

        G: dict = {}
        # ---- mel: two-stage DFT n_fft = P * Q (P = 64) on the GEMM, as the H-Codec STFT (csrc/elementwise.cu)
        P, Q = 64, n_fft // 64
        K2 = (nf - 1) // P + 1
        ang = lambda num, den: 2 * math.pi * (num % den).double() / den
        a, k1 = torch.arange(P)[None, :], torch.arange(P)[:, None]
        wA = torch.zeros(2 * P, 64, dtype=torch.float64)
        wA[0::2, :P], wA[1::2, :P] = torch.cos(ang(k1 * a, P)), -torch.sin(ang(k1 * a, P))
        b_, k2 = torch.arange(Q)[None, :], torch.arange(K2)[:, None]
        wB = torch.zeros(2 * K2, 128, dtype=torch.float64)
        wB[0::2, :Q], wB[0::2, Q:2 * Q] = torch.cos(ang(k2 * b_, Q)), torch.sin(ang(k2 * b_, Q))
        wB[1::2, :Q], wB[1::2, Q:2 * Q] = -torch.sin(ang(k2 * b_, Q)), torch.cos(ang(k2 * b_, Q))
        bb, kk = torch.arange(Q)[:, None], torch.arange(P)[None, :]
        tw = torch.stack([torch.cos(ang(bb * kk, n_fft)), -torch.sin(ang(bb * kk, n_fft))], -1)       # [b, k1, (cos, -sin)]
        fp = _pad_to(nf, 64)
        G.update(P=P, Q=Q, K2=K2, ldX=_pad_to(2 * K2, 4), fp=fp, wA=pl(wA), wB=pl(wB), tw=f32(tw), window=f32(hann_window(mp)),
                 fb=ops.pad_k_planes(f32(mel_filterbank(mp).t()), fp))
        # ---- ECAPA-TDNN up to its latent
        E = "speaker_encoder.speaker_encoder."
        G["l1"] = crb(E + "layer1.", ops.conv_planes(f32(sd[E + "layer1.conv.weight"])), sd[E + "layer1.conv.bias"])
        G["blocks"] = []
        for k in (2, 3, 4):
            p = f"{E}layer{k}.se_res2block."
            res2 = []
            for i in range(ECAPA_SCALE - 1):
                g = sd[f"{p}1.bns.{i}.weight"] / torch.sqrt(sd[f"{p}1.bns.{i}.running_var"] + 1e-5)
                res2.append(dict(w=ops.conv_planes(f32(sd[f"{p}1.convs.{i}.weight"])), b=f32(sd[f"{p}1.convs.{i}.bias"]), g=f32(g),
                                 t=f32(sd[f"{p}1.bns.{i}.bias"] - sd[f"{p}1.bns.{i}.running_mean"] * g)))
            G["blocks"].append(dict(
                dil=k, res2=res2,
                c0=crb(p + "0.", pl(sd[p + "0.conv.weight"][:, :, 0]), sd[p + "0.conv.bias"]),
                c2=crb(p + "2.", pl(sd[p + "2.conv.weight"][:, :, 0]), sd[p + "2.conv.bias"]),
                se=[f32(sd[p + n]) for n in ("3.linear1.weight", "3.linear1.bias", "3.linear2.weight", "3.linear2.bias")]))
        G["conv"], G["conv_b"] = pl(sd[E + "conv.weight"][:, :, 0]), f32(sd[E + "conv.bias"])
        # ---- perceiver: K padded to a multiple of 64
        Pp, dim = "speaker_encoder.perceiver_sampler.", s["latent_dim"]
        dp, inner = _pad_to(dim, 64), int(dim * 4 * 2 / 3)
        if dim == ECAPA_OUT:
            raise NotImplementedError("latent_dim == 1536 (PerceiverResampler without proj_context)")
        G.update(dim=dim, dp=dp, inner=inner, ip=_pad_to(inner, 64), proj=pl(sd[Pp + "proj_context.weight"]),
                 proj_b=f32(sd[Pp + "proj_context.bias"]), latents=f32(sd[Pp + "latents"]), layers=[])
        for layer in range(2):
            q = f"{Pp}layers.{layer}."
            G["layers"].append(dict(wq=ops.pad_k_planes(f32(sd[q + "0.to_q.weight"]), dp), wkv=ops.pad_k_planes(f32(sd[q + "0.to_kv.weight"]), dp),
                                    wo=pl(sd[q + "0.to_out.weight"]), w1=ops.pad_k_planes(f32(sd[q + "1.0.weight"]), dp), b1=f32(sd[q + "1.0.bias"]),
                                    w2=ops.pad_k_planes(f32(sd[q + "1.2.weight"]), _pad_to(inner, 64)), b2=f32(sd[q + "1.2.bias"])))
        G.update(gamma=f32(sd[Pp + "norm.gamma"]), w_in=f32(sd["speaker_encoder.quantizer.project_in.weight"]),
                 b_in=f32(sd["speaker_encoder.quantizer.project_in.bias"]))
        self._wg = G
        return G

    def _check_wav(self, wav):
        if not isinstance(wav, torch.Tensor) or wav.ndim not in (2, 3) or (wav.ndim == 3 and wav.shape[1] != 1):
            raise ValueError("ref_wav must be [B, L] or [B, 1, L]")
        if wav.device.type != "cuda":
            raise RuntimeError("unified_audio_b200.BiCodec runs on CUDA only (no CPU fallback): ref_wav is on the CPU")
        wav = wav.reshape(wav.shape[0], wav.shape[-1]).float().contiguous()
        if wav.shape[-1] <= self._mel_params()["n_fft"] // 2:
            raise ValueError(f"ref_wav needs more than n_fft / 2 = {self._mel_params()['n_fft'] // 2} samples (reflect padding)")
        return wav

    def _mel(self, G, wav):
        """MelSpectrogram (bicodec.py:201-221) -> fp32 mel [B*T, num_mels] (channel-last) and the planes of layer1's input buffer"""
        mp = self._mel_params()
        B, L = wav.shape
        T, M, nm = 1 + L // mp["hop_length"], B * (1 + L // mp["hop_length"]), mp["num_mels"]
        P, Q, K2, ldX, fp = G["P"], G["Q"], G["K2"], G["ldX"], G["fp"]
        ga = self._planes("mel_frames", (M * Q, 64), True)
        ops.mel_gather(wav, mp["hop_length"], mp["n_fft"], P, Q, G["window"], ga)
        Y = self._buf("mel_y", (M * Q, 2 * P))
        ops.gemm(ga, G["wA"], 2 * P, a_batch=1, a_rows_per_batch=M * Q, a_ld=64, m_per_batch=M * Q, out_f32=rowmap(Y, 2 * P, M * Q, 0))
        Z = self._planes("mel_z", (M * P, 128), True)
        ops.stft_twiddle(Y, 2 * P, M, P, Q, G["tw"], Z)
        X = self._buf("mel_x", (M * P, ldX))
        ops.gemm(Z, G["wB"], 2 * K2, a_batch=1, a_rows_per_batch=M * P, a_ld=128, m_per_batch=M * P, out_f32=rowmap(X, ldX, M * P, 0))
        mag = self._planes("mel_mag", (M, fp), True)
        ops.spec_magnitude(X, ldX, M, mp["n_fft"] // 2 + 1, P, mag, fp)
        cp = _pad_to(nm, 64)
        x0 = self._planes("ecapa_in", (B, T + 4, cp), True)
        mel = self._buf("mel", (M, nm))
        ops.gemm(mag, G["fb"], nm, a_batch=B, a_rows_per_batch=T, a_ld=fp, m_per_batch=T, out_f32=rowmap(mel, nm, T, 0),
                 out_planes=x0, out_planes_map=(cp, T + 4, 2))
        return mel, x0, T

    @torch.no_grad()
    def mel_spectrogram(self, wav: torch.Tensor) -> torch.Tensor:
        """The reference's mel_transformer(wav).squeeze(1): wav [B, L] or [B, 1, L] -> fp32 [B, num_mels, 1 + L // hop]"""
        G = self._prepare_global()
        wav = self._check_wav(wav)
        mel, _, T = self._mel(G, wav)
        return mel.reshape(wav.shape[0], T, -1).transpose(1, 2).contiguous()

    def _crb(self, a, cw, n, **kw):
        ops.gemm(a, cw["w"], n, bias=cw["b"], act=ACT_RELU, gamma=cw["g"], residual=rowmap(cw["t"], 0, 0, 0), **kw)

    @torch.no_grad()
    def get_global_tokens(self, batch, taps=None) -> torch.Tensor:
        """bicodec.py:174-178: batch["ref_wav"] [B, L] (or [B, 1, L]) -> int32 [B, 1, token_num], the layout detokenize takes.
        taps (a dict) receives channel-last fp32 copies: "mel" [B, T, num_mels], "latent" [B, T, 1536], "perceiver" [B, N, dim]
        and "z" [B, N, len(fsq_levels)], the project_in output that the FSQ bound rounds."""
        return self._global_tokens(batch["ref_wav"] if isinstance(batch, dict) else batch, taps)[0]

    def _global_tokens(self, wav, taps=None, keep_latent=False):
        """get_global_tokens on ref_wav -> (indices, the ECAPA latent as fp32 scratch [B*T, 1536] when taps or keep_latent is given,
        else None, and its 3-term planes, T)"""
        G = self._prepare_global()
        wav = self._check_wav(wav)
        B = wav.shape[0]
        mel, x0, T = self._mel(G, wav)
        M, C, w = B * T, ECAPA_C, ECAPA_C // ECAPA_SCALE
        # ---- ECAPA-TDNN (ecapa_tdnn.py:195-205): channel-last fp32 trunks, fp16 hi / lo planes for every contraction
        cat = self._planes("ecapa_cat", (M, 3 * C), True)
        trunk = [self._buf("ecapa_x0", (M, C)), self._buf("ecapa_x1", (M, C))]
        inp = self._planes("ecapa_o1", (M, C), True)
        self._crb(x0, G["l1"], C, a_batch=B, a_rows_per_batch=T + 4, a_ld=x0.hi.shape[-1], m_per_batch=T, taps=5,
                  out_f32=rowmap(trunk[0], C, T, 0), out_planes=inp, out_planes_map=(C, T, 0))
        in_ld, in_off = C, 0
        y, z = self._buf("ecapa_y", (M, C)), self._buf("ecapa_z", (M, C))
        yp, gate = self._planes("ecapa_yp", (M, C), True), self._buf("ecapa_se", (B, C))
        for bi, blk in enumerate(G["blocks"]):
            x_in, x_out, d = trunk[bi & 1], trunk[(bi + 1) & 1], blk["dil"]
            self._crb(inp, blk["c0"], C, a_batch=1, a_rows_per_batch=M, a_ld=in_ld, a_cols=C, a_col_off=in_off, m_per_batch=M,
                      out_f32=rowmap(y, C, M, 0))
            # Res2Conv1dReluBn (ecapa_tdnn.py:68-83): chunk i's conv reads spx[i] + out[i - 1]; out[i] overwrites spx[i] in y
            sp = self._planes(f"ecapa_sp{d}", (B, T + 2 * d, w), True)
            for i, rw in enumerate(blk["res2"]):
                ops.add_planes(y.view(-1)[w * i:], C, y.view(-1)[w * (i - 1):] if i else None, C, B, T, w, sp, w, T + 2 * d, d)
                self._crb(sp, rw, w, a_batch=B, a_rows_per_batch=T + 2 * d, a_ld=w, m_per_batch=T, taps=3, dilation=d,
                          out_f32=rowmap(y.view(-1)[w * i:], C, T, 0))
            ops.split_f16(y, yp)
            self._crb(yp, blk["c2"], C, a_batch=1, a_rows_per_batch=M, a_ld=C, m_per_batch=M, out_f32=rowmap(z, C, M, 0))
            ops.se_gate(z, B, T, C, *blk["se"], gate)
            ops.se_apply(z, gate, x_in, B, T, C, out=x_out, planes=cat, ld=3 * C, col_off=bi * C)
            inp, in_ld, in_off = cat, 3 * C, bi * C
        latp = self._planes("ecapa_latent_p", (M, ECAPA_OUT), True)
        lat32 = self._buf("ecapa_latent", (M, ECAPA_OUT)) if taps is not None or keep_latent else None
        ops.gemm(cat, G["conv"], ECAPA_OUT, a_batch=1, a_rows_per_batch=M, a_ld=3 * C, m_per_batch=M, bias=G["conv_b"], act=ACT_RELU,
                 out_f32=rowmap(lat32, ECAPA_OUT, M, 0) if lat32 is not None else None, out_planes=latp, out_planes_map=(ECAPA_OUT, M, 0))
        # ---- PerceiverResampler (perceiver_encoder.py:339-350); context rows 0..N-1 = the current latents, N.. = proj_context(x)
        s = self.cfg["speaker"]
        N, D, dp, ip = s["token_num"], G["dim"], G["dp"], G["ip"]
        Nk, R = N + T, B * N
        ctx = self._planes("pc_ctx", (B, Nk, dp), True)
        ops.gemm(latp, G["proj"], D, a_batch=B, a_rows_per_batch=T, a_ld=ECAPA_OUT, m_per_batch=T, bias=G["proj_b"], out_planes=ctx,
                 out_planes_map=(dp, Nk, N))
        lat = self._buf("pc_lat", (R, D))
        lat.view(B, N, D).copy_(G["latents"].expand(B, N, D))
        lp, att = self._planes("pc_lat_p", (R, dp), True), self._planes("pc_att", (R, HEADS * 64), True)
        q, kv = self._buf("pc_q", (R, HEADS * 64)), self._buf("pc_kv", (B * Nk, 2 * HEADS * 64))
        hid, ffh = self._planes("pc_hid", (R, ip), True), self._buf("pc_ffh", (R, 2 * G["inner"]))
        lm = rowmap(lat, D, R, 0)
        for L in G["layers"]:
            ops.rows_to_planes(lat, B, N, D, ctx, dp, Nk, 0)
            ops.rows_to_planes(lat, 1, R, D, lp, dp, R, 0)
            ops.gemm(lp, L["wq"], HEADS * 64, a_batch=1, a_rows_per_batch=R, a_ld=dp, m_per_batch=R, out_f32=rowmap(q, HEADS * 64, R, 0))
            ops.gemm(ctx, L["wkv"], 2 * HEADS * 64, a_batch=1, a_rows_per_batch=B * Nk, a_ld=dp, m_per_batch=B * Nk,
                     out_f32=rowmap(kv, 2 * HEADS * 64, B * Nk, 0))
            ops.cross_attention(q, kv, B, N, Nk, HEADS, att)
            ops.gemm(att, L["wo"], D, a_batch=1, a_rows_per_batch=R, a_ld=HEADS * 64, m_per_batch=R, residual=lm, out_f32=lm)
            ops.rows_to_planes(lat, 1, R, D, lp, dp, R, 0)
            ops.gemm(lp, L["w1"], 2 * G["inner"], a_batch=1, a_rows_per_batch=R, a_ld=dp, m_per_batch=R, bias=L["b1"],
                     out_f32=rowmap(ffh, 2 * G["inner"], R, 0))
            ops.geglu_planes(ffh, R, G["inner"], hid, ip)
            ops.gemm(hid, L["w2"], D, a_batch=1, a_rows_per_batch=R, a_ld=ip, m_per_batch=R, bias=L["b2"], residual=lm, out_f32=lm)
        # ---- RMSNorm + ResidualFSQ (one quantizer) -> int32 indices [B, 1, N]
        idx = torch.empty(B, 1, N, dtype=torch.int32, device=wav.device)
        nl = len(s["fsq_levels"])
        zt = torch.empty(R, nl, device=wav.device) if taps is not None else None
        xn = torch.empty(R, D, device=wav.device) if taps is not None else None
        ops.fsq_tokenize(lat, R, D, G["gamma"], G["w_in"], G["b_in"], s["fsq_levels"], s["fsq_num_quantizers"], idx, zt, xn)
        if taps is not None:
            taps.update(mel=mel.clone().reshape(B, T, -1), latent=lat32.clone().reshape(B, T, ECAPA_OUT), perceiver=xn.reshape(B, N, D),
                        z=zt.reshape(B, N, nl))
        return idx, lat32, latp, T

    # ------------------------------------------------------------------ semantic tokens
    def _prepare_semantic(self):
        if self._we is not None:
            return self._we
        if not self.semantic_tokens:
            raise RuntimeError("this BiCodec was built without the semantic-token path: construct it with BiCodec(..., semantic_tokens=True)")
        self._require_cuda()
        e, q = self.cfg.get("encoder", ENCODER_PARAMS), self.cfg["quantizer"]
        if any(w % 64 for w in (e["input_channels"], e["vocos_dim"], e["vocos_intermediate_dim"], e["out_channels"])):
            raise ValueError("BiCodec encoder widths must be multiples of 64")
        if q["input_dim"] != e["out_channels"]:
            raise ValueError("quantizer input_dim must equal the encoder's out_channels")
        keys = set(encoder_spec(self.cfg)) | {"quantizer.codebook.weight"}
        sd ={k: v.detach().float() for k, v in self.state_dict().items() if k in keys}
        # every encoder contraction is a 3-term split whatever `precision` says: the outputs are discrete
        E = dict(enc=_backbone_weights(sd, "encoder.encoder.", e["vocos_num_layers"], None, 1.0, True),
                 down=[_backbone_weights(sd, f"encoder.downsample.{i}.1.", 2, None, 3.0, True) for i in range(len(e["sample_ratios"]))],
                 proj=Planes.from_f32(sd["encoder.project.weight"], True), proj_b=sd["encoder.project.bias"].contiguous())
        v, g = sd["quantizer.in_project.weight_v"].double(), sd["quantizer.in_project.weight_g"].double()
        E["w_in"] = (v * (g / v.reshape(v.shape[0], -1).norm(dim=1).reshape(g.shape)))[:, :, 0].float().contiguous()
        E["b_in"] = sd["quantizer.in_project.bias"].contiguous()
        E["cb_n"] = torch.nn.functional.normalize(sd["quantizer.codebook.weight"].double(), dim=1).contiguous()
        self._we = E
        return E

    @torch.no_grad()
    def get_semantic_tokens(self, batch, taps=None) -> torch.Tensor:
        """bicodec.py:167-172: batch["feat"] [B, T, input_channels] (the channel-last wav2vec2 features; a bare tensor is also taken)
        -> int64 [B, T], the layout detokenize takes.  taps (a dict) receives fp32 copies: "encoder" [B, T, out_channels] (the
        Encoder's output, channel-last) and "z_e" [B, T, codebook_dim] (the in_project output, before normalisation)."""
        E = self._prepare_semantic()
        feat = batch["feat"] if isinstance(batch, dict) else batch
        e, q = self.cfg.get("encoder", ENCODER_PARAMS), self.cfg["quantizer"]
        if not isinstance(feat, torch.Tensor) or feat.ndim != 3 or feat.shape[2] != e["input_channels"]:
            raise ValueError(f"feat must be [B, T, {e['input_channels']}]")
        if feat.device.type != "cuda":
            raise RuntimeError("unified_audio_b200.BiCodec runs on CUDA only (no CPU fallback): feat is on the CPU")
        B, T, Cin = feat.shape
        M, dim, inter, C = B * T, e["vocos_dim"], e["vocos_intermediate_dim"], e["out_channels"]
        x = feat.float().contiguous().reshape(M, Cin)
        # ---- Encoder (feat_encoder.py:79-90); scratch names under "enc_", apart from the prenet's
        x = self._backbone(E["enc"], x, B, T, dim, inter, tag="_e", cin=Cin, split=True, scope="enc_")
        for i, bw in enumerate(E["down"]):
            x = self._backbone(bw, x, B, T, dim, inter, tag=f"_d{i}", split=True, scope="enc_")
        xpl = self._planes("enc_x_p", (M, dim), True)
        ops.split_f16(x, xpl)
        z = self._buf("enc_z", (M, C))
        ops.gemm(xpl, E["proj"], C, a_batch=1, a_rows_per_batch=M, a_ld=dim, m_per_batch=M, bias=E["proj_b"], out_f32=rowmap(z, C, M, 0))
        # ---- FactorizedVectorQuantize.tokenize (factorized_vector_quantize.py:148-152,169-187)
        idx = torch.empty(B, T, dtype=torch.int64, device=feat.device)
        z_e = torch.empty(B, T, q["codebook_dim"], device=feat.device) if taps is not None else None
        ops.fvq_tokenize(z, M, C, E["w_in"], E["b_in"], E["cb_n"], q["codebook_size"], q["codebook_dim"], idx, z_e)
        if taps is not None:
            taps.update(encoder=z.clone().reshape(B, T, C), z_e=z_e)
        return idx

    @torch.no_grad()
    def tokenize(self, batch):
        """bicodec.py:151-165: batch {"feat": [B, T, input_channels], "ref_wav": [B, L]} -> (semantic_tokens int64 [B, T],
        global_tokens int32 [B, 1, token_num]), the reference's order.  Needs both token paths."""
        missing = [f for f in ("semantic_tokens", "global_tokens") if not getattr(self, f)]
        if missing:
            raise RuntimeError(f"BiCodec.tokenize needs both token paths: construct it with {', '.join(f + '=True' for f in missing)}")
        return self.get_semantic_tokens(batch), self.get_global_tokens(batch)

    # ------------------------------------------------------------------ forward (eval): postnet, x-vector, codebook usage
    def _postnet_params(self):
        return self.cfg.get("postnet", POSTNET_PARAMS)

    def _prepare_forward(self):
        if self._wf is not None:
            return self._wf
        dev = self._require_cuda()
        p, pre = self._postnet_params(), self.cfg["prenet"]
        if any(w % 64 for w in (p["input_channels"], p["vocos_dim"], p["vocos_intermediate_dim"], p["out_channels"])):
            raise ValueError("BiCodec postnet widths must be multiples of 64")
        if p["input_channels"] != pre["out_channels"]:
            raise ValueError("postnet input_channels must equal the prenet's out_channels (the postnet reads the prenet output)")
        keys = set(postnet_spec(self.cfg)) | set(xvector_spec(self.cfg))
        sd = {k: v.detach().double().cpu() for k, v in self.state_dict().items() if k in keys}
        sp = self.policy["prenet"]
        f32 = {k: v.float().to(dev) for k, v in sd.items() if k.startswith("postnet.")}
        # the postnet follows the prenet's precision group; SamplingBlock(1)'s 3 x folded into the downsample embeds, as the encoder's
        F = dict(lin_pre=Planes.from_f32(f32["postnet.linear_pre.weight"], sp), lin_pre_b=f32["postnet.linear_pre.bias"].contiguous(),
                 down=[_backbone_weights(f32, f"postnet.downsample.{i}.1.", 2, None, 3.0, sp) for i in range(len(p["sample_ratios"]))],
                 bb=_backbone_weights(f32, "postnet.vocos_backbone.", p["vocos_num_layers"], None, 1.0, sp),
                 lin=Planes.from_f32(f32["postnet.linear.weight"], sp), lin_b=f32["postnet.linear.bias"].contiguous())
        # x-vector: linear1 split into its x part (first 1536 input channels) and its context part [mean | std]; eval BatchNorm1d
        # folded into the final Linear in fp64: W' = W diag(g), b' = b + W (beta - mean g), g = gamma / sqrt(var + 1e-5)
        E = "speaker_encoder.speaker_encoder."
        w1 = sd[E + "pool.linear1.weight"][:, :, 0]
        g = sd[E + "bn.weight"] / torch.sqrt(sd[E + "bn.running_var"] + 1e-5)
        w = sd[E + "linear.weight"]

        def pl(t):
            return Planes.from_f32(t.float().contiguous().to(dev), True)

        F.update(w1x=pl(w1[:, :ECAPA_OUT]), w1c=pl(w1[:, ECAPA_OUT:]), b1=sd[E + "pool.linear1.bias"].float().to(dev),
                 w2=pl(sd[E + "pool.linear2.weight"][:, :, 0]), b2=sd[E + "pool.linear2.bias"].float().to(dev),
                 wx=pl(w * g[None, :]), bx=(sd[E + "linear.bias"] + w @ (sd[E + "bn.bias"] - sd[E + "bn.running_mean"] * g)).float().to(dev))
        self._wf = F
        return F

    def _postnet(self, pre, B, T):
        """postnet(x) (bicodec.py:135, feat_decoder.py:81-97 without a condition) on the prenet output [B*T, input_channels] ->
        fresh pred_feat [B, out_channels, T] (channel-first, the reference's layout)"""
        F, p = self._prepare_forward(), self._postnet_params()
        M, cin, dim, inter, cout = B * T, p["input_channels"], p["vocos_dim"], p["vocos_intermediate_dim"], p["out_channels"]
        sp = self.policy["prenet"]
        apl = self._planes("post_in_p", (M, cin), sp)
        ops.split_f16(pre, apl) if sp else ops.rows_to_planes(pre, 1, M, cin, apl, cin, M, 0)
        x = self._buf("post_x", (M, dim))
        ops.gemm(apl, F["lin_pre"], dim, a_batch=1, a_rows_per_batch=M, a_ld=cin, m_per_batch=M, bias=F["lin_pre_b"],
                 out_f32=rowmap(x, dim, M, 0))
        for i, bw in enumerate(F["down"]):
            x = self._backbone(bw, x, B, T, dim, inter, tag=f"_d{i}", scope="post_")
        x = self._backbone(F["bb"], x, B, T, dim, inter, tag="_m", scope="post_")
        xpl = self._planes("post_out_p", (M, dim), sp)
        ops.split_f16(x, xpl) if sp else ops.rows_to_planes(x, 1, M, dim, xpl, dim, M, 0)
        y = self._buf("post_y", (M, cout))
        ops.gemm(xpl, F["lin"], cout, a_batch=1, a_rows_per_batch=M, a_ld=dim, m_per_batch=M, bias=F["lin_b"], out_f32=rowmap(y, cout, M, 0))
        out = torch.empty(B, cout, T, device=pre.device)
        ops.ssl_compress(y, B, T, cout, 0.0, True, out)          # power 0: a plain channel-first copy
        return out

    def _xvector(self, lat32, latp, B, T):
        """ECAPA_TDNN's x-vector linear(bn(ASTP(latent))) (ecapa_tdnn.py:206-208, pooling_layers.py:134-144) from the fp32 latent
        [B*T, 1536] and its planes -> fresh [B, out_dim].  Every contraction is a 3-term split."""
        F = self._prepare_forward()
        M, C, H, n = B * T, ECAPA_OUT, ASTP_BOTTLENECK, self.cfg["speaker"]["out_dim"]
        # linear1 over [x; mean; std]: the context part once per clip (+ b1), the x part per frame, then tanh of their sum
        ctx, cpl = self._buf("xv_ctx", (B, 2 * C)), self._planes("xv_ctx_p", (B, 2 * C), True)
        ops.asp_context(lat32, B, T, C, ctx, cpl, 2 * C)
        crow = self._buf("xv_ctx_row", (B, H))
        ops.gemm(cpl, F["w1c"], H, a_batch=1, a_rows_per_batch=B, a_ld=2 * C, m_per_batch=B, bias=F["b1"], out_f32=rowmap(crow, H, B, 0))
        h = self._buf("xv_h", (M, H))
        ops.gemm(latp, F["w1x"], H, a_batch=1, a_rows_per_batch=M, a_ld=C, m_per_batch=M, out_f32=rowmap(h, H, M, 0))
        hpl = self._planes("xv_h_p", (M, H), True)
        ops.asp_tanh_planes(h, crow, B, T, H, hpl, H)
        logits = self._buf("xv_logits", (M, C))
        ops.gemm(hpl, F["w2"], C, a_batch=1, a_rows_per_batch=M, a_ld=H, m_per_batch=M, bias=F["b2"], out_f32=rowmap(logits, C, M, 0))
        # attentive [mean | std] -> BatchNorm-folded Linear
        pooled, ppl = self._buf("xv_pool", (B, 2 * C)), self._planes("xv_pool_p", (B, 2 * C), True)
        ops.asp_pool(lat32, logits, B, T, C, pooled, ppl, 2 * C)
        out = torch.empty(B, n, device=lat32.device)
        ops.gemm(ppl, F["wx"], n, a_batch=1, a_rows_per_batch=B, a_ld=2 * C, m_per_batch=B, bias=F["bx"], out_f32=rowmap(out, n, B, 0))
        return out

    def forward(self, batch=None):
        """BiCodec.forward in evaluation mode (bicodec.py:113-149): batch {"feat": [B, T, 1024], "ref_wav": [B, L] (or [B, 1, L]),
        "wav": any tensor with B rows}, on the device -> the reference's dict:
          recons [B, 1, T * hop], pred_feat [B, out_channels, T] (the postnet on the prenet output, before + d_vector), x_vector and
          d_vector [B, out_dim], perplexity and cluster_size (0-d fp32: the codebook's perplexity and number of codes used in the
          batch), vq_loss, audios = batch["wav"].unsqueeze(1), with_speaker_loss = False.
        vq_loss is NaN, as the reference computes it in eval mode: the mean of two empty tensors (factorized_vector_quantize.py:121-131).
        z_q and d_vector come from the gathers detokenize uses.  The reference's forward has z_q = out_project(z_e + (q - z_e)) and
        its d_vector from the quantised latents, which differ from detokenize's by rounding only; with the gathers, forward(batch)
        ["recons"] equals detokenize(*tokenize(batch)) bit for bit - the reference's own check (bicodec.py:235-257), made exact.
        Needs full=True; refused in train mode (the FVQ losses, the cluster_size EMA and straight-through gradients are not built)."""
        if not self.full:
            raise RuntimeError("unified_audio_b200.BiCodec.forward needs the whole module: construct it with BiCodec(..., full=True) "
                               "and load a checkpoint that carries postnet.* and the x-vector branch")
        if self.training:
            raise RuntimeError("unified_audio_b200.BiCodec.forward runs in evaluation mode only: call .eval() (the FVQ losses, the "
                               "cluster_size EMA and straight-through gradients are not built)")
        if not isinstance(batch, dict) or any(not isinstance(batch.get(k), torch.Tensor) for k in ("feat", "ref_wav", "wav")):
            raise ValueError('BiCodec.forward takes a dict with tensors "feat", "ref_wav" and "wav"')
        feat, wav = batch["feat"], batch["wav"]
        if wav.device.type != "cuda":
            raise RuntimeError("unified_audio_b200.BiCodec runs on CUDA only (no CPU fallback): wav is on the CPU")
        ref = self._check_wav(batch["ref_wav"])
        if wav.ndim < 1 or feat.ndim != 3 or not feat.shape[0] == ref.shape[0] == wav.shape[0]:
            raise ValueError("feat [B, T, C], ref_wav and wav must have the same batch size B")
        with torch.no_grad():
            sem = self.get_semantic_tokens(feat)
            glob, lat32, latp, Tm = self._global_tokens(ref, keep_latent=True)
            B, T = sem.shape
            x_vector = self._xvector(lat32, latp, B, Tm)
            K = self.cfg["quantizer"]["codebook_size"]
            perplexity, active = torch.empty((), device=wav.device), torch.empty((), device=wav.device)
            ops.fvq_usage(sem.reshape(-1), K, self._buf("fvq_counts", (K,), torch.int32), perplexity, active)
            pre, dvec = self._prenet(sem, glob)
            pred_feat = self._postnet(pre, B, T)
            recons = self._wave(pre, dvec, B, T)
            return {"vq_loss": torch.full((), float("nan"), device=wav.device), "perplexity": perplexity, "cluster_size": active,
                    "recons": recons, "pred_feat": pred_feat, "x_vector": x_vector, "d_vector": dvec.clone(),
                    "audios": wav.unsqueeze(1), "with_speaker_loss": False}
