"""Parameter / buffer layout of H-Codec-2.0, restated from the reference modules so that
`Codec.state_dict()` keys and shapes equal the reference's
(QuarkAudio-HCodec/HCodec-2.0/vq/codec_encoder.py:30-58, codec_decoder.py:30-59,
semantic_module.py:157-194, encoder_modules/transformer.py:106-119,218-226,337-366).
tests/test_host.py checks it against the reference's own key list (tests/golden/h2_keys_*.json)."""
from __future__ import annotations

from collections import OrderedDict


def _transformer(prefix, dim, inter, layers, out):
    for i in range(layers):
        p = f"{prefix}layers.{i}."
        out[p + "self_attn.rnn.weight_ih_l0"] = (4 * dim, dim)
        out[p + "self_attn.rnn.weight_hh_l0"] = (4 * dim, dim)
        out[p + "self_attn.rnn.bias_ih_l0"] = (4 * dim,)
        out[p + "self_attn.rnn.bias_hh_l0"] = (4 * dim,)
        for n in "qkv":
            out[p + f"self_attn.{n}_proj.weight"] = (dim, dim)
            out[p + f"self_attn.{n}_proj.bias"] = (dim,)
        out[p + "self_attn.o_proj.weight"] = (dim, dim)
        out[p + "mlp.w1.weight"] = (inter, dim)
        out[p + "mlp.w2.weight"] = (dim, inter)
        out[p + "mlp.w3.weight"] = (inter, dim)
        out[p + "input_layernorm.weight"] = (dim,)
        out[p + "post_attention_layernorm.weight"] = (dim,)


def _convnext(prefix, dim, inter, n, out):
    for i in range(n):
        p = f"{prefix}{i}."
        out[p + "gamma"] = (dim,)
        out[p + "dwconv.conv.weight"] = (dim, 1, 7)
        out[p + "dwconv.conv.bias"] = (dim,)
        out[p + "norm.weight"] = (dim,)
        out[p + "norm.bias"] = (dim,)
        out[p + "pwconv1.linear.weight"] = (inter, dim)
        out[p + "pwconv1.linear.bias"] = (inter,)
        out[p + "pwconv2.linear.weight"] = (dim, inter)
        out[p + "pwconv2.linear.bias"] = (dim,)


def encoder_spec(dim, intermediate_dim, dimension, n_fft=1920, hop_length=960, convnext_layers=12,
                 transformer_layers=2, target_frame_rate=6.25, causal=False):
    assert not causal, "only the shipped non-causal configuration is implemented"
    out = OrderedDict()
    nf = n_fft // 2 + 1
    out["stft.window"] = (n_fft,)
    out["embed.conv.weight"] = (dim, 2 * nf, 3)
    out["embed.conv.bias"] = (dim,)
    out["norm.weight"] = (dim,)
    out["norm.bias"] = (dim,)
    _convnext("prior_net.", dim, intermediate_dim, convnext_layers, out)
    _transformer("post_net.1.", dim, min(dim * 4, 4096), transformer_layers, out)
    out["final_layer_norm.weight"] = (dim,)
    out["final_layer_norm.bias"] = (dim,)
    stride = int(50 / target_frame_rate)
    out["out.conv.weight"] = (dimension, dim, 2 * stride + 1)
    out["out.conv.bias"] = (dimension,)
    return out


def decoder_spec(input_channels, dim, intermediate_dim, convnext_layers=12, n_fft=1920, hop_length=960,
                 transformer_layers=2, target_frame_rate=6.25, causal=False):
    assert not causal, "only the shipped non-causal configuration is implemented"
    out = OrderedDict()
    f = int(50 / target_frame_rate)
    out["embed.conv.weight"] = (dim, input_channels, f + 1)
    out["embed.conv.bias"] = (dim,)
    out["norm.weight"] = (dim,)
    out["norm.bias"] = (dim,)
    _convnext("post_net.", dim, intermediate_dim, convnext_layers, out)
    out["final_layer_norm.weight"] = (dim,)
    out["final_layer_norm.bias"] = (dim,)
    for i in (0, 1):
        _resnet(f"prior_net.{i}.", dim, out)
    _transformer("prior_net.3.", dim, min(dim * 4, 4096), transformer_layers, out)
    for i in (5, 6):
        _resnet(f"prior_net.{i}.", dim, out)
    out["prior_net.7.weight"] = (dim,)
    out["prior_net.7.bias"] = (dim,)
    out["head.out.weight"] = (n_fft + 2, dim)
    out["head.out.bias"] = (n_fft + 2,)
    out["head.istft.window"] = (n_fft,)
    return out


def _resnet(p, dim, out):
    for j in (1, 2):
        out[p + f"norm{j}.weight"] = (dim,)
        out[p + f"norm{j}.bias"] = (dim,)
        out[p + f"conv{j}.conv.weight"] = (dim, dim, 3)
        out[p + f"conv{j}.conv.bias"] = (dim,)


def semantic_encoder_spec(input_channels, encode_channels, out_channels, channel_ratios=(1, 1), strides=(1, 1),
                          kernel_size=3, bias=True, block_dilations=(1, 1), unit_kernel_size=3):
    assert kernel_size == 3 and unit_kernel_size == 3 and tuple(block_dilations) == (1, 1) and bias
    out = OrderedDict()
    out["conv.conv.weight"] = (encode_channels, input_channels, 3)
    cin = encode_channels
    for i, st in enumerate(strides):
        cout = int(encode_channels * channel_ratios[i])
        p = f"conv_blocks.{i}."
        for u in (0, 1):
            out[p + f"res_units.{u}.conv1.conv.weight"] = (cin, cin, 3)
            out[p + f"res_units.{u}.conv2.weight"] = (cin, cin, 1)
        k = 3 if st == 1 else 2 * st
        out[p + "conv.conv.weight"] = (cout, cin, k)
        out[p + "conv.conv.bias"] = (cout,)
        cin = cout
    out["conv2.conv.weight"] = (out_channels, cin, 3)
    return out


def semantic_decoder_spec(code_dim, output_channels, decode_channels, channel_ratios=(1, 1), strides=(1, 1), kernel_size=3,
                          bias=True, block_dilations=(1, 1), unit_kernel_size=3):
    """vq/semantic_module.py:252-292 (Decoder), :205-249 (DecoderBlock: k3 conv at stride 1, ConvTranspose1d(2s, s) otherwise)."""
    if not (kernel_size == 3 and unit_kernel_size == 3 and tuple(block_dilations) == (1, 1) and bias):
        raise ValueError("semantic decoder: only kernel_size 3, unit_kernel_size 3, block_dilations (1, 1) and bias=True (the shipped "
                         "configs) are built")
    if len(channel_ratios) != len(strides) or any(int(s) < 1 for s in strides):
        raise ValueError(f"semantic decoder: one channel ratio per stride and strides >= 1, got {list(channel_ratios)} / {list(strides)}")
    out = OrderedDict()
    out["conv1.conv.weight"] = (int(decode_channels * channel_ratios[0]), code_dim, 3)
    cout = decode_channels
    for i, st in enumerate(strides):
        cin = int(decode_channels * channel_ratios[i])
        cout = int(decode_channels * channel_ratios[i + 1]) if i + 1 < len(strides) else decode_channels
        p = f"conv_blocks.{i}."
        if st == 1:
            out[p + "conv.conv.weight"] = (cout, cin, 3)
            out[p + "conv.conv.bias"] = (cout,)
        else:
            out[p + "conv.deconv.weight"] = (cin, cout, 2 * st)
            out[p + "conv.deconv.bias"] = (cout,)
        for u in (0, 1):
            out[p + f"res_units.{u}.conv1.conv.weight"] = (cout, cout, 3)
            out[p + f"res_units.{u}.conv2.weight"] = (cout, cout, 1)
    out["conv2.conv.weight"] = (output_channels, cout, 3)
    return out


BUFFERS = ("stft.window", "head.istft.window")
