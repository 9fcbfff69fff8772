"""Codec.forward and the semantic decoder without a GPU: the oracle's semantic decoder against the reference's own
`semantic_module.Decoder` (tests/golden/codec_forward_small.npz, oracle/make_golden_codec_forward.py), and the faces' host logic
with and without `semantic_decoder=True` (parameters under the reference's names, strict loads, refused train-mode forward)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import semantic_decoder as osd
from oracle.make_golden_codec_forward import CONFIGS, FORWARD, FRAMES, forward_case

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", list(CONFIGS))
def test_oracle_semantic_decoder_matches_reference_decoder(name):
    z = np.load(os.path.join(GOLD, "codec_forward_small.npz"))
    cfg = CONFIGS[name]
    sd = osd.make_state_dict(cfg, seed=3)
    for N in FRAMES:
        x = torch.from_numpy(z[f"{name}/z{N}"])
        for dt, tag, tol in ((torch.float32, "f32", 1e-6), (torch.float64, "f64", 1e-12)):
            want = torch.from_numpy(z[f"{name}/pred{N}_{tag}"])
            got = osd.semantic_decoder_forward({k: v.to(dt) for k, v in sd.items()}, cfg, x.to(dt))
            assert got.dtype == dt and got.shape == want.shape == (2, cfg["output_channels"], N * int(np.prod(cfg["strides"])))
            assert float((got - want).abs().max() / want.abs().max()) < tol, (name, N, tag)


def test_pinning_report_covers_every_config():
    rep = json.load(open(os.path.join(GOLD, "codec_forward_pinning_report.json")))
    assert set(rep["configs"]) == set(CONFIGS) and 1 in rep["frames"] and any(n % 2 for n in rep["frames"])
    dec = {k: r for k, r in rep["pinned"].items() if not k.startswith("forward/")}
    assert all(r["max_rel_err_oracle_vs_reference"] < 1e-6 for r in dec.values())
    fwd = {k[len("forward/"):]: r for k, r in rep["pinned"].items() if k.startswith("forward/")}
    assert set(fwd) == set(FORWARD) and all(r["commit_loss"] == 0.0 and r["pred_feat_rel"] < 1e-6 for r in fwd.values())
    assert fwd["h15"]["token_lengths_equal"] and fwd["h15"]["token_length_max"] > 1


# recon of H-Codec-1.5: the oracle's adaptive chain reproduces the reference's decode to ~1e-6 (h15_pinning_report.json), so the
# bound is 2e-6 there; everything else is within 1e-6 (bit-equal when this fixture was made)
RECON_TOL = {"h2": 1e-6, "h1": 1e-6, "h15": 2e-6}


@pytest.mark.parametrize("name", list(FORWARD))
def test_oracle_forward_matches_reference_forward(name):
    """oracle/semantic_decoder.py's forwards against the reference's own Codec.forward (eval mode) stored in the fixture"""
    z = np.load(os.path.join(GOLD, "codec_forward_small.npz"))
    cfg, sd, x, feat = forward_case(name)
    if name == "h15":
        out = osd.h15_forward(sd, cfg, x, feat)
        assert torch.equal(out["token_lengths"], torch.from_numpy(z[f"fwd/{name}/token_lengths"]))
        assert out["token_lengths"].dtype == torch.int64 and int(out["token_lengths"].max()) > 1
    else:
        out = dict(zip(("recon", "pred_feat", "commit_loss"), (osd.h2_forward if name == "h2" else osd.h1_forward)(sd, cfg, x, feat)))
    rel = lambda a, k: float((a - torch.from_numpy(z[f"fwd/{name}/{k}"])).abs().max() / np.abs(z[f"fwd/{name}/{k}"]).max())
    assert out["recon"].shape == z[f"fwd/{name}/recon"].shape and rel(out["recon"], "recon") < RECON_TOL[name]
    assert out["pred_feat"].shape == z[f"fwd/{name}/pred_feat"].shape and rel(out["pred_feat"], "pred_feat") < 1e-6
    assert out["commit_loss"].dim() == 0 and float(out["commit_loss"]) == 0.0 and float(z[f"fwd/{name}/commit_loss"]) == 0.0


# ----------------------------------------------------------------------------- faces
def _h2(flag):
    from oracle import weights
    from unified_audio_b200.codec import Codec
    meta = json.loads(str(np.load(os.path.join(GOLD, "h2_small.npz"))["meta"]))
    cfg = meta["cfg"]
    m = Codec(cfg["encoder_config"], cfg["decoder_config"], cfg["quantizer_config"], cfg["semantic_encoder_config"],
              cfg["semantic_decoder_config"], semantic_decoder=flag)
    ref = json.load(open(os.path.join(GOLD, "h2_keys_small.json")))
    sd = dict(weights.make_h2_state_dict(cfg, 1))
    return m, ref, sd, cfg["semantic_decoder_config"]


def _h1(flag):
    from oracle import hcodec1
    from unified_audio_b200.codec_h1 import CodecH1, semantic_decoder_config
    m = CodecH1({}, {}, {}, semantic_decoder=flag)
    ref = json.load(open(os.path.join(GOLD, "h1_keys.json")))
    return m, ref, dict(hcodec1.make_state_dict(hcodec1.H1, 1)), semantic_decoder_config(hcodec1.H1)


def _h15(flag):
    from oracle import hcodec15
    from unified_audio_b200.codec_h15 import CodecH15
    from unified_audio_b200.codec_h1 import semantic_decoder_config
    m = CodecH15(semantic_decoder=flag)
    ref = {k: list(v[0]) for k, v in hcodec15.param_specs(hcodec15.H15).items()}
    ref.update({k: list(v[0]) for k, v in osd.param_specs(osd.h1_config(hcodec15.H15)).items()})
    return m, ref, None, semantic_decoder_config(hcodec15.H15)


FACES = {"Codec": _h2, "CodecH1": _h1, "CodecH15": _h15}


@pytest.mark.parametrize("face", list(FACES))
def test_flag_off_keeps_state_dict_and_refuses_forward(face):
    m, ref, _, _ = FACES[face](False)
    mine = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert mine == {k: v for k, v in ref.items() if not k.startswith("semantic_decoder.")}
    with pytest.raises(RuntimeError, match="semantic_decoder=True"):
        m(torch.zeros(1, 1, 640), torch.zeros(1, 768, 2))
    with pytest.raises(RuntimeError, match="semantic_decoder=True"):
        m.semantic_decode(torch.zeros(1, 4, 1, dtype=torch.long))


@pytest.mark.parametrize("face", list(FACES))
def test_flag_on_holds_reference_keys(face):
    m, ref, _, dcfg = FACES[face](True)
    mine = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert mine == ref
    assert {k: tuple(v) for k, v in mine.items() if k.startswith("semantic_decoder.")} == \
        {k: tuple(v[0]) for k, v in osd.param_specs(dcfg).items()}


def _h15_kwargs(semantic_decoder):
    """the config blocks CodecH15 takes (conf/config_adaptive_v3.yaml's fields), one layer per mimi stack"""
    agg = dict(dim=512, in_out_dim=512, num_heads=8, num_layers=1, dim_feedforward=2048, causal=False)
    dec = dict(decoder=dict(input_channels=1024, dim=1024, intermediate_dim=2304))
    if semantic_decoder is not None:
        dec["semantic_decoder"] = semantic_decoder
    return (dict(encoder=dict(n_filters=32, dimension=512, ratios=[2, 4, 5, 8]),
                 semantic_encoder=dict(input_channels=1024, encode_channels=1024, out_channels=512, strides=[2, 1])),
            dec, dict(quantizer=dict(dim=512, codebook_size=1024, num_quantizers=4)),
            dict(use_similarity_alignment=True, similarity_threshold=0.7, max_tokens_per_group=8, manual_threshold=0.6,
                 use_query_token_aggregator=True, use_bottleneck_transformer=True,
                 aggregators=dict(semantic_aggregator=dict(agg), acoustic_aggregator=dict(agg)),
                 transformer_kwargs=dict(d_model=1024, num_heads=8, num_layers=1, causal=False, gating="none", norm="layer_norm",
                                         positional_embedding="rope", dim_feedforward=2048, input_dimension=1024,
                                         output_dimensions=[1024])))


def test_h15_constructor_takes_sizes_from_decoder_kwargs():
    """CodecH15(encoder_kwargs, decoder_kwargs, ...) sizes its semantic decoder from decoder_kwargs["semantic_decoder"]
    (codec_adaptive.py:44), here deliberately not the sizes the flat config would give"""
    from unified_audio_b200.codec_h15 import CodecH15
    sem = dict(code_dim=512, output_channels=1024, decode_channels=256, channel_ratios=[1, 1], strides=[2, 1])
    m = CodecH15(*_h15_kwargs(sem), semantic_decoder=True)
    assert m.sem_dec_cfg == sem
    got = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith("semantic_decoder.")}
    assert got == {k: tuple(v[0]) for k, v in osd.param_specs(sem).items()}
    assert m.state_dict()["semantic_decoder.conv_blocks.0.conv.deconv.weight"].shape == (256, 256, 4)
    plain = CodecH15(*_h15_kwargs(sem))
    assert not any(k.startswith("semantic_decoder.") for k in plain.state_dict())


def test_semantic_decoder_spec_refuses_unbuilt_configs():
    from unified_audio_b200 import spec
    base = dict(code_dim=8, output_channels=8, decode_channels=8)
    for bad in (dict(strides=[2, 1], channel_ratios=[1]), dict(strides=[2], channel_ratios=[1], kernel_size=5),
                dict(strides=[2], channel_ratios=[1], block_dilations=(1, 3)), dict(strides=[0], channel_ratios=[1])):
        with pytest.raises(ValueError):
            spec.semantic_decoder_spec(**base, **bad)


def _h15_shallow(flag):
    from oracle import hcodec15
    from unified_audio_b200.codec_h15 import CodecH15
    c = hcodec15.h15_shallow()
    m = CodecH15(_cfg={k: v for k, v in c.items() if k != "layer_scale"}, semantic_decoder=flag)
    return m, None, dict(hcodec15.make_state_dict(c, 1)), osd.h1_config(c)


STRICT = {"Codec": _h2, "CodecH1": _h1, "CodecH15": _h15_shallow}


@pytest.mark.parametrize("face", list(STRICT))
def test_flag_on_strict_loads(face):
    m, _, sd, dcfg = STRICT[face](True)
    full = dict(sd, **osd.make_state_dict(dcfg, 2))
    m.load_state_dict(full, strict=True)
    got = m.state_dict()
    assert all(torch.equal(got[k], full[k].to(got[k].dtype)) for k in full)
    with pytest.raises(RuntimeError):                 # a checkpoint without the decoder no longer loads strictly
        m.load_state_dict(sd, strict=True)
    m.train()
    with pytest.raises(RuntimeError, match="evaluation mode"):
        m(torch.zeros(1, 1, 640), torch.zeros(1, 768, 2))
    m.eval()
