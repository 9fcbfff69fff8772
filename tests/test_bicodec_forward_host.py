"""BiCodec.forward on the host: the oracle reproduces the outputs of the reference's own BiCodec.forward
(tests/golden/bicodec_forward_small.npz, oracle/make_golden_bicodec_forward.py), the keys `full=True` adds are the reference's, a full
face loads a reference checkpoint strictly and refuses one that lacks them, and forward refuses what it does not build."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")
E = "speaker_encoder.speaker_encoder."


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


def test_oracle_reproduces_reference_forward():
    from oracle import bicodec_forward as of
    from oracle.make_golden_bicodec_forward import small_config, small_state_dict
    z = np.load(os.path.join(GOLD, "bicodec_forward_small.npz"))
    cfg = small_config()
    sd64 = {k: v.double() for k, v in small_state_dict(cfg).items()}
    batch = {k: torch.from_numpy(z[k]).double() for k in ("feat", "ref_wav", "wav")}
    taps = {}
    out = of.forward(sd64, cfg, batch, taps)
    assert torch.equal(taps["semantic"], torch.from_numpy(z["semantic"]))
    assert torch.equal(taps["global_tokens"], torch.from_numpy(z["global_tokens"]))
    for k in ("recons", "pred_feat", "x_vector", "d_vector", "perplexity"):
        assert out[k].shape == z[k].shape and rel(out[k], z[k]) < 1e-5, k
    assert out["cluster_size"] == float(z["cluster_size"]) and 1 < out["cluster_size"] < z["semantic"].size
    assert np.isnan(z["vq_loss"]) and z["vq_loss"].shape == () and z["vq_loss"].dtype == np.float32
    assert torch.equal(out["audios"], batch["wav"].unsqueeze(1)) and out["with_speaker_loss"] is False


def test_oracle_pooling_edges():
    from oracle import bicodec_forward as of
    x = torch.tensor([[[1.0, 2.0, 4.0], [3.0, 3.0, 3.0]]], dtype=torch.float64)
    ctx = of.astp_context(x)
    assert torch.allclose(ctx, torch.tensor([[7 / 3, 3.0, (x[0, 0].var() + 1e-7).sqrt(), 1e-7 ** 0.5]], dtype=torch.float64))
    one_hot = torch.tensor([[[0.0, -1e4, -1e4], [0.0, 0.0, 0.0]]], dtype=torch.float64)
    pooled = of.astp_pool(x, one_hot)
    assert pooled[0, 0] == 1.0 and pooled[0, 2] == 1e-7 ** 0.5 and pooled[0, 1] == 3.0 and pooled[0, 3] == 1e-7 ** 0.5
    p, n = of.fvq_usage(torch.tensor([[5, 5, 5, 5]]), 8)
    assert n == 1 and abs(float(p) - 1.0) < 1e-9
    p, n = of.fvq_usage(torch.tensor([[0, 1, 2, 7]]), 8)
    assert n == 4 and abs(float(p) - 4.0) < 1e-6


def test_forward_keys_match_reference():
    from oracle import bicodec_forward as of
    from unified_audio_b200.bicodec import BICODEC_CONFIG, POSTNET_PARAMS, BiCodec, postnet_spec, xvector_spec
    assert POSTNET_PARAMS == of.POSTNET_PARAMS
    post = json.load(open(os.path.join(GOLD, "bicodec_postnet_keys.json")))
    gkeys = json.load(open(os.path.join(GOLD, "bicodec_global_keys.json")))
    xkeys = {k: v for k, v in gkeys.items() if k.startswith((E + "pool.", E + "bn.", E + "linear.")) and not k.endswith("num_batches_tracked")}
    assert len(xkeys) == 10
    assert {k: list(v) for k, v in postnet_spec(BICODEC_CONFIG).items()} == post
    assert {k: list(v) for k, v in xvector_spec(BICODEC_CONFIG).items()} == xkeys
    assert {k: list(v[0]) for k, v in of.forward_param_specs(of.BICODEC_FORWARD_FULL).items()} == {**post, **xkeys}
    full = set(BiCodec(full=True).state_dict())
    assert full == set(BiCodec(global_tokens=True, semantic_tokens=True).state_dict()) | set(post) | set(xkeys)


def full_checkpoint():
    """every key of a reference BiCodec checkpoint at the shipped configuration, postnet and x-vector branch included"""
    from oracle import bicodec as ob
    from oracle import bicodec_forward as of
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    sd = dict(ob.make_state_dict(ob.BICODEC_FULL, 1))
    sd.update(og.make_speaker_state_dict(og.BICODEC_GLOBAL_FULL, 1))
    sd.update(osm.make_semantic_state_dict(osm.BICODEC_SEMANTIC_FULL, 1))
    sd.update(of.make_forward_state_dict(of.BICODEC_FORWARD_FULL, 1))
    for k, shape in json.load(open(os.path.join(GOLD, "bicodec_global_keys.json"))).items():
        assert k in sd or k.endswith("num_batches_tracked"), k
        sd.setdefault(k, torch.zeros(shape, dtype=torch.int64))
    sd["quantizer.cluster_size"] = torch.zeros(8192)
    sd["mel_transformer.spectrogram.window"] = torch.zeros(640)
    return sd


def test_full_face_loads_reference_checkpoint_strictly():
    from unified_audio_b200.bicodec import BiCodec
    sd = full_checkpoint()
    m = BiCodec(full=True)
    m.load_state_dict(sd, strict=True)
    held = m.state_dict()
    for k in ("postnet.vocos_backbone.convnext.5.pwconv2.weight", E + "pool.linear1.weight", E + "bn.running_var", E + "linear.bias"):
        assert torch.equal(held[k], sd[k]), k
    assert not any(k.startswith("mel_transformer.") or k == "quantizer.cluster_size" or k.endswith("num_batches_tracked") for k in held)
    assert m.global_tokens and m.semantic_tokens
    for drop in ("postnet.linear.bias", E + "pool.linear1.weight"):
        with pytest.raises(RuntimeError, match=drop.replace(".", r"\.")):
            BiCodec(full=True).load_state_dict({k: v for k, v in sd.items() if k != drop}, strict=True)
    # faces without the flag still accept the whole checkpoint and hold none of it
    for flags in (dict(), dict(global_tokens=True, semantic_tokens=True)):
        f = BiCodec(**flags)
        f.load_state_dict(sd, strict=True)
        assert not any(k.startswith(("postnet.", E + "pool.", E + "bn.", E + "linear.")) for k in f.state_dict())


def test_full_flag_and_postnet_config_are_checked():
    from unified_audio_b200.bicodec import BICODEC_CONFIG, POSTNET_PARAMS, BiCodec
    for flags in (dict(global_tokens=False), dict(semantic_tokens=False), dict(global_tokens=False, semantic_tokens=False)):
        with pytest.raises(ValueError, match="full=True"):
            BiCodec(full=True, **flags)
    BiCodec(full=True, global_tokens=True, semantic_tokens=True)
    for bad in (dict(use_tanh_at_final=True), dict(sample_ratios=[2, 2]), dict(condition_dim=1024)):
        cfg = dict(BICODEC_CONFIG, postnet=dict(POSTNET_PARAMS, **bad))
        with pytest.raises(NotImplementedError):
            BiCodec(cfg, full=True)
        BiCodec(cfg)                    # without the flag the section is unused
    small = dict(BICODEC_CONFIG, postnet=dict(POSTNET_PARAMS, vocos_num_layers=2))
    assert not any(".convnext.2." in k for k in BiCodec(small, full=True).state_dict() if k.startswith("postnet.vocos_backbone."))


def test_forward_refusals():
    from unified_audio_b200.bicodec import BiCodec
    batch = {"feat": torch.zeros(1, 5, 1024), "ref_wav": torch.zeros(1, 4000), "wav": torch.zeros(1, 1600)}
    for m in (BiCodec(), BiCodec(global_tokens=True, semantic_tokens=True)):
        with pytest.raises(RuntimeError, match="full=True"):
            m.forward()
        with pytest.raises(RuntimeError, match="full=True"):
            m(batch)
    full = BiCodec(full=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        full(batch)
    full.train()
    with pytest.raises(RuntimeError, match="evaluation mode"):
        full(batch)
    full.eval()
    for bad in ({k: v for k, v in batch.items() if k != "wav"}, dict(batch, feat=None), [batch]):
        with pytest.raises(ValueError):
            full(bad)
