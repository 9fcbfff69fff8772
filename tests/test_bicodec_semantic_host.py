"""BiCodec semantic tokens on the host: the oracle reproduces the outputs of the reference's own classes
(tests/golden/bicodec_semantic_small.npz, oracle/make_golden_bicodec_semantic.py), the product's state-dict layout of the path is the
reference's, every combination of the two token flags loads a reference checkpoint strictly, and there is no CPU path."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


def test_oracle_reproduces_reference_semantic_tokens():
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    from oracle import wav2vec2 as ow
    from oracle.make_golden_bicodec_semantic import e2e_wav2vec2_config, small_config, small_state_dict
    z = np.load(os.path.join(GOLD, "bicodec_semantic_small.npz"))
    meta = json.loads(str(z["meta"]))
    cfg = small_config()
    sd64 = {k: v.double() for k, v in small_state_dict(cfg, meta["seed"]).items()}
    taps = {}
    tokens = osm.get_semantic_tokens(sd64, cfg, torch.from_numpy(z["feat"]).double(), taps)
    assert tokens.dtype == torch.int64 and torch.equal(tokens, torch.from_numpy(z["tokens"]))
    assert rel(taps["encoder"], z["encoder"]) < 1e-5 and rel(taps["z_e"], z["z_e"]) < 1e-5
    # the fixture decides every token away from a tie and uses many codes
    assert float(osm.fvq_margins(sd64, taps["encoder"]).min()) >= 1e-3
    assert len(set(tokens.reshape(-1).tolist())) >= 64
    assert torch.equal(og.get_global_tokens(sd64, cfg, torch.from_numpy(z["ref_wav"]).double()), torch.from_numpy(z["global_tokens"]))
    # end to end: wav -> wav2vec2 features -> semantic tokens, wav -> reference clip -> global tokens
    wav = torch.from_numpy(z["e2e_wav"])
    feat = ow.extract_wav2vec2_features(ow.make_state_dict(e2e_wav2vec2_config(), meta["w2v_seed"]), e2e_wav2vec2_config(), wav)
    assert torch.equal(osm.get_semantic_tokens(sd64, cfg, feat.double()), torch.from_numpy(z["e2e_semantic"]))
    clip = og.get_ref_clip(wav, meta["ref_segment_length"]).double()
    assert torch.equal(og.get_global_tokens(sd64, cfg, clip), torch.from_numpy(z["e2e_global"]))


def test_fvq_tokenize_picks_the_lowest_index_on_ties():
    from oracle import bicodec_semantic as osm
    cb = torch.tensor([[1.0, 0.0], [0.0, 1.0], [2.0, 0.0], [0.0, 0.0]], dtype=torch.float64)
    sd = {"quantizer.codebook.weight": cb, "quantizer.in_project.weight_v": torch.eye(2, dtype=torch.float64)[:, :, None],
          "quantizer.in_project.weight_g": torch.ones(2, 1, 1, dtype=torch.float64),
          "quantizer.in_project.bias": torch.zeros(2, dtype=torch.float64)}
    z = torch.tensor([[[3.0, 0.0], [0.0, 0.5], [0.0, 0.0]]], dtype=torch.float64)
    tok, _ = osm.fvq_tokenize(sd, z)
    assert tok.tolist() == [[0, 1, 3]]             # rows 0 and 2 of the codebook normalise to the same code; a zero row wins at 0
    assert float(osm.fvq_margins(sd, z)[0, 0]) == 0.0


def test_semantic_spec_matches_reference_keys():
    from oracle import bicodec_semantic as osm
    from unified_audio_b200.bicodec import BICODEC_CONFIG, ENCODER_PARAMS, BiCodec, bicodec_spec, encoder_spec
    keys = json.load(open(os.path.join(GOLD, "bicodec_semantic_keys.json")))
    assert ENCODER_PARAMS == osm.ENCODER_PARAMS
    assert {k: list(v) for k, v in encoder_spec(BICODEC_CONFIG).items()} == keys
    assert {k: list(v[0]) for k, v in osm.semantic_param_specs(osm.BICODEC_SEMANTIC_FULL).items()} == keys
    assert set(BiCodec(semantic_tokens=True).state_dict()) == set(bicodec_spec(BICODEC_CONFIG)) | set(keys)


def full_checkpoint():
    """every key of a reference BiCodec checkpoint at the shipped configuration (postnet and the x-vector branch as stand-ins)"""
    from oracle import bicodec as ob
    from oracle import bicodec_global as og
    from oracle import bicodec_semantic as osm
    sd = dict(ob.make_state_dict(ob.BICODEC_FULL, 1))
    sd.update(og.make_speaker_state_dict(og.BICODEC_GLOBAL_FULL, 1))
    sd.update(osm.make_semantic_state_dict(osm.BICODEC_SEMANTIC_FULL, 1))
    gkeys = json.load(open(os.path.join(GOLD, "bicodec_global_keys.json")))
    for k, shape in gkeys.items():
        sd.setdefault(k, torch.zeros(shape))
    sd["quantizer.cluster_size"] = torch.zeros(8192)
    sd["postnet.linear_pre.weight"] = torch.zeros(2, 2)
    sd["mel_transformer.spectrogram.window"] = torch.zeros(640)
    return sd


@pytest.mark.parametrize("global_tokens,semantic_tokens", [(False, False), (True, False), (False, True), (True, True)])
def test_every_flag_combination_loads_a_reference_checkpoint_strictly(global_tokens, semantic_tokens):
    from unified_audio_b200.bicodec import BiCodec
    sd = full_checkpoint()
    m = BiCodec(global_tokens=global_tokens, semantic_tokens=semantic_tokens)
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.state_dict()["quantizer.codebook.weight"], sd["quantizer.codebook.weight"])
    held = set(m.state_dict())
    assert any(k.startswith("encoder.") for k in held) == semantic_tokens
    assert ("quantizer.in_project.weight_v" in held) == semantic_tokens
    assert any(k.startswith("speaker_encoder.perceiver_sampler.") for k in held) == global_tokens
    assert not any(k.startswith(("postnet.", "mel_transformer.")) or k == "quantizer.cluster_size" for k in held)
    if semantic_tokens:
        missing = dict(sd)
        del missing["quantizer.in_project.weight_g"]
        with pytest.raises(RuntimeError):
            BiCodec(global_tokens=global_tokens, semantic_tokens=True).load_state_dict(missing, strict=True)


def test_encoder_config_is_checked():
    from unified_audio_b200.bicodec import BICODEC_CONFIG, ENCODER_PARAMS, BiCodec
    with pytest.raises(NotImplementedError):
        BiCodec(dict(BICODEC_CONFIG, encoder=dict(ENCODER_PARAMS, sample_ratios=[2, 2])), semantic_tokens=True)
    BiCodec(dict(BICODEC_CONFIG, encoder=dict(ENCODER_PARAMS, sample_ratios=[2, 2])))       # without the flag the section is unused


def test_semantic_path_has_no_cpu_path_and_tokenize_names_what_is_missing():
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.unise import BiCodecTokenizer
    feat = torch.zeros(1, 5, 1024)
    with pytest.raises(RuntimeError, match="semantic_tokens=True"):
        BiCodec().get_semantic_tokens({"feat": feat})
    with pytest.raises(RuntimeError, match="semantic_tokens=True"):
        BiCodec(global_tokens=True).tokenize({"feat": feat, "ref_wav": torch.zeros(1, 4000)})
    with pytest.raises(RuntimeError, match="global_tokens=True"):
        BiCodec(semantic_tokens=True).tokenize({"feat": feat, "ref_wav": torch.zeros(1, 4000)})
    both = BiCodec(global_tokens=True, semantic_tokens=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        both.get_semantic_tokens({"feat": feat})
    with pytest.raises(RuntimeError, match="CUDA"):
        both.get_semantic_tokens(feat)
    with pytest.raises(RuntimeError, match="CUDA"):
        both.tokenize({"feat": feat, "ref_wav": torch.zeros(1, 4000)})
    with pytest.raises(RuntimeError):
        both.forward()
    # the tokenizer refuses before it looks at the device, and names what it lacks
    wav = torch.zeros(1, 4000)
    with pytest.raises(NotImplementedError, match="feature_extractor"):
        BiCodecTokenizer(both).tokenize(wav)
    fe = torch.nn.Identity()
    for m, flag in ((BiCodec(), "global_tokens"), (BiCodec(global_tokens=True), "semantic_tokens"), (BiCodec(semantic_tokens=True), "global_tokens")):
        with pytest.raises(NotImplementedError, match=flag):
            BiCodecTokenizer(m, feature_extractor=fe).tokenize(wav)
    with pytest.raises(RuntimeError, match="CUDA"):
        BiCodecTokenizer(both, feature_extractor=fe).tokenize(wav)
