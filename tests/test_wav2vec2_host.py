"""wav2vec2-large-xlsr-53 front end without a GPU: the oracle against the transformers fixture, the checkpoint surface of
SSLFrontEnd(WAV2VEC2_XLSR53) against transformers.Wav2Vec2Model's keys, and the refusal to run off the GPU."""
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def test_oracle_wav2vec2_matches_transformers_fixture():
    """oracle/wav2vec2.py reproduces Wav2Vec2FeatureExtractor(do_normalize=True) and the mean of Wav2Vec2Model's hidden states
    11 / 14 / 16 (BiCodecTokenizer.extract_wav2vec2_features) on the committed fixture (oracle/make_golden_wav2vec2.py)."""
    from oracle import wav2vec2 as ow
    z = np.load(os.path.join(GOLD, "wav2vec2_small.npz"))
    meta = json.loads(str(z["meta"]))
    c = ow.wav2vec2_small()
    sd = ow.make_state_dict(c, meta["seed"])
    wav = torch.from_numpy(z["wav"])
    assert rel(ow.normalize(wav), torch.from_numpy(z["input_values"])) < 1e-6
    feat = ow.extract_wav2vec2_features(sd, c, wav)
    assert feat.shape == z["feat"].shape and rel(feat, torch.from_numpy(z["feat"])) < 1e-5
    hs = ow.hidden_states(sd, c, torch.from_numpy(z["input_values"]))
    assert len(hs) == c["layers"] + 1 and rel(hs[-1], torch.from_numpy(z["last"])) < 1e-5


def test_wav2vec2_keys_match_transformers():
    """SSLFrontEnd(WAV2VEC2_XLSR53) holds every key of transformers.Wav2Vec2Model at the XLSR-53 configuration (all 24 layers),
    with the same shapes; masked_spec_embed (pre-training only) is accepted at load and not kept."""
    from oracle import wav2vec2 as ow
    from unified_audio_b200.ssl import WAV2VEC2_XLSR53, ssl_spec
    ref = json.load(open(os.path.join(GOLD, "wav2vec2_keys.json")))
    assert ref.pop("masked_spec_embed") == [WAV2VEC2_XLSR53["hidden"]]
    mine = {k: list(v) for k, v in ssl_spec(WAV2VEC2_XLSR53).items()}
    assert mine == ref
    assert {k: list(s) for k, (s, _) in ow.param_specs(ow.WAV2VEC2_XLSR53).items()} == ref
    assert sum(k.startswith("encoder.layers.23.") for k in mine) == 16


def test_wav2vec2_front_end_loads_checkpoint_and_refuses_cpu():
    from oracle import wav2vec2 as ow
    from unified_audio_b200.ssl import SSLFrontEnd
    c = ow.wav2vec2_small()
    sd = ow.make_state_dict(c, 3)
    m = SSLFrontEnd(dict(c, kind="wav2vec2", do_normalize=True), in_rate=16000)
    m.load_state_dict(dict(sd, masked_spec_embed=torch.zeros(c["hidden"])), strict=True)
    got = m.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 4000))
    with pytest.raises(ValueError):       # the last state carries encoder.layer_norm: not one of the averaged residual states
        SSLFrontEnd(dict(c, kind="wav2vec2", hidden_state_ids=(11, 17)))
    assert m.min_samples() == 400         # receptive field of the XLSR-53 conv stack (k 10,3,3,3,3,2,2 / s 5,2,2,2,2,2,2)
    assert ow.feature_encoder(sd, c, torch.zeros(1, 400)).shape[-1] == 1


def test_make_golden_wav2vec2_reproduces_committed_fixture(tmp_path):
    pytest.importorskip("transformers")
    from oracle import make_golden_wav2vec2
    make_golden_wav2vec2.main(str(tmp_path), pin_full=False)
    assert json.load(open(tmp_path / "wav2vec2_keys.json")) == json.load(open(os.path.join(GOLD, "wav2vec2_keys.json")))
    new, old = np.load(tmp_path / "wav2vec2_small.npz"), np.load(os.path.join(GOLD, "wav2vec2_small.npz"))
    assert sorted(new.files) == sorted(old.files) and str(new["meta"]) == str(old["meta"])
    assert np.array_equal(new["wav"], old["wav"])
    for k in ("input_values", "feat", "last"):
        assert rel(torch.from_numpy(new[k]), torch.from_numpy(old[k])) < 1e-6, k
