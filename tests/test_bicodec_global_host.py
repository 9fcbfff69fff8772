"""BiCodec global (speaker) tokens on the host: the oracle reproduces the outputs of the reference's own classes
(tests/golden/bicodec_global_small.npz, oracle/make_golden_bicodec_global.py), the product's state-dict layout of the path is the
reference's, its mel window and filter bank are torchaudio's, and there is no CPU path."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")
XVECTOR = ("speaker_encoder.speaker_encoder.pool.", "speaker_encoder.speaker_encoder.bn.", "speaker_encoder.speaker_encoder.linear.")


def small_state_dict(z):
    from oracle import bicodec_global as og
    meta = json.loads(str(z["meta"]))
    cfg = og.bicodec_global_small()
    sd = og.make_speaker_state_dict(cfg, meta["seed"])
    sd["speaker_encoder.quantizer.project_in.weight"] = torch.from_numpy(z["project_in_weight"])
    sd["speaker_encoder.quantizer.project_in.bias"] = torch.from_numpy(z["project_in_bias"])
    return cfg, sd


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


def test_oracle_reproduces_reference_global_tokens():
    from oracle import bicodec_global as og
    z = np.load(os.path.join(GOLD, "bicodec_global_small.npz"))
    cfg, sd = small_state_dict(z)
    taps = {}
    tokens = og.get_global_tokens({k: v.double() for k, v in sd.items()}, cfg, torch.from_numpy(z["ref_wav"]).double(), taps)
    assert tokens.dtype == torch.int32 and torch.equal(tokens, torch.from_numpy(z["tokens"]))
    for k in ("mel", "latent", "perceiver", "z"):
        assert rel(taps[k], z[k]) < 1e-5, k
    # the fixture decides every FSQ dimension away from a rounding boundary and visits all levels
    levels = cfg["speaker"]["fsq_levels"]
    assert float(og.fsq_margins(taps["z"], levels).min()) > 1e-2
    q = torch.round(og.fsq_bound(taps["z"], levels))
    assert all(len(set(q[..., j].reshape(-1).tolist())) == levels[j] for j in range(len(levels)))
    for n in ("short", "long"):
        assert torch.equal(og.get_ref_clip(torch.from_numpy(z[n + "_wav"]), 3200), torch.from_numpy(z[n + "_clip"]))


def test_global_spec_matches_reference_keys():
    from oracle import bicodec_global as og
    from unified_audio_b200.bicodec import BICODEC_CONFIG, MEL_PARAMS, BiCodec, bicodec_spec, speaker_spec
    keys = json.load(open(os.path.join(GOLD, "bicodec_global_keys.json")))
    want = {k: v for k, v in keys.items() if not k.startswith(XVECTOR) and not k.endswith(".num_batches_tracked")}
    assert MEL_PARAMS == og.MEL_PARAMS
    assert {k: list(v) for k, v in speaker_spec(BICODEC_CONFIG).items()} == want
    assert {k: list(v[0]) for k, v in og.speaker_param_specs(og.BICODEC_GLOBAL_FULL).items()} == want
    m = BiCodec(global_tokens=True)
    assert set(m.state_dict()) == set(bicodec_spec(BICODEC_CONFIG)) | set(want)
    # a strict load needs the global-path keys, and ignores the x-vector branch, num_batches_tracked and the mel buffers
    from oracle import bicodec as ob
    sd = dict(ob.make_state_dict(ob.BICODEC_FULL, 1))
    sd.update(og.make_speaker_state_dict(og.BICODEC_GLOBAL_FULL, 1))
    extra = dict(sd)
    for k, shape in keys.items():
        if k.startswith(XVECTOR) or k.endswith(".num_batches_tracked"):
            extra[k] = torch.zeros(shape)
    extra["mel_transformer.spectrogram.window"] = torch.zeros(640)
    extra["encoder.linear_pre.weight"] = torch.zeros(2, 2)
    m.load_state_dict(extra, strict=True)
    missing = dict(sd)
    del missing["speaker_encoder.perceiver_sampler.latents"]
    with pytest.raises(RuntimeError):
        BiCodec(global_tokens=True).load_state_dict(missing, strict=True)
    # the default object is unchanged: the global-path keys are ignored, not required
    assert set(BiCodec().state_dict()) == set(bicodec_spec(BICODEC_CONFIG))
    BiCodec().load_state_dict(extra, strict=True)


def test_mel_window_and_filter_bank_are_torchaudio_buffers():
    torchaudio = pytest.importorskip("torchaudio")
    from unified_audio_b200.bicodec import MEL_PARAMS, hann_window, mel_filterbank
    for mp in (MEL_PARAMS, dict(MEL_PARAMS, num_mels=80)):
        t = torchaudio.transforms.MelSpectrogram(mp["sample_rate"], mp["n_fft"], mp["win_length"], mp["hop_length"], mp["mel_fmin"],
                                                 mp["mel_fmax"], n_mels=mp["num_mels"], power=1, norm="slaney", mel_scale="slaney")
        fb = t.mel_scale.fb.double()
        assert fb.shape == (mp["n_fft"] // 2 + 1, mp["num_mels"])
        assert float((mel_filterbank(mp) - fb).abs().max()) < 1e-5 * float(fb.abs().max())     # torchaudio builds it in fp32
        left = (mp["n_fft"] - mp["win_length"]) // 2
        w = hann_window(mp)
        assert float((w[left:left + mp["win_length"]] - t.spectrogram.window.double()).abs().max()) < 1e-6
        assert float(w[:left].abs().max()) == 0.0 and float(w[left + mp["win_length"]:].abs().max()) == 0.0


def test_default_bicodec_refuses_global_tokens_and_there_is_no_cpu_path():
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.unise import BiCodecTokenizer
    with pytest.raises(RuntimeError, match="global_tokens=True"):
        BiCodec().get_global_tokens({"ref_wav": torch.zeros(1, 4000)})
    m = BiCodec(global_tokens=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.get_global_tokens({"ref_wav": torch.zeros(1, 4000)})
    with pytest.raises(RuntimeError, match="CUDA"):
        m.mel_spectrogram(torch.zeros(1, 4000))
    with pytest.raises(RuntimeError, match="CUDA"):
        BiCodecTokenizer(m).get_ref_clip(torch.zeros(1, 4000))
    with pytest.raises(NotImplementedError):
        BiCodecTokenizer(m).tokenize(torch.zeros(1, 4000))
