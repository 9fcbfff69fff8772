"""wav2vec2-large-xlsr-53 front end on the GPU (BiCodecTokenizer.extract_wav2vec2_features) against the oracle
(oracle/wav2vec2.py, pinned against transformers.Wav2Vec2Model and Wav2Vec2FeatureExtractor by tests/golden/wav2vec2_small.npz)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-3


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def gpu_small():
    """reduced widths the kernels support (head_dim 64); 17 layers so that layer 17 and encoder.layer_norm stay dead"""
    return dict(conv_dim=[64] * 7, conv_kernel=[10, 3, 3, 3, 3, 2, 2], conv_stride=[5, 2, 2, 2, 2, 2, 2], hidden=128, layers=17, heads=2,
                ffn=256, pos_k=16, pos_groups=4, eps=1e-5, hidden_state_ids=(11, 14, 16))


def _build(c, sd):
    from unified_audio_b200.ssl import SSLFrontEnd
    m = SSLFrontEnd(dict(c, kind="wav2vec2", do_normalize=True), in_rate=16000)
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def test_wav2vec2_normalize_matches_feature_extractor(lib):
    """per-utterance normalisation on the device == Wav2Vec2FeatureExtractor's output in the fixture (NumPy fp32 statistics) and
    the oracle's fp64 statistics"""
    from oracle import wav2vec2 as ow
    from unified_audio_b200.ssl import SSLFrontEnd
    z = np.load(os.path.join(ROOT, "tests", "golden", "wav2vec2_small.npz"))
    c = gpu_small()
    m = SSLFrontEnd(dict(c, kind="wav2vec2", do_normalize=True)).cuda()
    wav = torch.from_numpy(z["wav"])
    got = m.normalize(wav.cuda())
    torch.cuda.synchronize()
    e_proc, e_or = rel(got, torch.from_numpy(z["input_values"])), rel(got, ow.normalize(wav))
    print(f"[wav2vec2 normalize] vs feature extractor {e_proc:.2e} vs fp64 oracle {e_or:.2e}")
    assert e_proc < 1e-6 and e_or < 1e-6


@pytest.mark.parametrize("cfg_name,B,samples", [("small", 3, 8000), ("xlsr53", 2, 80000)])
def test_wav2vec2_front_end_vs_oracle(lib, cfg_name, B, samples):
    """features of B x (samples / 16000) s against the oracle: conv features, hidden state 0, the last state averaged and the
    output; XLSR-53 at full width on 5 s segments (249 frames, as the reference's tokenize yields)"""
    from oracle import wav2vec2 as ow
    c = gpu_small() if cfg_name == "small" else ow.WAV2VEC2_XLSR53
    sd = ow.make_state_dict(c, 5)
    m = _build(c, sd)
    wav = 0.1 * torch.randn(B, samples, generator=torch.Generator().manual_seed(77)) + 0.02
    taps = {}
    got = m(wav.cuda(), taps=taps)
    torch.cuda.synchronize()
    x = ow.normalize(wav)
    feats = ow.feature_encoder(sd, c, x).transpose(1, 2)
    hs = ow.hidden_states(sd, c, x, layers=max(c["hidden_state_ids"]))
    ref = ow.extract_wav2vec2_features(sd, c, wav)
    last = max(c["hidden_state_ids"])
    e_f, e_0, e_l, e = rel(taps["features"], feats), rel(taps["hs0"], hs[0]), rel(taps[f"hs{last}"], hs[last]), rel(got, ref)
    print(f"[wav2vec2 {cfg_name} B={B} {samples / 16000:.1f}s] conv features {e_f:.2e} hs0 {e_0:.2e} hs{last} {e_l:.2e} "
          f"features (mean of states {c['hidden_state_ids']}) {e:.2e}; frames {got.shape[1]}")
    assert got.shape == ref.shape == (B, (samples - 400) // 320 + 1, c["hidden"])
    assert f"hs{last + 1}" not in taps                       # layers past the last averaged state are not run
    assert max(e_f, e_0, e_l, e) < TOL
    if cfg_name == "xlsr53":
        assert got.shape[1] == 249


def test_wav2vec2_rejects_input_shorter_than_the_receptive_field(lib):
    from oracle import wav2vec2 as ow
    c = gpu_small()
    m = _build(c, ow.make_state_dict(c, 9))
    with pytest.raises(ValueError, match="at least 400 samples"):
        m(torch.zeros(2, 399, device="cuda"))


def test_wav2vec2_dead_weights_do_not_reach_the_output(lib):
    """layers past the last averaged state and encoder.layer_norm are loaded (strict=True) but never read: NaN there changes
    nothing"""
    from oracle import wav2vec2 as ow
    c = gpu_small()
    sd = ow.make_state_dict(c, 9)
    wav = 0.1 * torch.randn(2, 6000, generator=torch.Generator().manual_seed(1))
    a = _build(c, sd)(wav.cuda())
    bad = {k: (torch.full_like(v, float("nan")) if k.startswith(("encoder.layers.16.", "encoder.layer_norm.")) else v) for k, v in sd.items()}
    b = _build(c, bad)(wav.cuda())
    torch.cuda.synchronize()
    assert bool(torch.isfinite(b).all()) and torch.equal(a, b)
    assert rel(a, ow.extract_wav2vec2_features(sd, c, wav)) < TOL
