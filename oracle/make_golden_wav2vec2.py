"""Pin oracle/wav2vec2.py against transformers.Wav2Vec2FeatureExtractor + Wav2Vec2Model; write the fixture.

Run in the build container:  python -m oracle.make_golden_wav2vec2
The wav2vec2-large-xlsr-53 weights are not available offline: both sides load the SAME seeded random weights (the
architecture is what is pinned).  Outputs: tests/golden/wav2vec2_small.npz, tests/golden/wav2vec2_keys.json (key -> shape of
Wav2Vec2Model at the XLSR-53 configuration) and tests/golden/wav2vec2_pinning_report.json.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def hf_config(c, **kw):
    from transformers import Wav2Vec2Config
    return Wav2Vec2Config(hidden_size=c["hidden"], num_hidden_layers=c["layers"], num_attention_heads=c["heads"],
                          intermediate_size=c["ffn"], conv_dim=tuple(c["conv_dim"]), conv_kernel=tuple(c["conv_kernel"]),
                          conv_stride=tuple(c["conv_stride"]), num_conv_pos_embeddings=c["pos_k"],
                          num_conv_pos_embedding_groups=c["pos_groups"], feat_extract_norm="layer", conv_bias=True,
                          do_stable_layer_norm=True, hidden_dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                          feat_proj_dropout=0.0, layerdrop=0.0, **kw)


def hf_model(c, sd):
    from transformers import Wav2Vec2Model
    m = Wav2Vec2Model(hf_config(c, mask_time_prob=0.0)).eval()
    assert set(m.state_dict()) == set(sd), set(m.state_dict()) ^ set(sd)
    m.load_state_dict(sd, strict=True)
    return m


def hf_features(m, wav):
    """audio_tokenizer.py:74-90 with the transformers modules: processor on NumPy, model, mean of states 11 / 14 / 16"""
    from transformers import Wav2Vec2FeatureExtractor
    proc = Wav2Vec2FeatureExtractor(feature_size=1, sampling_rate=16000, padding_value=0.0, do_normalize=True,
                                    return_attention_mask=True)
    inputs = proc(np.asarray(wav), sampling_rate=16000, return_tensors="pt", padding=True).input_values
    with torch.no_grad():
        out = m(inputs, output_hidden_states=True)
    hs = out.hidden_states
    return inputs, hs, (hs[11] + hs[14] + hs[16]) / 3


def synth_wav(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return 0.1 * torch.randn(B, T, generator=g) + 0.03 * torch.randn(B, 1, generator=g)     # per-utterance DC offset


def main(out_dir=GOLD, pin_full=True):
    from transformers import Wav2Vec2Model
    from oracle import wav2vec2 as ow
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
    report = {}
    cases = [("small", ow.wav2vec2_small(), 2, 16000, 5)]
    if pin_full:
        cases.append(("xlsr53", ow.WAV2VEC2_XLSR53, 1, 8000, 6))
    for name, c, B, T, seed in cases:
        sd = ow.make_state_dict(c, seed)
        m = hf_model(c, sd)
        wav = synth_wav(B, T, seed + 50)
        inputs, hs_ref, feat_ref = hf_features(m, wav)
        e_norm = rel(ow.normalize(wav), inputs)
        hs = ow.hidden_states(sd, c, inputs)
        errs = [rel(a, b) for a, b in zip(hs, hs_ref)]
        assert len(hs) == len(hs_ref) == c["layers"] + 1
        feat = ow.extract_wav2vec2_features(sd, c, wav)
        e_feat = rel(feat, feat_ref)
        report[name] = dict(normalize_rel_err=e_norm, max_hidden_state_rel_err=max(errs), features_rel_err=e_feat,
                            frames=int(hs[0].shape[1]), hidden_states=len(hs), batch=B, samples=T)
        print(name, report[name])
        assert e_norm < 1e-6 and max(errs) < 2e-5 and e_feat < 1e-5
        if name == "small":
            np.savez_compressed(os.path.join(out_dir, "wav2vec2_small.npz"), meta=json.dumps(dict(seed=seed)), wav=wav.numpy(),
                                input_values=inputs.numpy(), feat=feat_ref.numpy(), last=hs_ref[-1].numpy())
    with torch.device("meta"):
        full = Wav2Vec2Model(hf_config(ow.WAV2VEC2_XLSR53))          # the published configuration (mask_time_prob 0.05)
    keys = {k: list(v.shape) for k, v in full.state_dict().items()}
    json.dump(keys, open(os.path.join(out_dir, "wav2vec2_keys.json"), "w"), indent=0, sort_keys=True)
    if pin_full:
        json.dump(report, open(os.path.join(out_dir, "wav2vec2_pinning_report.json"), "w"), indent=1)
    return report


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else GOLD)
