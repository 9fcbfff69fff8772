"""CPU restatement of the SSL features the H-Codec-1.0 and H-Codec-1.5 tokenizers feed their codecs.

TEST INFRASTRUCTURE - see oracle/__init__.py.  Pinned by oracle/make_golden_hcodec_tokenizers.py against the reference's own
`HCodecTokenizer.extract_wav2vec2_features` (tests/golden/hcodec_tokenizers_small.npz).

    HCodec-1.0/audio_tokenizer.py:35-49 (HuBERT-base despite the method's name): wav 16 kHz (no resampling) -> pad 160/160 ->
        HubertModel(output_hidden_states) -> mean of all 1 + layers hidden states -> sign(x) |x|^0.3          [B, T/320, 768]
    HCodec-1.5/audio_tokenizer.py:52-66: wav 16 kHz -> pad 160/160 -> Wav2Vec2Model called bare (no Wav2Vec2FeatureExtractor
        normalisation) -> mean of hidden_states[k] for k in hidden_state_ids ((11, 14, 16) for XLSR-53) -> sign(x) |x|^0.3
                                                                                                              [B, T/320, 1024]
oracle.hubert.extract_ssl_features ties the compression to the 48 kHz resampler of H-Codec-2.0, and
oracle.wav2vec2.extract_wav2vec2_features normalises and does not pad (BiCodec), so neither is either of these.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import hubert as oh
from . import wav2vec2 as ow


def compress(x):
    """audio_tokenizer.py: symbol = (x > 0) * 2 - 1; symbol * |x| ** 0.3"""
    return ((x > 0).float() * 2 - 1) * x.abs() ** 0.3


@torch.no_grad()
def extract_hcodec1_features(sd, c, wav16k):
    return compress(torch.stack(oh.hubert_hidden_states(sd, c, F.pad(wav16k, (160, 160))), 1).mean(1))


@torch.no_grad()
def extract_hcodec15_features(sd, c, wav16k):
    ids = c["hidden_state_ids"]
    hs = ow.hidden_states(sd, c, F.pad(wav16k, (160, 160)), layers=max(ids))
    return compress(sum(hs[i] for i in ids) / len(ids))
