"""unified_audio_b200 - H100-native (sm_90a) implementation of QuarkAudio's audio-token hot path.

Public surface mirrors the reference (alibaba/unified-audio):
  Codec            <- QuarkAudio-HCodec/HCodec-2.0/vq/codec.py:17   (encode / decode)
  ResidualVQ       <- vector_quantize_pytorch.ResidualVQ as the reference constructs it
  LLM_SFT          <- QuarkAudio-UniSE/model/llm/llm_sft.py:13 (llm_forward / forward / generate)
  CodecH1          <- QuarkAudio-HCodec/HCodec-1.0/vq/codec.py:21   (encode / decode)
  CodecH15         <- QuarkAudio-HCodec/HCodec-1.5/vq/codec_adaptive.py:32 (adaptive frame rate: encode / decode with length-packed codes)
  BiCodec          <- QuarkAudio-UniSE/model/bicodec/bicodec.py:151-199 (detokenize; get_global_tokens, get_semantic_tokens and
                      tokenize with global_tokens=True / semantic_tokens=True)
  SSLFrontEnd      <- HuBERT-base / WavLM-base-plus / wav2vec2-XLSR-53 feature extraction as HCodecTokenizer.extract_ssl_features
                      (HCodec-2.0/audio_tokenizer.py:47-61), Model.extract_semantic_features (U/model/model.py:38-51) and
                      BiCodecTokenizer.extract_wav2vec2_features (U/model/bicodec/audio_tokenizer.py:74-90) drive them
  HCodecTokenizer  <- QuarkAudio-HCodec/HCodec-2.0/audio_tokenizer.py:21-79 (pad_wav / tokenize / detokenize)
  HCodecTokenizerH1  <- QuarkAudio-HCodec/HCodec-1.0/audio_tokenizer.py:18-66 (HuBERT-base features -> CodecH1)
  HCodecTokenizerH15 <- QuarkAudio-HCodec/HCodec-1.5/audio_tokenizer.py:38-86 (wav2vec2-XLSR-53 features, WAV2VEC2_XLSR53_RAW ->
                      CodecH15, length-packed codes)
  unise.Model      <- QuarkAudio-UniSE/model/model.py:20-286 (extract_semantic_features / test_step: 'se', 'tse', 'ss') with
                      unise.BiCodecTokenizer <- model/bicodec/audio_tokenizer.py:30-125 (get_ref_clip / tokenize / detokenize)
  Simulator        <- QuarkAudio-UniSE/dataloader/simulation/simulate.py:126-192 (simulate_data) and the post-load steps of
                      TrainDataLoadIter.process_one_sample (dataloader/data_module.py:106-140, 207-235): training batches on the GPU
Kernels live in csrc/ behind the C ABI of include/quark_b200.h (lib/libquark_b200.so).
"""
__version__ = "0.1.0"

from .codec import Codec  # noqa: E402,F401
from .codec_h1 import CodecH1  # noqa: E402,F401
from .codec_h15 import CodecH15  # noqa: E402,F401
from .rvq import ResidualVQ  # noqa: E402,F401
from .llm import LLM_SFT  # noqa: E402,F401
from .bicodec import BiCodec  # noqa: E402,F401
from . import adaptive  # noqa: E402,F401
from .ssl import HCodecTokenizer, HUBERT_BASE, SSLFrontEnd, WAV2VEC2_XLSR53, WAVLM_BASE_PLUS, pad_wav, wrap_segments  # noqa: E402,F401
from .ssl import HCodecTokenizerH1, HCodecTokenizerH15, WAV2VEC2_XLSR53_RAW  # noqa: E402,F401
from . import unise  # noqa: E402,F401
from .simulate import Simulator  # noqa: E402,F401
