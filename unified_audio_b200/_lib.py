"""ctypes binding of libquark_b200.so (the C ABI declared in include/quark_b200.h).

The library is built in-tree by unified_audio_b200/build.py (nvcc, sm_90a).  There is NO fallback:
if the shared library is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("QB_LIB") or os.path.join(_HERE, "lib", "libquark_b200.so")     # QB_LIB: A/B builds for experiments

ACT_NONE, ACT_GELU, ACT_SWIGLU, ACT_ELU, ACT_TANH, ACT_SNAKE, ACT_RELU = 0, 1, 2, 3, 4, 5, 6


class RowMap(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("ld", C.c_int64), ("rows_per_batch", C.c_int64), ("row_off", C.c_int64)]


class GemmDesc(C.Structure):
    _fields_ = [
        ("a_hi", C.c_void_p), ("a_lo", C.c_void_p), ("a_batch", C.c_int64), ("a_rows_per_batch", C.c_int64),
        ("a_ld", C.c_int64), ("taps", C.c_int32), ("stride", C.c_int32), ("m_per_batch", C.c_int64),
        ("w_hi", C.c_void_p), ("w_lo", C.c_void_p), ("n", C.c_int64), ("bias", C.c_void_p), ("gamma", C.c_void_p),
        ("residual", RowMap), ("act", C.c_int32), ("act2", C.c_int32), ("out_f32", RowMap), ("out_hi", RowMap),
        ("out_lo", RowMap), ("dilation", C.c_int32), ("act_param", C.c_void_p), ("act2_param", C.c_void_p),
        ("a_cols", C.c_int64),
    ]


class Tensor(C.Structure):       # qb_tensor
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("ndim", C.c_int32), ("shape", C.c_int64 * 4)]


class CodecCfg(C.Structure):     # qb_codec_cfg
    _fields_ = [(n, C.c_int32) for n in (
        "dim", "intermediate_dim", "dimension", "n_fft", "hop_length", "enc_convnext_layers", "enc_transformer_layers",
        "dec_convnext_layers", "dec_transformer_layers", "dec_input_channels", "frame_stride", "num_quantizers", "codebook_size",
        "sem_input_channels", "sem_encode_channels", "sem_out_channels", "sem_n_blocks")] + [("sem_strides", C.c_int32 * 8),
                                                                                             ("precision", C.c_int32)]


TAP_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64)
PRECISION_CODES = {"mixed": 0, "accurate": 1, "fast": 2, "mixed_dec16": 3}

# name -> (restype, argtypes); mirrors include/quark_b200.h one to one
_vp, _i64, _i32, _f32 = C.c_void_p, C.c_int64, C.c_int32, C.c_float
SIGNATURES = {
    "qb_last_error": (C.c_char_p, []),
    "qb_version": (C.c_int, []),
    "qb_launch_count": (C.c_int64, []),
    "qb_launch_count_reset": (None, []),
    "qb_gemm": (C.c_int, [C.POINTER(GemmDesc), _vp]),
    "qb_gemm_simt": (C.c_int, [C.POINTER(GemmDesc), _vp]),
    "qb_gemm_kernel_name": (C.c_char_p, [_i64, _i64, _i32]),
    "qb_split_f16": (C.c_int, [_vp, _vp, _vp, _i64, _vp]),
    "qb_rows_to_planes": (C.c_int, [_vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_bct_to_planes": (C.c_int, [_vp, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_layernorm": (C.c_int, [_vp, _vp, _vp, _f32, _i64, _i64, _i64, _vp, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_layernorm_act": (C.c_int, [_vp, _vp, _vp, _f32, _i64, _i64, _i64, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_rmsnorm": (C.c_int, [_vp, _vp, _f32, _i64, _i64, _vp, _vp, _vp, _vp]),
    "qb_dwconv7_ln": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp]),
    "qb_dwconv7_adaln": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp]),
    "qb_adalayernorm": (C.c_int, [_vp, _vp, _vp, _i64, _f32, _i64, _i64, _i64, _vp, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_snake_planes": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_addvec_planes": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_groupnorm_stats": (C.c_int, [_vp, _i64, _i64, _i64, _i32, _f32, _vp, _vp]),
    "qb_groupnorm_apply": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _i64, _i64,
                                      _i64, _vp]),
    "qb_stft_gather": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "qb_stft_twiddle": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp]),
    "qb_stft_post2": (C.c_int, [_vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_istft_pre": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _vp, _i64, _vp]),
    "qb_istft_ola": (C.c_int, [_vp, _vp, _i64, _i64, _i32, _i32, _vp, _vp]),
    "qb_reflect_pad_rows": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _i32, _i32, _vp]),
    "qb_dwconv": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp, _vp]),
    "qb_attention_hd": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "qb_attention_umma_workspace_bytes": (C.c_int64, [_i64, _i64, _i32, _i32, _i32]),
    "qb_attention_umma": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "qb_lstm_tc_units": (C.c_int32, [_i64]),
    "qb_lstm_tc_workspace_bytes": (C.c_int64, [_i64, _i64]),
    "qb_lstm_tc": (C.c_int, [_vp, _vp, _i32, _i64, _i64, _i64, _vp, _vp, _vp, _vp]),
    "qb_rvq_workspace_bytes": (C.c_int64, [_i64, _i32, _i32]),
    "qb_rvq_encode": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _f32, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "qb_rvq_decode": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _i32, _vp, _i64, _i64, _vp]),
    "qb_fvq_tokenize": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "qb_lm_qkv_prep": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp]),
    "qb_lm_flash_attn": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _vp]),
    "qb_lm_pack_weight": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "qb_lm_decode_layer_tc": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp,
                                        _vp, _vp, _vp, _vp]),
    "qb_lm_set_att_unroll": (C.c_int, [_i32]),
    "qb_lm_head_argmax_tc": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "qb_ssl_conv0_workspace_bytes": (C.c_int64, [_i64, _i64, _i32]),
    "qb_ssl_conv0_gn_gelu": (C.c_int, [_vp, _i64, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_ssl_conv0_bias": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "qb_wav_normalize": (C.c_int, [_vp, _i64, _i64, _f32, _vp, _vp]),
    "qb_wavlm_gate": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "qb_attention_relbias": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "qb_axpy": (C.c_int, [_vp, _f32, _i64, _i32, _vp, _vp]),
    "qb_ssl_compress": (C.c_int, [_vp, _i64, _i64, _i32, _f32, _i32, _vp, _vp]),
    "qb_pad_wav": (C.c_int, [_vp, _i64, _i64, _i64, _i64, _i32, _vp, _vp]),
    "qb_mel_gather": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "qb_spec_magnitude": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _i64, _vp]),
    "qb_add_planes": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i64, _vp]),
    "qb_se_gate": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp]),
    "qb_se_apply": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i32, _vp, _vp, _vp, _i64, _i64, _vp]),
    "qb_geglu_planes": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _i64, _vp]),
    "qb_cross_attention": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _i32, _vp, _vp, _vp]),
    "qb_fsq_tokenize": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp, _i32, C.POINTER(C.c_int32), _i32, _vp, _vp, _vp, _vp]),
    "qb_similarity_alignment": (C.c_int, [_vp, _i64, _i64, _i32, _f32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "qb_alignment_matrix": (C.c_int, [_vp, _i64, _i64, _i64, _vp, _vp]),
    "qb_pack_lengths": (C.c_int, [_vp, _vp, _i64, _i32, _i64, _i32, _vp, _vp]),
    "qb_unpack_lengths": (C.c_int, [_vp, _i64, _i32, _i64, _i32, _vp, _vp, _vp]),
    "qb_length_offsets": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp]),
    "qb_deaggregate": (C.c_int, [_vp, _i32, _vp, _vp, _i64, _i64, _i64, _i64, _vp, _vp]),
    "qb_agg_interleave": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp, _vp, _vp]),
    "qb_agg_gather": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp, _vp]),
    "qb_init": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "qb_handle_free": (None, [_vp]),
    "qb_memcpy_d2d": (C.c_int, [_vp, _vp, _i64, _vp]),
    "qb_handle_last_error": (C.c_char_p, [_vp]),
    "qb_codec_load": (C.c_int, [_vp, C.POINTER(CodecCfg), C.POINTER(Tensor), _i32, C.POINTER(_vp)]),
    "qb_codec_free": (None, [_vp]),
    "qb_codec_encode": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "qb_codec_decode": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _vp, _vp]),
    "qb_codec_set_tap": (C.c_int, [_vp, TAP_FN, _vp]),
    "qb_codec_rvq": (_vp, [_vp, _i32]),
    "qb_rvq_load": (C.c_int, [_vp, _vp, _i32, _i32, _i32, C.POINTER(_vp)]),
    "qb_rvq_free": (None, [_vp]),
    "qb_rvq_encode_rows": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "qb_rvq_decode_rows": (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    "qb_lm_loss": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _f32, _vp, _vp, _vp]),
    "qb_lm_attn_train_fwd": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _vp, _f32, C.c_uint64, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "qb_lm_attn_train_bwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i32, _vp, _vp, _f32, C.c_uint64, _i32, _vp, _vp,
                                       _vp]),
    "qb_lm_loss_bwd": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _f32, _vp, _f32, _vp, _vp, _vp, _i64, _vp]),
    "qb_rmsnorm_bwd": (C.c_int, [_vp, _vp, _vp, _f32, _i64, _i64, _vp, _i32, _vp, _vp]),
    "qb_col_sum_workspace_bytes": (C.c_int64, [_i64, _i64]),
    "qb_col_sum": (C.c_int, [_vp, _i64, _i64, _i64, C.c_double, _vp, _vp, _i32, _vp]),
    "qb_swiglu": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "qb_swiglu_bwd": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "qb_transpose_split": (C.c_int, [_vp, _i64, _i64, _i64, _i64, _vp, _vp, _vp]),
    "qb_embedding_bwd": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, C.c_double, _vp, _i32, _vp]),
    "qb_sim_active_rms": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp]),
    "qb_sim_place": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp]),
    "qb_sim_mix": (C.c_int, [_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "qb_sim_rir_prep": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "qb_sim_convolve": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "qb_sim_bandwidth": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _i32, _vp, _vp]),
    "qb_sim_clip": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "qb_sim_packet_loss": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "qb_sim_finish": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "qb_sim_enroll": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp]),
    "qb_lm_head_sample_tc":(C.c_int, [_vp, _i64, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _f32, _i32,
                                       _f32, _vp, _vp, _vp]),
}

_lib = None


def load():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found - build it with `python -m unified_audio_b200.build` "
                "(there is no CPU / PyTorch fallback for the product path)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(code: int):
    if code != 0:
        raise RuntimeError(f"libquark_b200 error {code}: {load().qb_last_error().decode()}")
