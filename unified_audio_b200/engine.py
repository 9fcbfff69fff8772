"""ctypes front end of the handle-level C ABI (include/quark_b200.h "Handle-level contract"; csrc/engine.cu):
per-device context, H-Codec-2.0 codec handle, residual-VQ handle.  `Codec` (codec.py) is a thin caller of these for the
product path; the UniSE LM (llm.py) composes the op-level entry points instead."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from ._lib import CodecCfg, PRECISION_CODES, TAP_FN, Tensor

_CONTEXTS: Dict[int, "Context"] = {}


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Context:
    """qb_handle: one per device."""

    def __init__(self, device: int):
        h = C.c_void_p()
        _lib.check(_lib.load().qb_init(int(device), C.byref(h)))
        self.h, self.device = h, device

    @staticmethod
    def get(device: torch.device) -> "Context":
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in _CONTEXTS:
            _CONTEXTS[idx] = Context(idx)
        return _CONTEXTS[idx]


def _tensor_array(named: Dict[str, torch.Tensor]):
    """state-dict -> qb_tensor[] (fp32, contiguous, CUDA); returns (array, keep-alive list)"""
    keep, arr = [], (Tensor * len(named))()
    for i, (k, v) in enumerate(named.items()):
        t = v.detach().float().contiguous()
        if not t.is_cuda:
            raise RuntimeError("libquark_b200 handles are built from CUDA tensors (no CPU fallback): call .cuda() first")
        if t.dim() > 4:
            raise ValueError(f"{k}: more than 4 dims")
        name = k.encode()
        keep += [t, name]
        arr[i].name, arr[i].data, arr[i].ndim = name, t.data_ptr(), t.dim()
        for j, s in enumerate(t.shape):
            arr[i].shape[j] = s
    return arr, keep


class CodecEngine:
    """qb_codec: owns the repacked weights + workspace of one H-Codec-2.0 model."""

    def __init__(self, device, enc: dict, dec: dict, quant: dict, sem: dict, precision: str, state_dict: Dict[str, torch.Tensor]):
        self.lib = _lib.load()
        self.ctx = Context.get(device)
        cfg = CodecCfg()
        cfg.dim, cfg.intermediate_dim, cfg.dimension = enc["dim"], enc["intermediate_dim"], enc["dimension"]
        cfg.n_fft, cfg.hop_length = enc.get("n_fft", 1920), enc.get("hop_length", 960)
        if dec.get("n_fft", 1920) != cfg.n_fft or dec.get("hop_length", 960) != cfg.hop_length:
            raise RuntimeError("encoder / decoder STFT geometry must match")
        if dec["dim"] != enc["dim"] or dec["intermediate_dim"] != enc["intermediate_dim"]:
            raise RuntimeError("the engine assumes equal encoder / decoder widths (shipped config)")
        cfg.enc_convnext_layers, cfg.enc_transformer_layers = enc["convnext_layers"], enc.get("transformer_layers", 2)
        cfg.dec_convnext_layers, cfg.dec_transformer_layers = dec["convnext_layers"], dec.get("transformer_layers", 2)
        cfg.dec_input_channels = dec["input_channels"]
        cfg.frame_stride = int(50 / enc["target_frame_rate"])
        if int(50 / dec["target_frame_rate"]) != cfg.frame_stride:
            raise RuntimeError("encoder / decoder frame rates must match")
        cfg.num_quantizers, cfg.codebook_size = quant["num_quantizers"], quant["codebook_size"]
        cfg.sem_input_channels, cfg.sem_encode_channels, cfg.sem_out_channels = sem["input_channels"], sem["encode_channels"], sem["out_channels"]
        if any(float(r) != 1.0 for r in sem["channel_ratios"]):
            raise RuntimeError("semantic encoder: only channel_ratios == 1 (shipped config) is implemented")
        cfg.sem_n_blocks = len(sem["strides"])
        for i, s in enumerate(sem["strides"]):
            cfg.sem_strides[i] = s
        cfg.precision = PRECISION_CODES[precision]
        self.cfg = cfg
        arr, keep = _tensor_array(state_dict)
        h = C.c_void_p()
        _lib.check(self.lib.qb_codec_load(self.ctx.h, C.byref(cfg), arr, len(state_dict), C.byref(h)))
        del keep
        self.h = h
        self._tap_cb = None

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.qb_codec_free(self.h)
                self.h = None
        except Exception:
            pass

    def set_taps(self, taps: Optional[dict]):
        """taps: dict filled with clones [B, C, rows] (channel-first like the reference's tensors) of every named intermediate"""
        if taps is None:
            _lib.check(self.lib.qb_codec_set_tap(self.h, TAP_FN(0), None))
            self._tap_cb = None
            return

        def cb(user, name, ptr, B, rows, Cc):
            n = B * rows * Cc
            buf = torch.empty(B, rows, Cc, device="cuda")
            # stream-ordered device copy of the engine's buffer (same stream as the kernels that produced it)
            _lib.check(self.lib.qb_memcpy_d2d(buf.data_ptr(), ptr, n * 4, _stream()))
            nm = name.decode()
            taps[nm] = buf if nm == "dec.final_norm" else buf.transpose(1, 2)     # (the reference keeps this one [B, T, C])
        self._tap_cb = TAP_FN(cb)
        _lib.check(self.lib.qb_codec_set_tap(self.h, self._tap_cb, None))

    def encode(self, wav: torch.Tensor, feat: torch.Tensor):
        B, T = wav.shape
        hop, st = self.cfg.hop_length, self.cfg.frame_stride
        if T % (hop * st) != 0:
            raise ValueError(f"waveform length {T} must be a multiple of {hop * st} (pad_wav, audio_tokenizer.py:63-66)")
        if tuple(feat.shape) != (B, self.cfg.sem_input_channels, T // hop):
            raise ValueError(f"feat must be [B, {self.cfg.sem_input_channels}, T/{hop}] = {(B, self.cfg.sem_input_channels, T // hop)}, got {tuple(feat.shape)}")
        N = T // (hop * st)
        wav, feat = wav.float().contiguous(), feat.float().contiguous()
        ac = torch.empty(B, self.cfg.num_quantizers, N, dtype=torch.int64, device=wav.device)
        sc = torch.empty_like(ac)
        _lib.check(self.lib.qb_codec_encode(self.h, wav.data_ptr(), B, T, feat.data_ptr(), ac.data_ptr(), sc.data_ptr(), _stream()))
        return ac, sc

    def decode(self, ac: torch.Tensor, sc: torch.Tensor):
        B, nq, N = ac.shape
        ac, sc = ac.long().contiguous(), sc.long().contiguous()
        wav = torch.empty(B, N * self.cfg.frame_stride * self.cfg.hop_length, device=ac.device)
        _lib.check(self.lib.qb_codec_decode(self.h, ac.data_ptr(), sc.data_ptr(), B, N, wav.data_ptr(), _stream()))
        return wav

    def load_semantic_decoder(self, cfg: dict, state_dict: Dict[str, torch.Tensor]):
        """qb_codec_load_semantic_decoder: cfg = the reference's semantic_decoder_config, state_dict = its semantic_decoder.* tensors"""
        if len(cfg["strides"]) > 8:
            raise ValueError("semantic decoder: at most 8 blocks")
        c = _lib.SemanticDecoderCfg()
        c.code_dim, c.output_channels, c.n_blocks = cfg["code_dim"], cfg["output_channels"], len(cfg["strides"])
        for i, s in enumerate(cfg["strides"]):
            c.strides[i] = s
        arr, keep = _tensor_array(state_dict)
        _lib.check(self.lib.qb_codec_load_semantic_decoder(self.h, C.byref(c), arr, len(state_dict)))
        del keep
        self.sem_dec_out, self.sem_dec_up = cfg["output_channels"], 1
        for s in cfg["strides"]:
            self.sem_dec_up *= s

    def semantic_decode(self, sc: torch.Tensor):
        """int64 [B, nq, N] -> pred_feat fp32 [B, output_channels, N * prod(strides)]"""
        B, nq, N = sc.shape
        if nq != self.cfg.num_quantizers:
            raise ValueError(f"semantic codes must have {self.cfg.num_quantizers} quantiser layers, got {nq}")
        sc = sc.long().contiguous()
        out = torch.empty(B, self.sem_dec_out, N * self.sem_dec_up, device=sc.device)
        _lib.check(self.lib.qb_codec_semantic_decode(self.h, sc.data_ptr(), B, N, out.data_ptr(), _stream()))
        return out

    def rvq(self, which: int) -> "RvqEngine":
        return RvqEngine(handle=self.lib.qb_codec_rvq(self.h, which), owner=self, nq=self.cfg.num_quantizers, D=self.cfg.dimension)


class RvqEngine:
    """qb_rvq: codebooks [nq, K, D] + search constants; row-level encode / decode."""

    def __init__(self, codebooks: Optional[torch.Tensor] = None, handle=None, owner=None, nq=None, D=None):
        self.lib = _lib.load()
        self.owner = owner
        if handle is not None:
            self.h, self.nq, self.D, self.owned = C.c_void_p(handle), nq, D, False
            return
        cb = codebooks.detach().float().contiguous()
        self.nq, K, self.D = cb.shape
        h = C.c_void_p()
        _lib.check(self.lib.qb_rvq_load(Context.get(cb.device).h, cb.data_ptr(), self.nq, K, self.D, C.byref(h)))
        self.h, self.owned = h, True

    def __del__(self):
        try:
            if getattr(self, "owned", False) and self.h:
                self.lib.qb_rvq_free(self.h)
                self.h = None
        except Exception:
            pass

    def encode_rows(self, x: torch.Tensor, want_quantized=True):
        x = x.float().contiguous()
        M = x.shape[0]
        idx = torch.empty(M, self.nq, dtype=torch.int64, device=x.device)
        quant = torch.empty(M, self.D, device=x.device) if want_quantized else None
        _lib.check(self.lib.qb_rvq_encode_rows(self.h, x.data_ptr(), M, idx.data_ptr(), quant.data_ptr() if quant is not None else None,
                                               _stream()))
        return idx, quant

    def decode_rows(self, idx: torch.Tensor):
        idx = idx.long().contiguous()
        out = torch.empty(idx.shape[0], self.D, device=idx.device)
        _lib.check(self.lib.qb_rvq_decode_rows(self.h, idx.data_ptr(), idx.shape[0], out.data_ptr(), _stream()))
        return out
