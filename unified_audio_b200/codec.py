"""H-Codec-2.0 `Codec` with the reference's surface, backed by the handle-level engine of libquark_b200.

Mirrors QuarkAudio-HCodec/HCodec-2.0/vq/codec.py:17-99:
    Codec(encoder_kwargs, decoder_kwargs, quantizer_kwargs, semantic_encoder_kwargs, semantic_decoder_kwargs)
    Codec.encode(x [B,T], feat [B,768,T50]) -> (acoustic_codes, semantic_codes)  int64 [B,nq,N]
    Codec.decode(acoustic_codes, semantic_codes)  -> wav [B, N*3840]
    Codec.forward(x, feat) -> (recon, pred_feat, commit_loss), evaluation mode, with semantic_decoder=True
state_dict keys/shapes are the reference's (spec.py); `semantic_decoder.*` keys (the module only forward calls, codec.py:71) are
accepted by load_state_dict and ignored unless the face is built with semantic_decoder=True.

`encode` / `decode` are one call each into the C ABI (csrc/engine.cu through engine.py): the engine owns the repacked
weights, the workspace and the ~340-kernel orchestration, with activations channel-last [B*T, C] end to end.  There is no
PyTorch / CPU fallback.  H-Codec-1.0 / 1.5 (codec_h1.py, codec_h15.py) launch their kernels op by op from Python instead;
they share `_CodecFace` with this class.  `_Face`, the base of every face of the package, is defined here too.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
from torch import nn

from . import ops, spec
from .rvq import ResidualVQ

# GEMM groups -> 3-term split (True) or single-pass fp16 (False).  Evidence: oracle/precision_study.py,
# DESIGN.md "precision policy".
PRECISION_POLICIES = {
    "mixed": dict(convnext=False, lstm_attn=False, mlp=True, mlp_dec=True, conv=True, head=True, dft=True),
    # decoder-side transformer MLP single-pass (it sits behind the RVQ indices, only the waveform budget applies):
    # measured on the shipped config 121.3 vs 125.4 ms per step, waveform error 6.5e-4 vs 2.3e-4 - inside 1e-3 but with
    # 1.5x instead of 4x margin, hence not the default
    "mixed_dec16": dict(convnext=False, lstm_attn=False, mlp=True, mlp_dec=False, conv=True, head=True, dft=True),
    "accurate": dict(convnext=True, lstm_attn=True, mlp=True, mlp_dec=True, conv=True, head=True, dft=True),
    "fast": dict(convnext=False, lstm_attn=False, mlp=False, mlp_dec=False, conv=False, head=False, dft=True),
}


class _Tree(nn.Module):
    """Bare parameter container whose nested attribute names reproduce the reference's module tree."""

    @staticmethod
    def build(specs: Dict[str, tuple]) -> "_Tree":
        root = _Tree()
        for name, shape in specs.items():
            node = root
            parts = name.split(".")
            for p in parts[:-1]:
                if p not in node._modules:
                    node.add_module(p, _Tree())
                node = node._modules[p]
            if name in spec.BUFFERS:
                node.register_buffer(parts[-1], torch.hann_window(shape[0]))
            else:
                node.register_parameter(parts[-1], nn.Parameter(torch.zeros(shape), requires_grad=False))
        return root


def _pad_to(n, m):
    return (n + m - 1) // m * m


class _Face(nn.Module):
    """What every face over libquark_b200 shares.  `_w` holds the weights prepared from the parameters (None = not prepared
    yet, or stale) and `_ws` the zero-initialised scratch buffers and shape-keyed tables.  Both are dropped whenever the
    parameters or the device change (`load_state_dict`, `.to()` / `.cuda()` / `.half()`); a face that derives more state
    from them drops it in `_drop_prepared`.  `load_state_dict` accepts the reference checkpoint's keys that the face does not
    hold (`_ignored_key`)."""

    _IGNORED_KEYS: tuple = ()          # checkpoint key prefixes accepted at load and not kept

    def __init__(self):
        super().__init__()
        self._w, self._ws = None, {}

    def _drop_prepared(self):
        self._w, self._ws = None, {}

    def _ignored_key(self, key: str) -> bool:
        return key.startswith(self._IGNORED_KEYS)

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        sd = {k: v for k, v in state_dict.items() if not self._ignored_key(k)}
        r = super().load_state_dict(sd, strict=strict, assign=assign)
        self._drop_prepared()
        return r

    def _apply(self, fn, *a, **k):
        self._drop_prepared()
        return super()._apply(fn, *a, **k)

    def _dev(self):
        return next(self.parameters()).device

    def _require_cuda(self):
        dev = self._dev()
        if dev.type != "cuda":
            raise RuntimeError(f"unified_audio_b200.{type(self).__name__} runs on CUDA only (no CPU fallback): call .cuda() first")
        return dev

    def _cached(self, key, build):
        """`_ws[key]`, built by `build()` on first use."""
        v = self._ws.get(key)
        if v is None:
            v = self._ws[key] = build()
        return v

    def _buf(self, name, shape, dtype=torch.float32):
        """Zero-initialised scratch tensor: kernels rely on the pad rows / columns they never write staying zero."""
        return self._cached(("buf", name, tuple(shape), dtype), lambda: torch.zeros(shape, dtype=dtype, device=self._dev()))

    def _planes(self, name, shape, split=True):
        """Zero-initialised fp16 hi (+ lo if `split`) planes."""
        return self._cached(("planes", name, tuple(shape), bool(split)), lambda: ops.Planes.zeros(shape, split, self._dev()))


class _CodecFace(_Face):
    """The codec faces add CUDA-graph capture, the encode -> decode round trip and the evaluation-mode `forward`.  Their
    checkpoints carry `semantic_decoder.*` (vq/semantic_module.py:252-299, which only `forward` calls): a face built with
    `semantic_decoder=True` holds those parameters under the reference's names and a strict load requires them; without it
    they are accepted at load and not kept, and `forward` is refused."""

    _IGNORED_KEYS = ("semantic_decoder.",)

    def _add_semantic_decoder(self, enabled: bool, kwargs: dict):
        """Decoder(**kwargs) of vq/semantic_module.py:252-292 as parameters, when `enabled`."""
        self.sem_dec_cfg = dict(kwargs) if enabled else None
        if enabled:
            self.semantic_decoder = _Tree.build(spec.semantic_decoder_spec(**kwargs))
            self._IGNORED_KEYS = ()

    def _check_forward(self):
        if self.sem_dec_cfg is None:
            raise RuntimeError(f"unified_audio_b200.{type(self).__name__}.forward needs the semantic decoder: construct the face with "
                               "semantic_decoder=True and load a checkpoint that carries semantic_decoder.*")
        if self.training:
            raise RuntimeError(f"unified_audio_b200.{type(self).__name__}.forward runs in evaluation mode only: call .eval() "
                               "(quantize dropout, codebook updates and gradients through the codec are not built)")

    def _commit_loss(self):
        """vector_quantize_pytorch's ResidualVQ returns zero commitment losses in eval mode (oracle/rvq.py states the same; the package
        itself is not pinned), so the reference's (commit_loss + commit_loss_semantic).mean() is a 0-d fp32 zero."""
        return torch.zeros((), dtype=torch.float32, device=self._dev())

    # ------------------------------------------------------------------ CUDA-graph replay of a fixed-shape call
    def graphed(self, fn_name: str, *example_inputs, warmup: int = 2) -> "GraphedCall":
        """Capture `encode`, `decode` or `roundtrip` (encode -> decode) for the shapes of `example_inputs` into ONE CUDA
        graph: a step is ~340 kernel launches, a third of them a few microseconds long (RVQ layers, norms, small GEMMs) -
        replaying the graph removes the host launch gaps.  Returns a callable taking tensors of the same shapes (device or
        pinned host; they are copied into the graph's static inputs) and returning the static output tensors."""
        fn = dict(encode=self.encode, decode=self.decode, roundtrip=self.roundtrip)[fn_name]
        return GraphedCall(fn, example_inputs, warmup)

    @torch.no_grad()
    def roundtrip(self, x, feat):
        """encode -> decode: (acoustic, semantic, reconstructed wav)."""
        ac, sc = self.encode(x, feat)
        return ac, sc, self.decode(ac, sc)

class Codec(_CodecFace):
    def __init__(self, encoder_kwargs: dict, decoder_kwargs: dict, quantizer_kwargs: dict,
                 semantic_encoder_kwargs: dict, semantic_decoder_kwargs: Optional[dict] = None,
                 precision: str = "mixed", semantic_decoder: bool = False):
        super().__init__()
        if semantic_decoder and not semantic_decoder_kwargs:
            raise ValueError("semantic_decoder=True needs semantic_decoder_kwargs (the reference's semantic_decoder_config)")
        if precision not in PRECISION_POLICIES:
            raise KeyError(f"unknown precision policy {precision!r} (one of {', '.join(PRECISION_POLICIES)})")
        self.enc_cfg, self.dec_cfg = dict(encoder_kwargs), dict(decoder_kwargs)
        self.sem_cfg = dict(semantic_encoder_kwargs)
        self.encoder = _Tree.build(spec.encoder_spec(**encoder_kwargs))
        self.decoder = _Tree.build(spec.decoder_spec(**decoder_kwargs))
        self.quantizer = ResidualVQ(**quantizer_kwargs)
        self.semantic_quantizer = ResidualVQ(**quantizer_kwargs)
        self.semantic_encoder = _Tree.build(spec.semantic_encoder_spec(**semantic_encoder_kwargs))
        self._add_semantic_decoder(semantic_decoder, semantic_decoder_kwargs or {})
        self.precision = precision
        self._engine = None
        self.eval()

    def _drop_prepared(self):
        super()._drop_prepared()
        self._engine = None

    def engine(self):
        """The qb_codec handle of this model (built lazily from the current parameters)."""
        if self._engine is None:
            from .engine import CodecEngine
            dev = self._require_cuda()
            sd = self.state_dict()
            self._engine = CodecEngine(dev, self.enc_cfg, self.dec_cfg, dict(num_quantizers=self.quantizer.num_quantizers,
                                                                             codebook_size=self.quantizer.codebook_size),
                                       self.sem_cfg, self.precision,
                                       {k: v for k, v in sd.items() if not k.startswith("semantic_decoder.")})
            if self.sem_dec_cfg is not None:
                self._engine.load_semantic_decoder(self.sem_dec_cfg, {k: v for k, v in sd.items() if k.startswith("semantic_decoder.")})
        return self._engine

    @torch.no_grad()
    def encode(self, x, feat, taps=None):
        """vq/codec.py:75-87: x [B,T] fp32, feat [B,768,T/960] fp32 -> (acoustic, semantic) int64 [B,nq,N]."""
        eng = self.engine()
        if taps is None:
            return eng.encode(x, feat)
        eng.set_taps(taps)
        try:
            return eng.encode(x, feat)
        finally:
            eng.set_taps(None)

    @torch.no_grad()
    def decode(self, acoustic_codes, semantic_codes, taps=None):
        """vq/codec.py:89-99: int64 [B,nq,N] x2 -> wav [B, N*3840]."""
        eng = self.engine()
        if taps is None:
            return eng.decode(acoustic_codes, semantic_codes)
        eng.set_taps(taps)
        try:
            return eng.decode(acoustic_codes, semantic_codes)
        finally:
            eng.set_taps(None)

    @torch.no_grad()
    def semantic_decode(self, semantic_codes):
        """vq/codec.py:71 on the codes' quantised rows: int64 [B,nq,N] -> pred_feat fp32 [B, output_channels, N*prod(strides)]
        (one qb_codec_semantic_decode).  Needs semantic_decoder=True."""
        if self.sem_dec_cfg is None:
            raise RuntimeError("Codec.semantic_decode needs the semantic decoder: construct the face with semantic_decoder=True")
        return self.engine().semantic_decode(semantic_codes)

    def forward(self, x, feat):
        """vq/codec.py:54-72 in evaluation mode: (recon [B, T], pred_feat fp32 [B, C_ssl, T_feat], commit_loss 0-d fp32).  recon is
        decode(*encode(x, feat)) - the reference's quantised sum of codebook rows is get_output_from_indices(codes) - and pred_feat
        the semantic decoder on the semantic stream's codebook rows."""
        self._check_forward()
        with torch.no_grad():
            ac, sc = self.encode(x, feat)
            return self.decode(ac, sc), self.semantic_decode(sc), self._commit_loss()


class GraphedCall:
    """A fixed-shape call captured in a CUDA graph (static input / output buffers, `torch.cuda.graphs`)."""

    def __init__(self, fn, example_inputs, warmup: int = 2):
        self.inputs = [t.detach().to("cuda", copy=True) for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):              # warm-up off the capture: lazy weight preparation, workspaces, attributes
            for _ in range(max(warmup, 1)):
                fn(*self.inputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        n0 = ops.launch_count()
        with torch.cuda.graph(self.graph):
            self.outputs = fn(*self.inputs)
        self.launches_per_replay = ops.launch_count() - n0      # library kernels recorded in the graph

    def __call__(self, *inputs):
        if inputs:
            if len(inputs) != len(self.inputs):
                raise ValueError("graphed call: wrong number of inputs")
            for dst, src in zip(self.inputs, inputs):
                if src.shape != dst.shape or src.dtype != dst.dtype:
                    raise ValueError(f"graphed call captured for {tuple(dst.shape)} {dst.dtype}, got {tuple(src.shape)} {src.dtype}")
                if src.data_ptr() != dst.data_ptr():
                    dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.outputs

    # ------------------------------------------------------------------ streaming host I/O
    def stream(self, host_inputs, host_outputs):
        """One step of a serving loop with HOST tensors on both sides, copies overlapped with compute: the H2D copy of this step's
        (pinned) inputs runs on a copy stream into a staging buffer while the previous step still computes; the step itself is a
        device-to-device move into the graph's static inputs + the replay + a device-to-device move of its outputs into a second
        staging buffer, from which the copy stream drains them into `host_outputs` (pinned) under the next step.  Call
        `finish()` (or torch.cuda.synchronize()) before reading `host_outputs` of the last step."""
        cur = torch.cuda.current_stream()
        if getattr(self, "_io", None) is None:
            outs = self.outputs if isinstance(self.outputs, (tuple, list)) else (self.outputs,)
            # two copy streams: on one, the H2D of step i + 1 would queue behind the D2H of step i, which waits for step i's compute
            self._io = dict(stream=torch.cuda.Stream(), d2h_stream=torch.cuda.Stream(), in_stage=[torch.empty_like(t) for t in self.inputs],
                            out_stage=[torch.empty_like(t) for t in outs], h2d=torch.cuda.Event(), staged=torch.cuda.Event(),
                            consumed=torch.cuda.Event(), drained=torch.cuda.Event())
            self._io["consumed"].record(cur)
            self._io["drained"].record(cur)
        io = self._io
        with torch.cuda.stream(io["stream"]):
            io["stream"].wait_event(io["consumed"])            # the previous step has moved its inputs out of the staging buffer
            for dst, src in zip(io["in_stage"], host_inputs):
                dst.copy_(src, non_blocking=True)
            io["h2d"].record(io["stream"])
        cur.wait_event(io["h2d"])
        for dst, src in zip(self.inputs, io["in_stage"]):
            dst.copy_(src, non_blocking=True)
        io["consumed"].record(cur)
        self.graph.replay()
        outs = self.outputs if isinstance(self.outputs, (tuple, list)) else (self.outputs,)
        cur.wait_event(io["drained"])                           # the previous step's outputs have left the staging buffer
        for dst, src in zip(io["out_stage"], outs):
            dst.copy_(src, non_blocking=True)
        io["staged"].record(cur)
        with torch.cuda.stream(io["d2h_stream"]):
            io["d2h_stream"].wait_event(io["staged"])
            for dst, src in zip(host_outputs, io["out_stage"]):
                dst.copy_(src, non_blocking=True)
            io["drained"].record(io["d2h_stream"])

    def finish(self):
        if getattr(self, "_io", None) is not None:
            torch.cuda.current_stream().wait_event(self._io["drained"])
