"""UniSE inference and validation surface (`Model.test_step`, `Model.validation_step`) on the device: the callers of the AR-LM hot path.

Mirrors QuarkAudio-UniSE/model/model.py:20-286 (a LightningModule in the reference; a plain nn.Module here - the Lightning task
and checkpoint callbacks are out of scope, SURVEY 2):
    Model(config, tokenizer=BiCodecTokenizer(BiCodec), dnn=LLM_SFT, semantic_model=SSLFrontEnd(WAVLM_BASE_PLUS))
    .extract_semantic_features(wavs [B, T] @ 16 kHz) -> [B, T/320, 768]        model.py:37-51
    .stft_logmel(x [B, T]) -> [B, ceil(T/320), 80]                               model.py:53-79
    .validation_step((mode, enroll, mix, speech, interf, fs, lengths, names))    model.py:134-160, modes 'se' / 'tse' / 'rtse'
    .validation_epoch(batches) -> batch-size-weighted epoch means, across ranks   model.py:160 (log_dict on_epoch, sync_dist)
    .training_step(batch) -> {"loss" (differentiable), "train_acc"}, .configure_optimizers()   model.py:96-124, 327-353
    .broadcast_parameters(), .sync_gradients()    data-parallel training as train.py:35's DDP strategy averages gradients
    .test_step((mode, enroll, src, tgt, fs, lengths, names), batch_idx)          model.py:170-286, modes 'se' / 'tse' / 'ss'
and audio_tokenizer.py:30-125 for `BiCodecTokenizer.detokenize(global_tokens, semantic_tokens)` and, given the wav2vec2 front end,
`BiCodecTokenizer.tokenize(wav) -> (global_tokens, semantic_tokens)`.

Everything between the waveform in and the waveform out stays on the GPU: wrap-pad + 5 s segmenting (`qb_pad_wav`, no NumPy round
trip), WavLM features (csrc/ssl.cu + the conv-GEMM / attention kernels), `LLM_SFT.generate` (csrc/llm.cu), `BiCodec.detokenize`.
`stft_logmel` is dead compute on this path - `generate` reads only `mix_mel.size(1)` (llm_sft.py:166) - so `test_step` hands the LM a
shape-only tensor (`mel_like`); `stft_logmel` itself is provided for callers that want the values (torch.stft: plumbing, not a kernel
of this library).  No CPU fallback: the three sub-modules refuse to run off the GPU.
"""
from __future__ import annotations

import math
import os
from typing import Optional

import torch
from torch import nn

from . import ops
from .ssl import wrap_segments

STFT_CONFIG = dict(hop_length=320, win_length=640, n_fft=640, n_mels=80)      # U/conf/config.yaml:124-128
SEG_LEN = 5 * 16000                                                            # model.py:175
# 5 s segments that go through WavLM / generate / detokenize together in Model.enhance_batch.  The faces keep their scratch buffers
# per shape, and at shipped widths 128 segments per call ran out of an 80 GB H100 (in the BiCodec decoder's buffers); 32 is one LM
# decode chunk.  Measured peak device memory: README (scripts/unise_enhance_bench.py).
MAX_SEGMENTS = 32
# the generate passes of test_step (model.py:174-286): 'se', 'tse', and in 'ss' an 'se' pass followed by 'tse' and 'rtse'
GENERATE_PASSES = ("se", "tse", "rtse")
_M64 = (1 << 64) - 1


def _mix64(z: int) -> int:
    """SplitMix64's finaliser (Steele, Lea and Flood 2014): a bijection of 64-bit ints"""
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def segment_key(utterance_seed: int, generate_pass: str, segment: int) -> int:
    """The 64-bit key of one generate row of a sampled `Model.enhance` / `enhance_batch` (LLM_SFT.generate's `row_seeds`): a pure
    function of the utterance's seed, the generate pass ('se', 'tse' or 'rtse') and the row's 5 s segment index in that pass,
        h = mix64((utterance_seed + G) mod 2^64);  then h = mix64(((h XOR x) + G) mod 2^64) for x = the pass index (se 0, tse 1,
        rtse 2), then for x = the segment,
    with mix64 SplitMix64's finaliser and G = 0x9E3779B97F4A7C15.  'ss' draws its first pass (one row: the first 5 s) as 'se'
    segment 0."""
    if generate_pass not in GENERATE_PASSES:
        raise ValueError(f"generate_pass must be one of {GENERATE_PASSES}, got {generate_pass!r}")
    if segment < 0:
        raise ValueError(f"segment must be >= 0, got {segment}")
    G = 0x9E3779B97F4A7C15
    h = _mix64((int(utterance_seed) + G) & _M64)
    for x in (GENERATE_PASSES.index(generate_pass), int(segment)):
        h = _mix64(((h ^ x) + G) & _M64)
    return h


class BiCodecTokenizer(nn.Module):
    """audio_tokenizer.py:30-125.  `tokenize` (UniSE tokenizes clean speech with it, model.py:96-102,134-140) needs the wav2vec2
    front end, `feature_extractor` = SSLFrontEnd(WAV2VEC2_XLSR53) (extract_wav2vec2_features, audio_tokenizer.py:74-90), and a
    BiCodec built with global_tokens=True and semantic_tokens=True; without them it raises NotImplementedError.  detokenize needs
    neither.  ref_segment_length = int(sample_rate * ref_segment_duration) // latent_hop_length * latent_hop_length
    (audio_tokenizer.py:60-64): 96000 for the published 16 kHz, 6 s, 320-sample configuration."""

    def __init__(self, model, ref_segment_length: int = 96000, feature_extractor: Optional[nn.Module] = None):
        super().__init__()
        self.model = model
        self.ref_segment_length = int(ref_segment_length)
        self.feature_extractor = feature_extractor

    @torch.no_grad()
    def get_ref_clip(self, wav: torch.Tensor) -> torch.Tensor:
        """audio_tokenizer.py:54-72: wav [B, L] -> [B, ref_segment_length]; a shorter wav is repeated (torch.tile) and cut, i.e.
        wrap-padded on the device (`qb_pad_wav`)."""
        if wav.device.type != "cuda":
            raise RuntimeError("unified_audio_b200.unise.BiCodecTokenizer runs on CUDA only (no CPU fallback)")
        if wav.ndim != 2:
            raise ValueError("wav must be [B, L]")
        n = self.ref_segment_length
        if n > wav.shape[-1]:
            return ops.pad_wav(wav, 0, n, wrap=True)
        return wav[:, :n].float().contiguous()

    def require_tokenize(self) -> None:
        """Raise the NotImplementedError `tokenize` raises when this tokenizer cannot tokenize; it names what is missing."""
        missing = [] if self.feature_extractor is not None else ["a feature_extractor (SSLFrontEnd(WAV2VEC2_XLSR53))"]
        missing += [f"BiCodec(..., {f}=True)" for f in ("global_tokens", "semantic_tokens") if not getattr(self.model, f, False)]
        if missing:
            raise NotImplementedError("BiCodecTokenizer.tokenize needs " + " and ".join(missing))

    @torch.no_grad()
    def tokenize(self, wav: torch.Tensor):
        """audio_tokenizer.py:92-105: wav [B, L] @ 16 kHz -> (global_tokens int32 [B, 1, token_num], semantic_tokens int64 [B, T']),
        the reference's order; everything stays on the device."""
        self.require_tokenize()
        if wav.device.type != "cuda":
            raise RuntimeError("unified_audio_b200.unise.BiCodecTokenizer runs on CUDA only (no CPU fallback)")
        ref_wav = self.get_ref_clip(wav)
        feat = self.feature_extractor(wav)
        semantic_tokens, global_tokens = self.model.tokenize({"wav": wav, "ref_wav": ref_wav, "feat": feat})
        return global_tokens, semantic_tokens

    @torch.no_grad()
    def detokenize(self, global_tokens: torch.Tensor, semantic_tokens: torch.Tensor) -> torch.Tensor:
        """global_tokens [B, 1, 32], semantic_tokens [B, T] -> wav [B, 1, T * 320]   (audio_tokenizer.py:108-125)"""
        return self.model.detokenize(semantic_tokens, global_tokens)


class Model(nn.Module):
    def __init__(self, config: Optional[dict] = None, *, tokenizer: BiCodecTokenizer, dnn, semantic_model):
        super().__init__()
        self.config = dict(config or {})
        self.stft_conf = dict(self.config.get("stft_config", STFT_CONFIG))
        self.tokenizer, self.dnn, self.semantic_model = tokenizer, dnn, semantic_model

    # ------------------------------------------------------------------ state (model.py:81-91): tokenizer / semantic_model excluded
    def state_dict(self, *args, **kwargs):
        state = super().state_dict(*args, **kwargs)
        for key in list(state.keys()):
            if key.startswith(("tokenizer.", "semantic_model.")):
                del state[key]
        return state

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        """A Lightning checkpoint's `state_dict` holds the LM under `dnn.` (model.py:28)."""
        sd = {k[4:]: v for k, v in state_dict.items() if k.startswith("dnn.")}
        return self.dnn.load_state_dict(sd, strict=False)

    # ------------------------------------------------------------------ features
    @torch.no_grad()
    def extract_semantic_features(self, wavs: torch.Tensor) -> torch.Tensor:
        """model.py:37-51: pad 160 / 160, WavLM-base-plus, mean of the 13 hidden states (no compression)."""
        return self.semantic_model(wavs)

    def mel_frames(self, n_samples: int) -> int:
        return math.ceil(n_samples / self.stft_conf["hop_length"])

    def mel_like(self, x: torch.Tensor) -> torch.Tensor:
        """A tensor with stft_logmel's shape and no arithmetic behind it: the LM reads `mix_mel.size(1)` only (llm_sft.py:166)."""
        return torch.zeros(1, device=x.device).expand(x.shape[0], self.mel_frames(x.shape[-1]), self.stft_conf["n_mels"])

    @torch.no_grad()
    def stft_logmel(self, x: torch.Tensor) -> torch.Tensor:
        """model.py:53-79 verbatim in meaning (torch.stft + HTK mel filter bank + log); not on the generate path (see module doc)."""
        from torchaudio.functional import melscale_fbanks
        if x.ndim != 2:
            raise AssertionError("x: (B, T)")
        hop, win, n_fft, n_mels = (self.stft_conf[k] for k in ("hop_length", "win_length", "n_fft", "n_mels"))
        pad_length = math.ceil(x.size(-1) / hop) * hop - x.size(-1)
        x = torch.nn.functional.pad(x, ((win - hop) // 2, pad_length + (win - hop) // 2))
        spec = torch.stft(x, n_fft, hop, win_length=win, window=torch.hann_window(win).to(x.device), onesided=True, center=False,
                          return_complex=True).transpose(1, 2)
        if not hasattr(self, "fb"):
            self.fb = melscale_fbanks(n_freqs=n_fft // 2 + 1, f_min=0.0, f_max=8000.0, n_mels=n_mels, sample_rate=16000).to(x.device)
        return torch.log(spec.abs() @ self.fb + 1e-10)

    def forward(self, batch):
        """model.py:93-94: the reference's forward is empty; inference goes through test_step."""
        return None

    # ------------------------------------------------------------------ validation (model.py:134-160)
    @staticmethod
    def _validation_inputs(batch):
        """batch -> (mode, enroll, mix, the waveform the mode tokenizes: `interf` for 'rtse', `speech` otherwise, model.py:137-140).
        Refuses what the reference would only fail on later, inside the tokenizer or the LM."""
        mode, enroll, mix, speech, interf, fs, lengths, names = batch
        if mode not in ("se", "tse", "rtse"):
            raise ValueError(f"unknown mode {mode!r} (the reference's validation_step handles 'se', 'tse', 'rtse')")
        name = "interf" if mode == "rtse" else "speech"
        wav = interf if mode == "rtse" else speech
        if wav is None:
            raise ValueError(f"mode {mode!r} tokenizes `{name}`, which is None")
        sizes = {"mix": mix.shape[0], name: wav.shape[0]}
        if enroll is not None:
            sizes["enroll"] = enroll.shape[0]
        if len(set(sizes.values())) > 1:
            raise ValueError(f"batch sizes differ: {sizes}")
        return mode, enroll, mix, wav

    @torch.no_grad()
    def validation_step(self, batch, batch_idx=0):
        """model.py:134-160: batch = (mode, enroll, mix, speech, interf, fs, lengths, names) on the device, mode 'se' / 'tse' / 'rtse'.
        Tokenizes `speech` ('se', 'tse') or `interf` ('rtse') with `BiCodecTokenizer.tokenize`, extracts WavLM features of `mix` and,
        when `enroll` is not None, of `enroll` (which then joins the LM prefix), and runs the teacher-forced `LLM_SFT.forward`.
        Returns {"valid_loss", "valid_acc"}: 0-d fp32 device tensors, what the reference logs; no host synchronisation.

        The reference's log-mels (`stft_logmel` of mix and enroll) are dead compute here: `LLM_SFT.forward` reads only the mix mel's
        batch size and device (llm_sft.py:60) and whether the enrollment mel is None, so the step passes shape-only tensors
        (`mel_like`), as `test_step` does.  `semantic_tokens` keep wav2vec2's unpadded length (80 000 samples -> 249 tokens) while the
        WavLM features of `mix` are padded 160 / 160 (-> 250 frames); nothing assumes the two are equal."""
        self.tokenizer.require_tokenize()
        _, enroll, mix, wav = self._validation_inputs(batch)
        if any(t is not None and t.device.type != "cuda" for t in (enroll, mix, wav)):
            raise RuntimeError("unified_audio_b200.unise.Model runs on CUDA only (no CPU fallback)")
        return self._validation_step(batch)

    def _validation_step(self, batch):
        """validation_step's control flow (model.py:135-160) over the three components; pinned against the reference's own
        `validation_step` driven with stand-ins (oracle/make_golden_unise_validation.py -> tests/golden/unise_validation_glue.npz)."""
        mode, enroll, mix, wav = self._validation_inputs(batch)
        global_tokens, semantic_tokens = self.tokenizer.tokenize(wav)
        mix_feats = self.extract_semantic_features(mix)
        enroll_mel = enroll_feats = None
        if enroll is not None:
            enroll_mel, enroll_feats = self.mel_like(enroll), self.extract_semantic_features(enroll)
        loss, acc = self.dnn(task_name=mode, enroll_mel=enroll_mel, enroll_feats=enroll_feats, mix_mel=self.mel_like(mix),
                             mix_feats=mix_feats, global_ids=global_tokens.squeeze(1), semantic_ids=semantic_tokens)
        return {"valid_loss": loss, "valid_acc": acc}

    # ------------------------------------------------------------------ training (model.py:96-124, 327-353)
    def training_step(self, batch, batch_idx=0, dropout_seed: Optional[int] = None):
        """model.py:96-124: the composition of validation_step (same inputs, same checks) with the LM in train mode, so its attention
        dropout (llm_base_config["dropout_p"]) applies.  The tokenizer and WavLM run frozen, without autograd, in whatever mode they
        are in (eval unless the caller changed it), as validation_step runs them.  Returns {"loss", "train_acc"}: `loss` carries the
        LM's grad_fn, so `loss.backward()` fills the `.grad` of `dnn`'s parameters once they require grad (`configure_optimizers`
        turns that on).  The LM's previous mode is restored before returning."""
        self.tokenizer.require_tokenize()
        mode, enroll, mix, wav = self._validation_inputs(batch)
        if any(t is not None and t.device.type != "cuda" for t in (enroll, mix, wav)):
            raise RuntimeError("unified_audio_b200.unise.Model runs on CUDA only (no CPU fallback)")
        global_tokens, semantic_tokens = self.tokenizer.tokenize(wav)
        mix_feats = self.extract_semantic_features(mix)
        enroll_mel = enroll_feats = None
        if enroll is not None:
            enroll_mel, enroll_feats = self.mel_like(enroll), self.extract_semantic_features(enroll)
        was_training = self.dnn.training
        self.dnn.train()
        try:
            loss, acc = self.dnn(task_name=mode, enroll_mel=enroll_mel, enroll_feats=enroll_feats, mix_mel=self.mel_like(mix),
                                 mix_feats=mix_feats, global_ids=global_tokens.squeeze(1), semantic_ids=semantic_tokens,
                                 dropout_seed=dropout_seed)
        finally:
            self.dnn.train(was_training)
        return {"loss": loss, "train_acc": acc}

    def configure_optimizers(self):
        """model.py:327-353: AdamW over the LM's parameters with config["opt"], and a per-step LambdaLR: cosine warm-up over
        sch.warmup_steps, then step_decay ** (step - warmup_steps) floored at sch.min_factor.  Makes the LM's parameters require
        grad first.  Returns ([optimizer], [{"scheduler", "interval": "step", "frequency": 1}]) as the reference does."""
        self.dnn.requires_grad_(True)
        opt = torch.optim.AdamW(self.dnn.parameters(), **self.config["opt"])
        sch_cfg = self.config["sch"]

        def warmup_lambda(step):
            warmup_steps, step_decay = sch_cfg["warmup_steps"], sch_cfg["step_decay"]
            if step < warmup_steps:
                return 0.5 * (1 + math.cos(math.pi * (1 - step / warmup_steps)))
            return max(step_decay ** (step - warmup_steps), sch_cfg["min_factor"])

        sch = {"scheduler": torch.optim.lr_scheduler.LambdaLR(opt, warmup_lambda), "interval": "step", "frequency": 1}
        return [opt], [sch]

    # ------------------------------------------------------------------ data-parallel training (train.py:35, strategy 'ddp')
    def broadcast_parameters(self, group=None) -> None:
        """Copy rank 0's LM parameters to every rank of `group` (`parallel.broadcast_parameters`), as DDP does when it wraps the
        model; the LM repacks its inference weights at its next call.  No-op without torch.distributed or with one rank."""
        from .parallel import broadcast_parameters
        broadcast_parameters(self.dnn, group)

    def sync_gradients(self, group=None) -> None:
        """Average the LM's gradients across the ranks of `group` with one all-reduce (`parallel.average_gradients`): what DDP with
        find_unused_parameters=True leaves in `.grad`, including `.grad is None` on a parameter no rank used (`enroll_sos_embedding`
        when every rank ran 'se').  Call it after `loss.backward()` and before clipping; every rank then holds the same gradients,
        so clipping and the optimizer step keep the ranks' parameters equal.  No-op without torch.distributed or with one rank."""
        from .parallel import average_gradients
        average_gradients(self.dnn, group)

    def validation_epoch(self, batches, group=None) -> dict:
        """A validation epoch as the reference logs it (`log_dict(..., on_epoch=True, sync_dist=True)`, model.py:160).  Each batch's
        tensors are moved to the LM's device and scored by `validation_step`.  Running sums of B·loss, B·acc and B (B = the batch's
        clip count) stay on the device in fp64; when torch.distributed is initialised they are summed across the ranks of `group`
        with one all_reduce (`parallel.all_reduce_sum`), and read on the host once, at the end.
        Returns {"valid_loss": Σ B·loss / Σ B, "valid_acc": Σ B·acc / Σ B} as floats, over every batch of every rank."""
        from .parallel import all_reduce_sum
        dev = next(self.dnn.parameters()).device
        sums = torch.zeros(3, dtype=torch.float64, device=dev)
        n = 0
        for i, batch in enumerate(batches):
            batch = tuple(x.to(dev, non_blocking=True) if torch.is_tensor(x) else x for x in batch)
            out = self.validation_step(batch, i)
            b = batch[2].shape[0]
            sums[:2] += b * torch.stack((out["valid_loss"], out["valid_acc"])).double()
            n += b
        sums[2] = n
        loss, acc, total = all_reduce_sum(sums, group).tolist()
        if total == 0:
            raise ValueError("validation_epoch: no batch on any rank")
        return {"valid_loss": loss / total, "valid_acc": acc / total}

    # ------------------------------------------------------------------ inference (model.py:170-286)
    def _segments(self, src: torch.Tensor) -> torch.Tensor:
        return wrap_segments(src.float().contiguous(), SEG_LEN)          # np.pad(..., 'wrap') + reshape(-1, seg_len) on the device

    def _generate(self, task, enroll_feats, seg_src, do_sample, utterance_seed=None, **gen_kw):
        if enroll_feats is not None:                                    # torch.cat([enroll] * n_segments) (model.py:207-208)
            n = seg_src.size(0)
            enroll_feats = torch.cat([enroll_feats for _ in range(n)], 0)
        if utterance_seed is not None:
            gen_kw = dict(gen_kw, row_seeds=[segment_key(utterance_seed, task, i) for i in range(seg_src.size(0))])
        return self._generate_rows(task, enroll_feats, None, seg_src, do_sample, **gen_kw)

    @staticmethod
    def _check_seed_args(gen_kw, name):
        if "seed" in gen_kw or "row_seeds" in gen_kw:
            raise ValueError(f"`{name}` sets generate's random streams: it cannot be combined with `seed` / `row_seeds`")

    def _generate_rows(self, task, enroll_feats, enroll_lengths, seg_src, do_sample, **gen_kw):
        """WavLM features of the segments, then generate with one enrollment row per segment (right-padded to the longest when
        `enroll_lengths` is given)"""
        mix_mel = self.mel_like(seg_src)
        mix_feats = self.extract_semantic_features(seg_src)
        enroll_mel = None
        if enroll_feats is not None:
            enroll_mel = mix_mel            # placeholder: only `is None` is tested for the enrollment mel (llm_sft.py:110-121)
        if enroll_lengths is not None:
            gen_kw = dict(gen_kw, enroll_lengths=enroll_lengths)
        gids, sids = self.dnn.generate(task_name=task, enroll_mel=enroll_mel, enroll_feats=enroll_feats, mix_mel=mix_mel,
                                       mix_feats=mix_feats, do_sample=do_sample, **gen_kw)
        return gids, sids

    def _detok(self, gids, sids, n_samples):
        est = self.tokenizer.detokenize(gids.unsqueeze(1), sids).squeeze(1)          # (B, t)
        return est.reshape(-1)[:n_samples]

    @torch.no_grad()
    def enhance(self, mode: str, enroll: Optional[torch.Tensor], src: torch.Tensor, do_sample: bool = False, return_ids: bool = False,
                utterance_seed: Optional[int] = None, **gen_kw):
        """The body of test_step with tensors in and a device tensor out.  src [1, T] (the reference's test loader yields one
        utterance per batch; like the reference, a batch of several is folded into the segment axis), enroll [1, Te] for 'tse'.
        'ss' returns (s1, s2).

        `utterance_seed` (with do_sample=True; not together with `seed` / `row_seeds` in gen_kw): every generate row draws from
        its own stream, keyed `segment_key(utterance_seed, pass, segment)`, so `enhance_batch` with this seed for the utterance
        returns the same result.  Greedy decoding ignores it."""
        if src.device.type != "cuda":
            raise RuntimeError("unified_audio_b200.unise.Model runs on CUDA only (no CPU fallback)")
        if utterance_seed is not None:
            self._check_seed_args(gen_kw, "utterance_seed")
            gen_kw = dict(gen_kw, utterance_seed=int(utterance_seed))
        return self._enhance(mode, enroll, src, do_sample, return_ids, **gen_kw)

    def _enhance(self, mode, enroll, src, do_sample=False, return_ids=False, **gen_kw):
        """test_step's control flow (model.py:174-286) over the four components; pinned against the reference's own `test_step`
        driven with stub components (oracle/make_golden_unise.py -> tests/golden/unise_glue.npz, tests/test_host.py)."""
        n_samples = src.size(-1)
        if mode == "se":                                                 # model.py:174-193
            seg = self._segments(src)
            seg = seg / src.abs().max(dim=-1, keepdim=True)[0]
            gids, sids = self._generate("se", None, seg, do_sample, **gen_kw)
            est = self._detok(gids, sids, n_samples)
            return (est, gids, sids) if return_ids else est
        if mode == "tse":                                                # model.py:197-224
            seg = self._segments(src)
            enroll_feats = self.extract_semantic_features(enroll)
            gids, sids = self._generate("tse", enroll_feats, seg, do_sample, **gen_kw)
            est = self._detok(gids, sids, n_samples)
            return (est, gids, sids) if return_ids else est
        if mode == "ss":                                                 # model.py:225-286: se on the first 5 s, then tse, then rtse
            first = src[:, :SEG_LEN] if n_samples > SEG_LEN else self._segments(src)[:src.size(0)]
            gids, sids = self._generate("se", None, first, do_sample, **gen_kw)
            enr = self.tokenizer.detokenize(gids.unsqueeze(1), sids).squeeze(1)[:, :SEG_LEN]
            enr = enr / (torch.max(torch.abs(enr)) + 1e-5) * 0.99
            enroll_feats = self.extract_semantic_features(enr)
            seg = self._segments(src)
            g1, s1 = self._generate("tse", enroll_feats, seg, do_sample, **gen_kw)
            est1 = self._detok(g1, s1, n_samples)
            g2, s2 = self._generate("rtse", enroll_feats, seg, do_sample, **gen_kw)
            est2 = self._detok(g2, s2, n_samples)
            return est1, est2
        raise ValueError(f"unknown mode {mode!r} (the reference's test_step handles 'se', 'tse', 'ss')")

    # ------------------------------------------------------------------ batched inference: many utterances per call
    @torch.no_grad()
    def enhance_batch(self, mode: str, enrolls, srcs, do_sample: bool = False, return_ids: bool = False,
                      max_segments: int = MAX_SEGMENTS, utterance_seeds=None, **gen_kw):
        """`enhance` over many utterances at once: srcs = list of [1, T_u] device tensors (any lengths), enrolls = list of [1, Te_u]
        ('tse', any lengths) or None.  Returns a list with, for each utterance, what `enhance` returns for it alone.

        Each utterance keeps its own wrap padding, its own 'se' peak normalisation and its own enrollment; their 5 s segments then
        share the WavLM / generate / detokenize calls, at most `max_segments` segments per call.  In 'tse' each enrollment's WavLM
        features are taken alone (WavLM's first GroupNorm spans time: padding would change them) and the LM prefixes differ in length
        (generate's `enroll_lengths`).  Greedy tokens are those of `enhance` when the LM's decode attention keeps the same number of
        keys in flight on both sides (LLM_SFT.att_unroll / lane_att_unroll; lanes only run when generate gets more than 32 rows).

        With do_sample, `utterance_seeds` (one int per utterance) gives every generate row its own random stream, keyed
        `segment_key(utterance_seeds[u], pass, segment)`: each utterance then gets exactly what `enhance(..., do_sample=True,
        utterance_seed=utterance_seeds[u])` gives it alone (same condition on the decode attention).  Without it the draws
        differ from `enhance`'s: with `seed` a row's uniforms depend on where it sits in the batch."""
        srcs = list(srcs) if srcs is not None else []
        if any(t is not None and t.device.type != "cuda" for t in srcs + list(enrolls or [])):
            raise RuntimeError("unified_audio_b200.unise.Model runs on CUDA only (no CPU fallback)")
        return self._enhance_batch(mode, enrolls, srcs, do_sample, return_ids, max_segments, utterance_seeds, **gen_kw)

    @staticmethod
    def _check_batch(mode, enrolls, srcs, max_segments):
        if mode not in ("se", "tse", "ss"):
            raise ValueError(f"unknown mode {mode!r} (the reference's test_step handles 'se', 'tse', 'ss')")
        if not srcs:
            raise ValueError("enhance_batch: no utterance")
        if any(s.ndim != 2 or s.shape[0] != 1 or s.shape[1] < 1 for s in srcs):
            raise ValueError(f"enhance_batch: every src must be [1, T], got {[tuple(s.shape) for s in srcs]}")
        if mode == "tse" and enrolls is None:
            raise ValueError("'tse' needs one enrollment per utterance")
        if enrolls is not None:
            enrolls = list(enrolls)
            if len(enrolls) != len(srcs):
                raise ValueError(f"{len(enrolls)} enrollments for {len(srcs)} utterances")
            if mode == "tse" and any(e.ndim != 2 or e.shape[0] != 1 or e.shape[1] < 1 for e in enrolls):
                raise ValueError(f"enhance_batch: every enrollment must be [1, Te], got {[tuple(e.shape) for e in enrolls]}")
        if max_segments < 1:
            raise ValueError(f"max_segments must be >= 1, got {max_segments}")
        return enrolls

    def _enhance_batch(self, mode, enrolls, srcs, do_sample=False, return_ids=False, max_segments=MAX_SEGMENTS, utterance_seeds=None,
                       **gen_kw):
        """_enhance's control flow per mode (model.py:174-286), applied per utterance, with the segments of all utterances batched;
        pinned against the reference's `test_step` fixture and against `_enhance` (tests/test_unise_batch_host.py)."""
        enrolls = self._check_batch(mode, enrolls, srcs, max_segments)
        if utterance_seeds is not None:
            utterance_seeds = [int(s) for s in utterance_seeds]
            if len(utterance_seeds) != len(srcs):
                raise ValueError(f"{len(utterance_seeds)} utterance_seeds for {len(srcs)} utterances")
            self._check_seed_args(gen_kw, "utterance_seeds")
        lens = [s.size(-1) for s in srcs]
        segs = [self._segments(s) for s in srcs]
        rows = [0]
        for sg in segs:
            rows.append(rows[-1] + sg.size(0))

        def keyed(task, n_rows=None):      # generate's keyword arguments for one pass: row u's segments keyed by its utterance's seed
            if utterance_seeds is None:
                return gen_kw
            n_rows = n_rows or [rows[u + 1] - rows[u] for u in range(len(srcs))]
            return dict(gen_kw, row_seeds=[segment_key(s, task, i) for s, n in zip(utterance_seeds, n_rows) for i in range(n)])
        cut = lambda x, u: x[rows[u]:rows[u + 1]]
        trim = lambda est, u: cut(est, u).reshape(-1)[:lens[u]]
        if mode == "se":                                                 # model.py:174-193, per utterance its own peak
            seg = torch.cat([sg / s.abs().max(dim=-1, keepdim=True)[0] for sg, s in zip(segs, srcs)], 0)
            est, gids, sids = self._run_segments("se", None, None, seg, do_sample, max_segments, **keyed("se"))
            return [(trim(est, u), cut(gids, u), cut(sids, u)) if return_ids else trim(est, u) for u in range(len(srcs))]
        if mode == "tse":                                                # model.py:197-224
            feats = [self.extract_semantic_features(e) for e in enrolls]          # each enrollment alone
            te = [f.size(1) for f in feats]
            pad = feats[0].new_zeros(1, max(te), feats[0].size(2))
            per_row = [torch.cat([f, pad[:, :max(te) - f.size(1)]], 1) for f in feats]
            ef = torch.cat([per_row[u] for u in range(len(srcs)) for _ in range(rows[u + 1] - rows[u])], 0)
            el = [te[u] for u in range(len(srcs)) for _ in range(rows[u + 1] - rows[u])]
            est, gids, sids = self._run_segments("tse", ef, el, torch.cat(segs, 0), do_sample, max_segments, **keyed("tse"))
            return [(trim(est, u), cut(gids, u), cut(sids, u)) if return_ids else trim(est, u) for u in range(len(srcs))]
        # 'ss', model.py:225-286: se on each utterance's first 5 s, then tse and rtse with that as the enrollment
        first = torch.cat([s[:, :SEG_LEN] if n > SEG_LEN else sg[:1] for s, sg, n in zip(srcs, segs, lens)], 0)
        enr = self._run_segments("se", None, None, first, do_sample, max_segments, **keyed("se", [1] * len(srcs)))[0][:, :SEG_LEN]
        enr = enr / (torch.amax(torch.abs(enr), dim=-1, keepdim=True) + 1e-5) * 0.99       # each utterance by its own peak
        ef = self.extract_semantic_features(enr)
        ef = torch.cat([ef[u:u + 1] for u in range(len(srcs)) for _ in range(rows[u + 1] - rows[u])], 0)
        seg = torch.cat(segs, 0)
        est1, _, _ = self._run_segments("tse", ef, None, seg, do_sample, max_segments, **keyed("tse"))
        est2, _, _ = self._run_segments("rtse", ef, None, seg, do_sample, max_segments, **keyed("rtse"))
        return [(trim(est1, u), trim(est2, u)) for u in range(len(srcs))]

    def _run_segments(self, task, enroll_feats, enroll_lengths, seg, do_sample, max_segments, **gen_kw):
        """seg [S, SEG_LEN] (+ one enrollment row per segment) -> detokenized [S, SEG_LEN], global ids [S, 32], semantic ids [S, T],
        at most max_segments segments per WavLM / generate / detokenize call"""
        est, gids, sids = [], [], []
        for s0 in range(0, seg.size(0), max_segments):
            sl = slice(s0, s0 + max_segments)
            kw = gen_kw if "row_seeds" not in gen_kw else dict(gen_kw, row_seeds=gen_kw["row_seeds"][sl])
            g, s = self._generate_rows(task, None if enroll_feats is None else enroll_feats[sl],
                                       None if enroll_lengths is None else enroll_lengths[sl], seg[sl], do_sample, **kw)
            est.append(self.tokenizer.detokenize(g.unsqueeze(1), s).squeeze(1))
            gids.append(g)
            sids.append(s)
        if len(est) == 1:
            return est[0], gids[0], sids[0]
        return torch.cat(est, 0), torch.cat(gids, 0), torch.cat(sids, 0)

    def test_epoch(self, batches, max_segments: int = MAX_SEGMENTS):
        """test_step over many batches, with consecutive batches of the same mode enhanced together (`enhance_batch`, at most
        max_segments 5 s segments per call).  Returns, and writes under `save_enhanced`, exactly what test_step returns and writes
        for each batch, in order."""
        batches = list(batches)
        out, i = [], 0
        while i < len(batches):
            mode, j, n_seg = batches[i][0], i, 0
            while j < len(batches) and batches[j][0] == mode and (j == i or n_seg + self._n_segments(batches[j][2]) <= max_segments):
                n_seg += self._n_segments(batches[j][2])
                j += 1
            group = batches[i:j]
            ests = self.enhance_batch(mode, [b[1] for b in group] if mode == "tse" else None, [b[2] for b in group],
                                      do_sample=False, max_segments=max_segments)
            out += [self._test_output(b, e) for b, e in zip(group, ests)]
            i = j
        return out

    @staticmethod
    def _n_segments(src):
        return -(-src.size(-1) // SEG_LEN)

    def test_step(self, batch, batch_idx=0):
        """model.py:170-286: batch = (mode, enroll, src, tgt, fs, lengths, names); greedy decoding (do_sample = False, model.py:173).
        Returns the enhanced waveform(s) as NumPy (the reference's last step before its optional sf.write) and writes
        `<save_enhanced>/<name>.wav` (`_s1` / `_s2` for 'ss') when the config asks for it."""
        mode, enroll, src, tgt, fs, lengths, names = batch
        return self._test_output(batch, self.enhance(mode, enroll, src, do_sample=False))

    def _test_output(self, batch, out):
        mode, enroll, src, tgt, fs, lengths, names = batch
        outs = out if isinstance(out, tuple) else (out,)
        arrays = [o.cpu().numpy() for o in outs]
        save_dir = self.config.get("save_enhanced")
        if save_dir is not None:
            suffixes = ("_s1", "_s2") if mode == "ss" else ("",)
            for a, sfx in zip(arrays, suffixes):
                _write_wav(os.path.join(str(save_dir), f"{names[0]}{sfx}.wav"), a, int(fs[0]))
        return arrays if mode == "ss" else arrays[0]


def _write_wav(path: str, data, rate: int) -> None:
    try:
        import soundfile as sf           # the reference's writer (model.py:196); not in every image
        sf.write(path, data, samplerate=rate)
    except ImportError:
        from scipy.io import wavfile
        wavfile.write(path, rate, data)
