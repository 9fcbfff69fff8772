"""UniSE's training mixtures on the GPU: `Simulator` replaces `simulate_data` (QuarkAudio-UniSE/dataloader/simulation/simulate.py:126-192)
and the steps of `TrainDataLoadIter.process_one_sample` after the file reads (dataloader/data_module.py:106-140, 207-235).

Raw 16 kHz utterances, noise and room impulse responses go in as CUDA tensors; out comes the batch tuple `Model.training_step`
consumes, `(mode, enroll, mix, speech, interf, fs, lengths, names)`, as data_iter_fn (data_module.py:238-266) stacks it.  Every random
parameter is drawn on the host from the lengths alone; the signal path runs in csrc/simulate.cu on packed ragged rows.  File reads,
the choice of speakers / utterances / noise / RIR, the mode and the cut duration per batch stay with the caller."""
from __future__ import annotations

import copy
import random
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import ops
from .ssl import resample_kernel

MODES = ("se", "tse", "rtse")
PACKET_FS = 16000


def packet_loss_indices(nprng, length, fs, packet_ms, rate, max_run) -> List[int]:
    """get_packet_loss_indices (simulate.py:80-112), drawing as it does: runs of randint(1, max_run) packets until the rest fits in one
    run, then distinct starts from choice(range(packets), runs, replace=False).  Returns the sorted set of packet indices."""
    duration_ms = length / fs * 1000
    packets = int(duration_ms // packet_ms)
    lost = int(round(rate * duration_ms / packet_ms, 0))
    runs = []
    for _ in range(lost):
        runs.append(nprng.randint(1, max_run))
        if lost - sum(runs) <= max_run:
            runs.append(lost - sum(runs))
            break
    starts = nprng.choice(range(packets), len(runs), replace=False)
    return sorted({int(s) + j for s, n in zip(starts, runs) for j in range(n)})


class Simulator:
    """Training-example simulation with the reference's parameter distributions (simulation_config: the dict of
    conf/simulation_train.yaml).

    Random parameters come from the simulator's own `random.Random` (`rng`) and `np.random.RandomState` (`nprng`), seeded by `seed`,
    with the calls simulate_data / process_one_sample make to the global `random` / `np.random`, in their order: SIR, SNR, fs_new, the
    two quantiles, the loss rate, the interferer offset, the reverberation and noise coins, the noise offset, the shuffle of the three
    degradations, their coins (with the packet-loss draws after the packet-loss coin), the cut offset, the normalisation uniform and the
    enrollment offset.  One draw differs: normalize_mix_speech_inferf (data_module.py:130-140) draws its uniform only when the cut
    example's peaks allow it, and those peaks live on the device; the simulator always draws the underlying `random()` and the device
    uses it only in that branch.  Each example's distribution is unchanged; only the position of that draw in the generator stream
    differs (the reference's stream order is not reproducible anyway: its 16 loader threads share the global generators)."""

    def __init__(self, simulation_config: dict, fs: int = 16000, seed: Optional[int] = None):
        if fs != PACKET_FS:
            raise ValueError(f"Simulator: fs must be 16000 (the loader resamples every file to 16 kHz), got {fs}")
        cfg = copy.deepcopy(simulation_config)
        for key in ("se_interference", "tse_interference", "reverberation", "noise", "bandwidth_limitation", "clipping", "packet_loss"):
            if key not in cfg:
                raise ValueError(f"Simulator: simulation_config has no '{key}' section")
        bad = [f for f in cfg["bandwidth_limitation"]["fs_new"] if f not in (4000, 8000, 16000)]
        if bad:
            raise ValueError(f"Simulator: bandwidth_limitation.fs_new must be 4000, 8000 or 16000, got {bad}")
        if cfg["packet_loss"]["max_continuous_packet_loss"] < 2:
            raise ValueError("Simulator: packet_loss.max_continuous_packet_loss must be at least 2 (np.random.randint(1, n))")
        self.cfg, self.fs = cfg, fs
        self.packet = cfg["packet_loss"]["packet_duration_ms"] * fs // 1000
        self.rng, self.nprng = random.Random(seed), np.random.RandomState(seed)
        self._taps = {}

    # ------------------------------------------------------------------ host draws
    def se_interference(self) -> bool:
        """process_one_sample's coin (data_module.py:184): does an 'se' example get an interfering speaker?  A loader calls this before
        it reads the interferer's file and passes interf[i] = None when it returns False."""
        return self.rng.random() < self.cfg["se_interference"]["prob"]

    def draw(self, mode: str, len_speech: int, len_noise: int, len_interf: Optional[int] = None, len_enroll: Optional[int] = None,
             cut: int = 80000, enroll_len: int = 80000) -> dict:
        """Every random parameter of one example from the lengths (in samples)."""
        c, rng = self.cfg, self.rng
        p = {"mode": mode}
        p["sir"] = rng.uniform(*c["tse_interference" if mode in ("tse", "rtse") else "se_interference"]["sir"])
        p["snr"] = rng.uniform(*c["noise"]["snr"])
        p["fs_new"] = rng.choice(c["bandwidth_limitation"]["fs_new"])
        p["min_q"] = rng.uniform(*c["clipping"]["min_quantile"])
        p["max_q"] = rng.uniform(*c["clipping"]["max_quantile"])
        p["loss_rate"] = rng.uniform(*c["packet_loss"]["packet_loss_rate"])
        p["interf"] = len_interf is not None
        p["interf_offset"] = self._offset(len_speech, len_interf) if p["interf"] else None
        p["reverb"] = rng.random() < c["reverberation"]["prob"]
        p["noise"] = rng.random() < c["noise"]["prob"]
        p["noise_offset"] = self._offset(len_speech, len_noise) if p["noise"] else None
        order = [0, 1, 2]                     # 0 bandwidth limitation, 1 clipping, 2 packet loss
        rng.shuffle(order)
        probs = [c["bandwidth_limitation"]["prob"], c["clipping"]["prob"], c["packet_loss"]["prob"]]
        p["order"], p["apply"], p["lost"] = order, [], []
        for k in order:
            on = rng.random() < probs[k]
            p["apply"].append(on)
            if k == 2 and on:
                pl = c["packet_loss"]
                p["lost"] = packet_loss_indices(self.nprng, len_speech, self.fs, pl["packet_duration_ms"], p["loss_rate"],
                                                pl["max_continuous_packet_loss"])
        p["cut_offset"] = rng.randint(0, len_speech - cut) if len_speech >= cut else None
        p["norm_r"] = rng.random()
        p["enroll_offset"] = rng.randint(0, len_enroll - enroll_len) if len_enroll is not None and len_enroll >= enroll_len else None
        return p

    def _offset(self, len_speech, len_other):
        """mix_noise's offset (simulate.py:13-23): None when the lengths agree"""
        if len_other < len_speech:
            return int(self.nprng.randint(0, len_speech - len_other))
        if len_other > len_speech:
            return int(self.nprng.randint(0, len_other - len_speech))
        return None

    # ------------------------------------------------------------------ the batch
    def batch(self, mode: str, speech: Sequence[torch.Tensor], noise: Sequence[torch.Tensor], rir: Sequence[torch.Tensor],
              interf: Optional[Sequence[Optional[torch.Tensor]]] = None, enroll: Optional[Sequence[torch.Tensor]] = None,
              cut_duration: float = 5.0, enroll_duration: float = 5.0, names: Optional[List[str]] = None):
        """One training batch from raw 16 kHz signals (lists of 1-D fp32 CUDA tensors of any lengths, one entry per example).
        interf: per-example interfering speaker, required in 'tse' / 'rtse'; in 'se' entries may be None (follow
        `se_interference()`).  enroll: required in 'tse' / 'rtse'.  Returns (mode, enroll [B, enroll_duration * 16000] or None,
        mix, speech, interf (None in 'se') [B, cut_duration * 16000] fp32, fs, lengths int64 [B], names) on the inputs' device."""
        B, cut, enroll_len = self._check(mode, speech, noise, rir, interf, enroll, cut_duration, enroll_duration)
        interf = list(interf) if interf is not None else [None] * B
        params = [self.draw(mode, speech[i].numel(), noise[i].numel(), None if interf[i] is None else interf[i].numel(),
                            None if enroll is None else enroll[i].numel(), cut, enroll_len) for i in range(B)]
        return self.apply(params, speech, noise, rir, interf, enroll, cut, enroll_len, names)

    def _check(self, mode, speech, noise, rir, interf, enroll, cut_duration, enroll_duration):
        if mode not in MODES:
            raise ValueError(f"Simulator.batch: mode must be one of {MODES}, got {mode!r}")
        B = len(speech)
        if B == 0:
            raise ValueError("Simulator.batch: empty batch")
        if rir is None or noise is None:
            raise ValueError("Simulator.batch: noise and rir are required")
        lists = {"noise": noise, "rir": rir, "interf": interf, "enroll": enroll}
        for name, lst in lists.items():
            if lst is not None and len(lst) != B:
                raise ValueError(f"Simulator.batch: {name} has {len(lst)} entries for {B} utterances")
        if mode != "se" and (interf is None or any(t is None for t in interf)):
            raise ValueError(f"Simulator.batch: mode {mode!r} needs an interfering utterance per example")
        if mode != "se" and enroll is None:
            raise ValueError(f"Simulator.batch: mode {mode!r} needs an enrollment utterance per example")
        if mode == "se" and enroll is not None:
            raise ValueError("Simulator.batch: 'se' takes no enrollment")
        dev = speech[0].device
        for name, lst in {"speech": speech, **lists}.items():
            for i, t in enumerate(lst or []):
                if t is None:
                    continue
                if not (isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.dim() == 1 and t.is_cuda and t.device == dev):
                    raise ValueError(f"Simulator.batch: {name}[{i}] must be a 1-D float32 CUDA tensor on {dev}")
                if t.numel() == 0:
                    raise ValueError(f"Simulator.batch: {name}[{i}] is empty")
        cut, enroll_len = int(cut_duration * self.fs), int(enroll_duration * self.fs)
        if cut < 1 or (mode != "se" and enroll_len < 1):
            raise ValueError(f"Simulator.batch: cut_duration {cut_duration} / enroll_duration {enroll_duration} give no samples")
        return B, cut, enroll_len

    def _resample_taps(self, dev):
        if dev not in self._taps:
            t = {}
            for fs_new, tag in ((4000, "4"), (8000, "2")):
                kd, wd, _, _ = resample_kernel(self.fs, fs_new)
                ku, wu, _, _ = resample_kernel(fs_new, self.fs)
                t["down" + tag], t["kd" + tag], t["wd" + tag] = kd.reshape(-1).contiguous().to(dev), kd.shape[1], wd
                t["up" + tag], t["ku"], t["wu"] = ku.contiguous().to(dev), ku.shape[1], wu
            self._taps[dev] = t
        return self._taps[dev]

    def apply(self, params: List[dict], speech, noise, rir, interf, enroll, cut: int, enroll_len: int, names=None):
        """The signal path for drawn parameters (one dict of `draw` per example); batch() = draw + apply."""
        B = len(speech)
        mode = params[0]["mode"]
        dev = speech[0].device
        interf = list(interf) if interf is not None else [None] * B
        Ls = [int(t.numel()) for t in speech]
        maxL = max(Ls)
        I, D = _Packer(), _Packer()
        offs = I.add("offs", _cum(Ls))
        frames = [0 if L < 1024 else (L + (-(L - 1024)) % 512 % 1024 - 1024) // 512 + 1 for L in Ls]
        I.add("frame_off", _cum(frames))
        Li = [0 if t is None else int(t.numel()) for t in interf]
        Ln, Lr = [int(t.numel()) for t in noise], [int(t.numel()) for t in rir]
        I.add("interf_offs", _cum(Li))
        I.add("noise_offs", _cum(Ln))
        I.add("rir_offs", _cum(Lr))
        I.add("shift_i", [_shift(Ls[i], Li[i], p["interf_offset"]) for i, p in enumerate(params)])
        I.add("shift_n", [_shift(Ls[i], Ln[i], p["noise_offset"]) for i, p in enumerate(params)])
        I.add("cut_off", [-1 if p["cut_offset"] is None else p["cut_offset"] for p in params])
        has_i = [int(p["interf"]) for p in params]
        I.add("has_interf", has_i, np.int32)
        I.add("reverb", [int(p["reverb"]) for p in params], np.int32)
        I.add("reverb_interf", [int(p["reverb"] and p["interf"]) for p in params], np.int32)
        I.add("noise", [int(p["noise"]) for p in params], np.int32)
        I.add("fs_new", [p["fs_new"] for p in params], np.int32)
        slots = []
        for s in range(3):
            on = [[int(p["order"][s] == k and p["apply"][s]) for p in params] for k in range(3)]
            lost = [(i, j) for i, p in enumerate(params) if on[2][i] for j in p["lost"]]
            slots.append((any(on[0]), any(on[1]), lost))
            I.add(f"bw{s}", on[0], np.int32)
            I.add(f"clip{s}", on[1], np.int32)
            if lost:
                I.add(f"lost{s}", [j for _, j in lost])
                I.add(f"lost_row{s}", [i for i, _ in lost], np.int32)
        if enroll is not None:
            Le = [int(t.numel()) for t in enroll]
            I.add("enroll_offs", _cum(Le))
            I.add("enroll_cut", [-1 if p["enroll_offset"] is None else p["enroll_offset"] for p in params])
        D.add("sir", [p["sir"] for p in params], np.float64)
        D.add("snr", [p["snr"] for p in params], np.float64)
        D.add("q", [v for p in params for v in (p["min_q"], p["max_q"])], np.float64)
        D.add("norm_r", [p["norm_r"] for p in params], np.float64)
        iv, dv = I.upload(dev), D.upload(dev)

        x_speech = torch.cat(list(speech))
        noisy = x_speech.clone()
        total = noisy.numel()
        rms_a = torch.empty(B, dtype=torch.float64, device=dev)
        rms_b = torch.empty(B, dtype=torch.float64, device=dev)
        rms = lambda x, out: ops.sim_active_rms(x, iv["offs"], iv["frame_off"], B, maxL, max(frames), out)
        x_interf = None
        if any(has_i):                                   # mix_noise(speech, interf, sir); interf = noisy - speech
            placed = torch.empty_like(noisy)
            ops.sim_place(torch.cat([t for t in interf if t is not None]), iv["interf_offs"], iv["offs"], iv["shift_i"], B, maxL, placed)
            rms(x_speech, rms_a)
            rms(placed, rms_b)
            x_interf = torch.zeros_like(noisy)
            ops.sim_mix(noisy, placed, iv["offs"], B, maxL, dv["sir"], rms_a, rms_b, iv["has_interf"], x_interf)
        if any(p["reverb"] for p in params):             # add_reverberation with the RIR, and with its early part for the targets
            h = torch.cat(list(rir))
            hn, win = torch.empty_like(h), torch.empty(B, 2, dtype=torch.int64, device=dev)
            status = torch.empty(B, dtype=torch.int32, device=dev)
            ops.sim_rir_prep(h, iv["rir_offs"], B, iv["reverb"], hn, win, status)
            bad = status.nonzero().flatten().tolist()     # the one device-to-host read: only when an example is reverberated
            if bad:
                raise ValueError(f"Simulator.batch: rir[{bad[0]}] peaks at its last sample; the reference's get_rir_start_sample "
                                 "fails there (np.argmax of an empty tail)")
            y = torch.empty_like(noisy)
            ops.sim_convolve(noisy, iv["offs"], B, maxL, hn, iv["rir_offs"], None, iv["reverb"], y)
            noisy, y = y, torch.empty_like(noisy)
            ops.sim_convolve(x_speech, iv["offs"], B, maxL, hn, iv["rir_offs"], win, iv["reverb"], y)
            x_speech = y
            if x_interf is not None:
                y = torch.empty_like(noisy)
                ops.sim_convolve(x_interf, iv["offs"], B, maxL, hn, iv["rir_offs"], win, iv["reverb_interf"], y)
                x_interf = y
        if any(p["noise"] for p in params):              # mix_noise(noisy, noise, snr)
            placed = torch.empty_like(noisy)
            ops.sim_place(torch.cat(list(noise)), iv["noise_offs"], iv["offs"], iv["shift_n"], B, maxL, placed)
            rms(noisy, rms_a)
            rms(placed, rms_b)
            ops.sim_mix(noisy, placed, iv["offs"], B, maxL, dv["snr"], rms_a, rms_b, iv["noise"])
        tmp = stats = None
        for s, (bw, clip, lost) in enumerate(slots):     # the shuffled degradations, slot by slot
            if bw:
                tmp = torch.empty(total, device=dev) if tmp is None else tmp
                ops.sim_bandwidth(noisy, iv["offs"], B, maxL, iv["fs_new"], iv[f"bw{s}"], self._resample_taps(dev), tmp)
            if clip:
                stats = torch.empty(B, 4, device=dev) if stats is None else stats
                ops.sim_clip(noisy, iv["offs"], B, maxL, dv["q"], iv[f"clip{s}"], stats)
            if lost:
                ops.sim_packet_loss(noisy, iv["offs"], iv[f"lost{s}"], iv[f"lost_row{s}"], self.packet)
        out_mix = torch.empty(B, cut, device=dev)
        out_speech = torch.empty(B, cut, device=dev)
        out_interf = torch.empty(B, cut, device=dev) if mode != "se" else None
        ops.sim_finish(noisy, x_speech, x_interf, iv["offs"], B, iv["has_interf"], iv["cut_off"], dv["norm_r"], cut, out_mix, out_speech,
                       out_interf)
        out_enroll = None
        if enroll is not None:
            out_enroll = torch.empty(B, enroll_len, device=dev)
            ops.sim_enroll(torch.cat(list(enroll)), iv["enroll_offs"], B, iv["enroll_cut"], enroll_len, out_enroll)
        fs = torch.full((B,), self.fs, dtype=torch.int64, device=dev)
        lengths = torch.full((B,), cut, dtype=torch.int64, device=dev)
        return (mode, out_enroll, out_mix, out_speech, out_interf, fs, lengths,
                list(names) if names is not None else [str(i) for i in range(B)])


def _cum(lengths):
    return [0] + list(np.cumsum(lengths, dtype=np.int64))


def _shift(L, Lo, offset):
    """place_kernel's index shift: wrap padding puts other[0] at `offset`; a cut starts at `offset`"""
    if offset is None or Lo == 0:
        return 0
    return (-offset) % Lo if Lo < L else offset


class _Packer:
    """named per-row host arrays -> one host-to-device copy, device views by name (each array starts 8-byte aligned)"""

    def __init__(self):
        self.parts = []

    def add(self, name, values, dtype=np.int64):
        self.parts.append((name, np.asarray(values, dtype=dtype)))

    def upload(self, dev):
        if not self.parts:
            return {}
        pad = lambda a: np.concatenate([a.view(np.uint8), np.zeros(-a.nbytes % 8, dtype=np.uint8)])
        buf = torch.from_numpy(np.concatenate([pad(a) for _, a in self.parts])).to(dev)
        out, o = {}, 0
        for name, a in self.parts:
            dt = {np.dtype(np.int64): torch.int64, np.dtype(np.int32): torch.int32, np.dtype(np.float64): torch.float64}[a.dtype]
            out[name] = buf[o:o + a.nbytes].view(dt)
            o += a.nbytes + (-a.nbytes % 8)
        return out
