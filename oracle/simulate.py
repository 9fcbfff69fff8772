"""CPU oracle of UniSE's training-data simulation: `simulate_data` (QuarkAudio-UniSE/dataloader/simulation/simulate.py:126-192)
and the post-load steps of `TrainDataLoadIter.process_one_sample` (dataloader/data_module.py:106-140, 207-235).

TEST INFRASTRUCTURE.  A NumPy / SciPy restatement in two halves:
  draw(rng, nprng, ...)   every random parameter of one example, from the lengths alone, making the reference's generator calls in
                          its order (the one exception is documented at `draw`)
  apply(p, waves, fp64)   the signal path for those parameters.  fp64=False preserves the reference's dtypes: float32 in, float32
                          through mixing and reverberation, float64 from the clipping stage on (np.quantile returns float64 and
                          np.clip promotes), float32 out as data_iter_fn's `.float()`.  fp64=True runs every stage in float64.
                          Its last stages are `finish` (peak rule, cut, normalisation) and `enroll`, which the kernel tests call
                          directly.
Bandwidth limitation uses torchaudio's sinc_interp_hann resampler (the taps of unified_audio_b200.ssl.resample_kernel, fp32) in
place of the reference's soxr_hq, which is not available offline (DESIGN.md section 3).
tests/golden/simulation_small.npz (oracle/make_golden_simulation.py) pins `apply` bit for bit against the reference's own code."""
from __future__ import annotations

import numpy as np
import scipy.signal
import torch
import torch.nn.functional as F

from oracle.hubert import resample_kernel

FRAME, SHIFT, THRESHOLD = 1024, 512, 0.01


# --------------------------------------------------------------------------- parameter draw
def packet_loss_indices(nprng, length, fs, packet_ms, rate, max_run):
    """get_packet_loss_indices: sorted packet indices zeroed (runs of 1..max_run-1 packets at distinct random starts)"""
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


def draw(rng, nprng, cfg, mode, len_speech, len_noise, len_interf=None, len_enroll=None, have_rir=True, cut=80000, enroll_len=80000,
         fs=16000):
    """Every random parameter of one example.  `rng` stands for the reference's `random`, `nprng` for `np.random`.
    The reference draws the normalisation uniform of normalize_mix_speech_inferf only when the cut example's peaks allow it; this
    draws its underlying `random()` always (`norm_r`), so only the position of that one draw in the stream differs."""
    p = {"mode": mode}
    p["sir"] = rng.uniform(*cfg["tse_interference" if mode in ("tse", "rtse") else "se_interference"]["sir"])
    p["snr"] = rng.uniform(*cfg["noise"]["snr"])
    p["fs_new"] = rng.choice(cfg["bandwidth_limitation"]["fs_new"])
    p["min_q"] = rng.uniform(*cfg["clipping"]["min_quantile"])
    p["max_q"] = rng.uniform(*cfg["clipping"]["max_quantile"])
    p["loss_rate"] = rng.uniform(*cfg["packet_loss"]["packet_loss_rate"])
    p["interf"] = len_interf is not None
    p["interf_offset"] = _offset(nprng, len_speech, len_interf) if p["interf"] else None
    p["reverb"] = rng.random() < cfg["reverberation"]["prob"] and have_rir
    p["noise"] = rng.random() < cfg["noise"]["prob"]
    p["noise_offset"] = _offset(nprng, len_speech, len_noise) if p["noise"] else None
    order = [0, 1, 2]
    rng.shuffle(order)
    p["order"], p["apply"], p["lost"] = order, [], []
    probs = [cfg["bandwidth_limitation"]["prob"], cfg["clipping"]["prob"], cfg["packet_loss"]["prob"]]
    for k in order:
        on = rng.random() < probs[k]
        p["apply"].append(on)
        if k == 2 and on:
            pl = cfg["packet_loss"]
            p["lost"] = packet_loss_indices(nprng, len_speech, fs, pl["packet_duration_ms"], p["loss_rate"], pl["max_continuous_packet_loss"])
    p["cut_offset"] = rng.randint(0, len_speech - cut) if len_speech >= cut else None
    p["norm_r"] = rng.random()
    p["enroll_offset"] = None
    if len_enroll is not None and len_enroll >= enroll_len:
        p["enroll_offset"] = rng.randint(0, len_enroll - enroll_len)
    return p


class _Replay:
    """`random` and `np.random` stand-ins that hand back a recorded call list ([name, args, kwargs, result(, underlying random())])
    in order, checking each call's name and arguments: draw() over a replay rebuilds the parameters the reference drew."""

    def __init__(self, calls):
        self.calls = list(calls)
        self.py, self.np = _ReplayFace(self, "random."), _ReplayFace(self, "np.random.")

    def pop(self, tag, args):
        assert self.calls, f"replay: {tag}{args} past the end of the recorded calls"
        c = self.calls.pop(0)
        assert c[0] == tag and _same(c[1], args), f"replay: called {tag}{args}, recorded {c[:2]}"
        return c


class _ReplayFace:
    def __init__(self, rp, prefix):
        self.rp, self.prefix = rp, prefix

    def uniform(self, a, b):
        return self.rp.pop(self.prefix + "uniform", [a, b])[3]

    def random(self):
        """the normalisation draw: the reference called uniform(0.1, 0.99) or uniform(lo, 1) (its underlying random() is replayed)
        or, in normalize_mix_speech_inferf, maybe nothing"""
        c = self.rp.calls[0] if self.rp.calls else None
        if c is not None and c[0] == "random.uniform":
            return self.rp.calls.pop(0)[4]
        if c is None or c[0] != "random.random":
            return None
        return self.rp.pop("random.random", [])[3]

    def choice(self, seq, *args, **kw):
        return np.asarray(self.rp.pop(self.prefix + "choice", [list(seq)] + list(args))[3]) if args else \
            self.rp.pop(self.prefix + "choice", [list(seq)])[3]

    def shuffle(self, x):
        x[:] = self.rp.pop(self.prefix + "shuffle", [list(x)])[3]

    def randint(self, a, b):
        return self.rp.pop(self.prefix + "randint", [a, b])[3]


def _same(a, b):
    if isinstance(a, (list, tuple)) or isinstance(b, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def replay(calls, cfg, mode, len_speech, len_noise, len_interf=None, len_enroll=None, cut=80000, enroll_len=80000, fs=16000):
    """draw()'s parameters rebuilt from the reference's recorded generator calls (after the 'se' interference coin).  norm_r is the
    underlying random() of normalize_src_tgt's / normalize_mix_speech_inferf's uniform, or None when the reference drew none."""
    rp = _Replay(calls)
    p = draw(rp.py, rp.np, cfg, mode, len_speech, len_noise, len_interf, len_enroll, True, cut, enroll_len, fs)
    assert not rp.calls, f"replay: recorded calls left over: {rp.calls}"
    return p


def _offset(nprng, len_speech, len_other):
    if len_other < len_speech:
        return int(nprng.randint(0, len_speech - len_other))
    if len_other > len_speech:
        return int(nprng.randint(0, len_other - len_speech))
    return None


# --------------------------------------------------------------------------- stages (x: [1, T])
def non_silence(x):
    """detect_non_silence: framed variance (frame 1024, shift 512, zero padding to whole frames, boxcar), frames above 0.01 of the
    mean frame power, one flag per shift, the last flag repeated to the end.  Rows shorter than a frame or of zero power: all True."""
    T = x.shape[-1]
    if T < FRAME:
        return np.ones(x.shape, dtype=bool)
    pad = (-(T - FRAME) % SHIFT) % FRAME
    xp = np.pad(x, [(0, 0), (0, pad)])
    frames = np.lib.stride_tricks.sliding_window_view(xp, FRAME, axis=-1)[:, ::SHIFT]
    power = frames.var(axis=-1)
    mean = power.mean(axis=-1, keepdims=True)
    if np.all(mean == 0):
        return np.ones(x.shape, dtype=bool)
    flags = np.repeat(power / mean > THRESHOLD, SHIFT, axis=-1)
    return np.pad(flags, [(0, 0), (0, T - flags.shape[-1])], mode="edge")


def non_silence_margin(x):
    """smallest |power / mean - 0.01| over the frames of x (inf when detection is bypassed), in x's dtype"""
    T = x.shape[-1]
    if T < FRAME:
        return float("inf")
    pad = (-(T - FRAME) % SHIFT) % FRAME
    power = np.lib.stride_tricks.sliding_window_view(np.pad(x, [(0, 0), (0, pad)]), FRAME, axis=-1)[:, ::SHIFT].var(axis=-1)
    mean = power.mean(axis=-1, keepdims=True)
    return float("inf") if np.all(mean == 0) else float(np.abs(power / mean - THRESHOLD).min())


def active_rms(x):
    return x[non_silence(x)].std()


def place(other, length, offset):
    """mix_noise's alignment: `other` wrap-padded from `offset` (shorter) or cut at `offset` (longer) to `length` samples"""
    n = other.shape[-1]
    if n < length:
        return np.pad(other, [(0, 0), (offset, length - n - offset)], mode="wrap")
    if n > length:
        return other[:, offset:offset + length]
    return other


def mix(x, other, snr, offset):
    other = place(other, x.shape[-1], offset)
    scale = 10 ** (-snr / 20) * active_rms(x) / (active_rms(other) + 1e-10)
    return other * scale + x


def rir_window(h):
    """get_rir_start_sample on h [K]: (start, end) of the early part around the first absolute peak"""
    a = np.abs(h)
    peak = np.argmax(a)
    thr = 0.1 * a[peak]
    start = int(np.argmax(a[:peak + 1] > thr))
    end = int(np.argmax(a[peak + 1:] < thr)) + int(peak) + 1
    return start, end


def reverb(x, h):
    """scipy.signal.convolve(x, h, 'full') truncated to len(x)"""
    return scipy.signal.convolve(x, h, mode="full")[:, :x.shape[1]]


def resample(x, orig, new):
    """torchaudio sinc_interp_hann resampling of x [C, T] in x's dtype, taps as the product's (fp32)"""
    k, width, o, n = resample_kernel(orig, new)
    t = torch.from_numpy(np.ascontiguousarray(x))
    y = F.conv1d(F.pad(t, (width, width + o))[:, None], k.to(t.dtype), stride=o)
    y = y.transpose(1, 2).reshape(t.shape[0], -1)[:, :-(-n * t.shape[1] // o)]
    return y.numpy()


def bandwidth(x, fs, fs_new):
    if fs_new == fs:
        return x
    return resample(resample(x, fs, fs_new), fs_new, fs)[:, :x.shape[1]]


def clip(x, min_q, max_q):
    lo, hi = np.quantile(x, np.array([min_q, max_q]), axis=-1)
    return np.stack([np.clip(x[i], lo[i], hi[i]) for i in range(x.shape[0])], axis=0)


def packet_loss(x, lost, fs=16000, packet_ms=20):
    x = x.copy()
    for i in lost:
        x[:, i * packet_ms * fs // 1000:(i + 1) * packet_ms * fs // 1000] = 0
    return x


def pad_or_cut(x, length, offset):
    if x.shape[-1] < length:
        return np.pad(x, [(0, 0), (0, length - x.shape[-1])], mode="wrap")
    return x[:, offset:offset + length]


# --------------------------------------------------------------------------- the whole example
def apply(p, speech, noise, rir=None, interf=None, enroll=None, cut=80000, enroll_len=80000, fs=16000, fp64=False):
    """One example for the parameters of `draw` -> (enroll, mix, speech, interf) as data_iter_fn stacks them (float32 unless fp64;
    enroll None when not given, interf None when the example has no interferer)."""
    dt = np.float64 if fp64 else np.float32
    as2 = lambda w: None if w is None else np.asarray(w, dtype=dt).reshape(1, -1)
    speech, noise, rir, interf, enroll = map(as2, (speech, noise, rir, interf, enroll))
    if p["interf"]:
        noisy = mix(speech, interf, p["sir"], p["interf_offset"])
        interf = noisy - speech
    else:
        noisy, interf = speech.copy(), None
    if p["reverb"]:
        h = rir / (np.max(np.abs(rir)) + 1e-5)
        s, e = rir_window(h[0])
        early = np.zeros_like(h)
        early[:, s:e] = h[:, s:e]
        noisy = reverb(noisy, h)
        speech = reverb(speech, early)
        if interf is not None:
            interf = reverb(interf, early)
    if p["noise"]:
        noisy = mix(noisy, noise, p["snr"], p["noise_offset"])
    for k, on in zip(p["order"], p["apply"]):
        if not on:
            continue
        if k == 0:
            noisy = bandwidth(noisy, fs, p["fs_new"])
        elif k == 1:
            noisy = clip(noisy, p["min_q"], p["max_q"])
        else:
            noisy = packet_loss(noisy, p["lost"], fs)
    noisy, speech, interf = finish(noisy, speech, interf, cut, p["cut_offset"], p["norm_r"])
    if enroll is not None:
        enroll = _enroll(enroll, enroll_len, p["enroll_offset"])
    out = lambda w: None if w is None else w[0].astype(dt)
    return out(enroll), out(noisy), out(speech), out(interf)


def finish(noisy, speech, interf, cut, cut_offset, norm_r):
    """The peak rule (above 0.99 every signal becomes v / peak * 0.99), pad_or_cut to `cut` samples, then normalize_src_tgt (interf
    None) or normalize_mix_speech_inferf with the uniform's underlying random() `norm_r` -> (noisy, speech, interf), each [1, cut].
    In float32 with a Python float norm_r every operation stays in float32 (NEP 50) except 0.1 + (0.99 - 0.1) * norm_r, which is
    Python arithmetic in double: the rounding csrc/simulate.cu's finish_kernel reproduces."""
    peak = max(np.max(np.abs(noisy)), np.max(np.abs(speech)))
    if interf is not None:
        peak = max(peak, np.max(np.abs(interf)))
    if peak > 0.99:
        noisy, speech = noisy / peak * 0.99, speech / peak * 0.99
        if interf is not None:
            interf = interf / peak * 0.99
    noisy, speech = pad_or_cut(noisy, cut, cut_offset), pad_or_cut(speech, cut, cut_offset)
    if interf is None:
        tgt, src = np.max(np.abs(speech)) + 1e-5, np.max(np.abs(noisy)) + 1e-5
        factor = min((0.1 + (0.99 - 0.1) * norm_r) / tgt, 0.99 / max(tgt, src))
        noisy, speech = noisy * factor, speech * factor
    else:
        interf = pad_or_cut(interf, cut, cut_offset)
        a, b, c = np.max(np.abs(noisy)), np.max(np.abs(speech)), np.max(np.abs(interf))
        factor = 0.99 / (max(a, b, c) + 1e-5)
        least = min(a, b, c)
        if least * factor > 0.1:
            lo = 0.1 / (least * factor)
            factor = (lo + (1 - lo) * norm_r) * factor
        noisy, speech, interf = noisy * factor, speech * factor, interf * factor
    return noisy, speech, interf


def enroll(e, enroll_len, offset):
    """The enrollment: pad_or_cut to `enroll_len` samples at `offset`, then e / (max|e| + 1e-5) * 0.99 -> [1, enroll_len]"""
    e = pad_or_cut(e, enroll_len, offset)
    return e / (np.max(np.abs(e)) + 1e-5) * 0.99


_enroll = enroll          # apply's argument `enroll` shadows the function there
