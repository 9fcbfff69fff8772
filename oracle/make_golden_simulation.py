"""Pin UniSE's training-data simulation against the REFERENCE'S OWN CODE: `simulate_data` (QuarkAudio-UniSE/dataloader/simulation/
simulate.py:126-192) and the post-load steps of `TrainDataLoadIter.process_one_sample` (dataloader/data_module.py:171-235).

TEST INFRASTRUCTURE.  Run in the build container only:  python -m oracle.make_golden_simulation [--out PATH]

`dataloader/__init__.py` needs soundfile and pytorch_lightning, so the `dataloader` package is a stub whose `__path__` is the
reference's directory and its `simulation` sub-package is imported as shipped; `librosa.resample` is the torchaudio
sinc_interp_hann resampler the product uses (oracle.simulate.resample) since soxr is not available.  A `TrainDataLoadIter` is built
without its `__init__`, its file reads return the seeded inputs of CASES, and the speaker / noise / RIR selection draws go to a
generator of their own (they are the caller's job, out of the simulation's scope).  Every call the reference makes to `random` and
`np.random` for the simulation is recorded with its arguments and result.  For each case the fixture holds the seed, the recorded
calls and the reference's outputs (float32, as data_iter_fn stacks them); the inputs are re-made from CASES.  Before writing, the
script checks that oracle.simulate.apply(recorded draws) reproduces every output bit for bit.
"""
import argparse
import copy
import io
import json
import os
import random
import sys
import types
import zipfile

import numpy as np

from oracle import simulate as osim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/QuarkAudio-UniSE/dataloader"
OUT = os.path.join(ROOT, "tests", "golden", "simulation_small.npz")
REPORT = os.path.join(ROOT, "tests", "golden", "simulation_pinning_report.json")
FS, CUT, ENROLL = 16000, 4000, 2000          # cut_duration 0.25 s, enroll_duration 0.125 s: keeps the fixture small

SHIPPED = {   # conf/simulation_train.yaml
    "se_interference": {"prob": 0.2, "sir": [2.0, 20.0]}, "tse_interference": {"sir": [-5.0, 5.0]}, "reverberation": {"prob": 0.3},
    "noise": {"prob": 0.8, "snr": [-5.0, 20.0]},
    "bandwidth_limitation": {"prob": 0.3, "fs_new": [4000, 8000, 16000], "res_type": "soxr_hq"},
    "clipping": {"prob": 0.3, "min_quantile": [0.0, 0.1], "max_quantile": [0.9, 1.0]},
    "packet_loss": {"prob": 0.3, "packet_duration_ms": 20, "packet_loss_rate": [0.05, 0.25], "max_continuous_packet_loss": 10},
}


def config(forced, se_interf=None, fs_new=None):
    c = copy.deepcopy(SHIPPED)
    if forced:
        for k in ("reverberation", "noise", "bandwidth_limitation", "clipping", "packet_loss"):
            c[k]["prob"] = 1.0
    if se_interf is not None:
        c["se_interference"]["prob"] = se_interf
    if fs_new is not None:
        c["bandwidth_limitation"]["fs_new"] = [fs_new]
    return c


# name: (mode, seed, config kwargs, speech len, noise len ('zero:' = all-zero), interf len, enroll len, rir kind, rir len)
CASES = {
    "se_forced_noise_short":      ("se", 1, dict(forced=True, se_interf=0.0, fs_new=4000), 12000, 5000, None, None, "delayed", 3000),
    "se_interf_forced_noise_long": ("se", 2, dict(forced=True, se_interf=1.0, fs_new=8000), 9000, 16000, 7000, None, "delayed", 2000),
    "tse_forced_noise_equal":     ("tse", 3, dict(forced=True), 10000, 10000, 13000, 6000, "delayed", 4000),
    "rtse_forced_long_tail":      ("rtse", 4, dict(forced=True, fs_new=4000), 16000, 3000, 16000, 1500, "no_fall", 1200),
    "se_forced_short_row":        ("se", 5, dict(forced=True, se_interf=0.0, fs_new=8000), 800, 2500, None, None, "delayed", 600),
    "tse_forced_zero_noise":      ("tse", 6, dict(forced=True, fs_new=4000), 7000, "zero:7500", 5000, 2500, "delayed", 1500),
    "se_interf_forced_short":     ("se", 7, dict(forced=True, se_interf=1.0, fs_new=4000), 3000, 900, 700, None, "delayed", 800),
    "se_shipped_a":               ("se", 11, dict(forced=False), 14000, 6000, None, None, "delayed", 2500),
    "se_shipped_b":               ("se", 12, dict(forced=False, se_interf=1.0), 11000, 15000, 9000, None, "delayed", 2500),
    "tse_shipped":                ("tse", 13, dict(forced=False), 15000, 4000, 12000, 3000, "delayed", 2500),
    "rtse_shipped":               ("rtse", 14, dict(forced=False), 6000, 8000, 6000, 1000, "no_fall", 900),
}


def speech_like(g, n):
    """voiced bursts with pauses: some frames fall under the non-silence threshold"""
    t = np.arange(n) / FS
    f0 = g.uniform(90, 250)
    x = sum(np.sin(2 * np.pi * f0 * h * t + g.uniform(0, 6.3)) / h for h in range(1, 6))
    env = (np.sin(2 * np.pi * g.uniform(1.5, 4) * t + g.uniform(0, 6.3)) > -0.2) * (0.2 + 0.8 * g.random(n) ** 0.1)
    return (0.3 * x * env + 0.003 * g.standard_normal(n)).astype(np.float32)


def rir_like(g, kind, n):
    """decaying noise with its peak some samples in; 'no_fall' keeps every sample after the peak above a tenth of it"""
    d = int(g.integers(5, 40))
    tail = g.standard_normal(n) * np.exp(-np.arange(n) / (0.15 * n))
    h = np.concatenate([0.01 * g.standard_normal(d), [1.0], 0.5 * tail[:n - d - 1]])
    if kind == "no_fall":
        h[d + 1:] = np.sign(h[d + 1:] + 1e-12) * (0.2 + 0.5 * np.abs(h[d + 1:]))
    return h.astype(np.float32)


def make_inputs(name):
    """the case's inputs, 1-D float32: dict speech, noise, interf, enroll (None when absent), rir"""
    mode, seed, _, ls, ln, li, le, rk, lr = CASES[name]
    g = np.random.default_rng(1000 + seed)
    w = {"speech": speech_like(g, ls)}
    if isinstance(ln, str):
        w["noise"] = np.zeros(int(ln.split(":")[1]), dtype=np.float32)
    else:
        w["noise"] = (0.2 * g.standard_normal(ln)).astype(np.float32)
    w["interf"] = speech_like(g, li) if li else None
    w["enroll"] = speech_like(g, le) if le else None
    w["rir"] = rir_like(g, rk, lr)
    return w


# --------------------------------------------------------------------------- the reference, imported piecewise
def import_reference():
    """-> the reference's TrainDataLoadIter, with dataloader/simulation imported as shipped"""
    import importlib
    lib = types.ModuleType("librosa")
    lib.resample = lambda y, orig_sr, target_sr, res_type=None: osim.resample(y, orig_sr, target_sr)
    lib.load = None
    sf = types.ModuleType("soundfile")
    pl = types.ModuleType("pytorch_lightning")
    pl.LightningDataModule = object
    pkg = types.ModuleType("dataloader")
    pkg.__path__ = [REF]
    for name, mod in (("librosa", lib), ("soundfile", sf), ("pytorch_lightning", pl), ("dataloader", pkg)):
        sys.modules[name] = mod
    importlib.import_module("dataloader.simulation")
    dm = importlib.import_module("dataloader.data_module")
    return dm.TrainDataLoadIter


class Recorder:
    """wraps the module-level functions of `random` and `np.random` the reference calls and records [name, args, kwargs, result]
    (`random.uniform` also its underlying `random()`, as a fifth entry).  Speaker / utterance / noise / RIR selection
    (random.sample, random.choice over loader lists) is served by a separate generator and not recorded."""

    def __init__(self):
        self.calls, self.select, self.saved = [], random.Random(99), {}

    def __enter__(self):
        base_random = random.random

        def wrap(mod, name, tag):
            fn = getattr(mod, name)
            self.saved[(mod, name)] = fn

            def rec(*args, **kw):
                if tag == "random.sample" or (tag == "random.choice" and not all(isinstance(v, int) for v in args[0])):
                    return getattr(self.select, name)(*args, **kw)
                if tag == "random.uniform":            # random.Random.uniform: a + (b - a) * random()
                    a, b = args
                    r = base_random()
                    out = a + (b - a) * r
                    self.calls.append([tag, _plain(args), {}, _plain(out), r])
                    return out
                if tag == "random.shuffle":
                    before = list(args[0])
                    fn(*args, **kw)
                    self.calls.append([tag, [before], {}, list(args[0])])
                    return None
                out = fn(*args, **kw)
                self.calls.append([tag, _plain(args), _plain(kw), _plain(out)])
                return out
            setattr(mod, name, rec)
        for n in ("uniform", "random", "choice", "shuffle", "randint", "sample"):
            wrap(random, n, "random." + n)
        for n in ("randint", "choice"):
            wrap(np.random, n, "np.random." + n)
        return self

    def __exit__(self, *a):
        for (mod, name), fn in self.saved.items():
            setattr(mod, name, fn)


def _plain(v):
    if isinstance(v, (list, tuple, range)):
        return [_plain(x) for x in v]
    if isinstance(v, dict):
        return {k: _plain(x) for k, x in v.items()}
    if isinstance(v, np.ndarray):
        return [_plain(x) for x in v.tolist()]
    if isinstance(v, (np.integer,)):
        return int(v)
    if isinstance(v, (np.floating,)):
        return float(v)
    return v


def run_reference(Loader, name):
    """one process_one_sample of the case -> (recorded calls, enroll, mix, speech, interf, output dtypes)"""
    mode, seed, ckw, *_ = CASES[name]
    w = make_inputs(name)
    it = Loader.__new__(Loader)
    it.simulation_config, it.enroll_duration = config(**ckw), ENROLL / FS
    Info = types.SimpleNamespace
    it.spk_list = ["a", "b"]
    it.spk2speech = {"a": [Info(utt="s1"), Info(utt="s2")], "b": [Info(utt="i1"), Info(utt="i2")]}
    it.noise_list, it.rir_list = [Info(utt="n")], [Info(utt="r")]
    loads = [w["speech"]] + ([w["enroll"]] if mode != "se" else []) + ([w["interf"]] if w["interf"] is not None else [])
    loads = iter(loads)
    files = iter([w["noise"], w["rir"]])
    it.load_wav_with_timeout = lambda info, fs=None, timeout=1.0: (next(loads)[None].copy(), FS)
    it.load_wav = lambda info, fs=None: (next(files)[None].copy(), FS)
    random.seed(seed)
    np.random.seed(seed)
    with Recorder() as r:
        enroll, mix, speech, interf, fs, length, _ = it.process_one_sample(FS, CUT / FS, mode)
    assert fs == FS and length == CUT
    dtypes = [None if a is None else str(a.dtype) for a in (enroll, mix, speech, interf)]
    f32 = lambda a: None if a is None else a[0].astype(np.float32)
    return r.calls, f32(enroll), f32(mix), f32(speech), f32(interf), dtypes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=OUT)
    args = ap.parse_args()
    Loader = import_reference()
    arrays, meta, report = {}, {}, {"cases": {}}
    for name in CASES:
        calls, enroll, mix, speech, interf, dtypes = run_reference(Loader, name)
        meta[name] = {"calls": calls, "dtypes": dtypes}
        for k, a in (("enroll", enroll), ("mix", mix), ("speech", speech), ("interf", interf)):
            if a is not None:
                arrays[f"{name}/{k}"] = a
        report["cases"][name] = {"calls": len(calls), "dtypes": dtypes, "check": check_case(name, calls, (enroll, mix, speech, interf))}
    arrays["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    write_npz(args.out, arrays)
    with open(REPORT, "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(f"wrote {args.out} ({os.path.getsize(args.out)} bytes) and {REPORT}")


def recorded_params(name, calls):
    """oracle.simulate.draw's parameters replayed from the reference's recorded calls (the se-interference coin first in 'se')"""
    mode, _, ckw, ls, ln, li, le, *_ = CASES[name]
    n_noise = int(ln.split(":")[1]) if isinstance(ln, str) else ln
    if mode == "se":
        assert calls[0][0] == "random.random" and (calls[0][3] < config(**ckw)["se_interference"]["prob"]) == (li is not None)
        calls = calls[1:]
    return osim.replay(calls, config(**ckw), mode, ls, n_noise, li, le, cut=CUT, enroll_len=ENROLL, fs=FS)


def check_case(name, calls, want):
    p = recorded_params(name, calls)
    w = make_inputs(name)
    got = osim.apply(p, w["speech"], w["noise"], w["rir"], w["interf"], w["enroll"], cut=CUT, enroll_len=ENROLL, fs=FS)
    for g, r, k in zip(got, want, ("enroll", "mix", "speech", "interf")):
        assert (g is None) == (r is None), (name, k)
        if g is not None:
            assert g.dtype == r.dtype and np.array_equal(g, r), (name, k, float(np.abs(g.astype(np.float64) - r).max()))
    return "bit-identical"


def write_npz(path, arrays):
    """np.savez_compressed with fixed zip timestamps, so a rerun reproduces the file byte for byte"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[k]))
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(zi, buf.getvalue())


if __name__ == "__main__":
    main()
