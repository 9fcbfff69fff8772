"""Time UniSE's training-data simulation (unified_audio_b200.Simulator) on the GPU against the CPU oracle, and the training step with
and without it in front.  B seeded utterances of 4-12 s (speech-like bursts), noise of 2-15 s, interferers and enrollments of 4-12 s,
RIRs of 0.3-1.5 s, cut_duration 5 s, for modes 'se' and 'tse', with the shipped probabilities of conf/simulation_train.yaml and with
every probability forced to 1.  Reports:
  - GPU ms per batch (CUDA events over --iters batches after --warmup, inputs already on the device) and its split by stage (kernel
    time from torch.profiler in a separate pass);
  - the CPU oracle's ms per batch (oracle/simulate.py in the reference's dtypes, one thread) on the same host;
  - ms per full training step (Model.training_step + backward + clip_grad_norm_(5.0) + AdamW, the models of
    scripts/unise_train_bench.py) on a fixed batch and with Simulator.batch in front, shipped probabilities.
Prints one JSON line with the card and its power limit; fails without a GPU."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_simulation as G  # noqa: E402
from oracle import simulate as osim  # noqa: E402
from scripts.bicodec_global_bench import card  # noqa: E402

FS, CUT = 16000, 80000
STAGES = {"frame_power": "non-silence + rms", "active_rms": "non-silence + rms", "place": "place + mix", "mix": "place + mix",
          "rir_prep": "rir window", "convolve": "reverberation", "resample": "bandwidth", "order_stat": "clipping", "clip_kernel": "clipping",
          "packet_loss": "packet loss", "finish": "peak rule + cut + normalise", "enroll": "enrollment"}


def make_inputs(B, seed, mode):
    g = np.random.default_rng(seed)
    w = []
    for _ in range(B):
        w.append({"speech": G.speech_like(g, int(g.integers(4 * FS, 12 * FS))),
                  "noise": (0.2 * g.standard_normal(int(g.integers(2 * FS, 15 * FS)))).astype(np.float32),
                  "rir": G.rir_like(g, "delayed", int(g.integers(int(0.3 * FS), int(1.5 * FS)))),
                  "interf": G.speech_like(g, int(g.integers(4 * FS, 12 * FS))),
                  "enroll": G.speech_like(g, int(g.integers(4 * FS, 12 * FS))) if mode != "se" else None})
    return w


def on_device(w, sim, mode):
    c = lambda a: None if a is None else torch.from_numpy(a).cuda()
    speech, noise, rir = [c(x["speech"]) for x in w], [c(x["noise"]) for x in w], [c(x["rir"]) for x in w]
    interf = [c(x["interf"]) if mode != "se" or sim.se_interference() else None for x in w]
    enroll = [c(x["enroll"]) for x in w] if mode != "se" else None
    return speech, noise, rir, interf, enroll


def gpu_leg(cfg, mode, w, iters, warmup):
    from unified_audio_b200 import Simulator
    sim = Simulator(cfg, seed=1)
    args = on_device(w, sim, mode)
    for _ in range(warmup):
        sim.batch(mode, *args)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        sim.batch(mode, *args)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            sim.batch(mode, *args)
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        stage = next((v for k, v in STAGES.items() if k in e.key), "other (cat / copies)")
        split[stage] = split.get(stage, 0.0) + e.device_time_total / 1e3 / iters
    return ms, {k: round(v, 3) for k, v in sorted(split.items())}


def cpu_leg(cfg, mode, w):
    """one batch through the oracle in the reference's dtypes on one thread, parameters from the same draws"""
    from unified_audio_b200 import Simulator
    torch.set_num_threads(1)
    sim = Simulator(cfg, seed=1)
    interf = [x["interf"] if mode != "se" or sim.se_interference() else None for x in w]
    t = time.perf_counter()
    for x, i in zip(w, interf):
        p = sim.draw(mode, len(x["speech"]), len(x["noise"]), None if i is None else len(i), None if x["enroll"] is None else len(x["enroll"]),
                     CUT, CUT)
        osim.apply(p, x["speech"], x["noise"], x["rir"], i, x["enroll"], cut=CUT, enroll_len=CUT)
    return (time.perf_counter() - t) * 1e3


def train_legs(B, iters, warmup, inputs):
    from scripts.unise_train_bench import CONF
    from scripts.unise_validation_bench import build_model, make_batch
    from unified_audio_b200 import Simulator
    dev = torch.device("cuda")
    model = build_model(dev)
    model.config = dict(CONF)
    [opt], [sch] = model.configure_optimizers()
    sch = sch["scheduler"]

    def step(batch):
        out = model.training_step(batch)
        out["loss"].backward()
        torch.nn.utils.clip_grad_norm_(model.dnn.parameters(), 5.0)
        opt.step()
        sch.step()
        opt.zero_grad(set_to_none=True)

    legs = []
    for mode in ("se", "tse"):
        fixed = make_batch(mode, B, dev)
        sim = Simulator(G.config(forced=False), seed=2)
        args = on_device(inputs[mode], sim, mode)
        res = {"mode": mode}
        for tag, make in (("fixed_batch", lambda: fixed), ("simulated_batch", lambda: sim.batch(mode, *args))):
            for _ in range(warmup):
                step(make())
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(iters):
                step(make())
            t1.record()
            torch.cuda.synchronize()
            res[f"ms_per_step_{tag}"] = round(t0.elapsed_time(t1) / iters, 3)
        legs.append(res)
    return legs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-train", action="store_true", help="skip the training-step legs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unise_simulate_bench: needs a CUDA device")
    inputs = {mode: make_inputs(args.batch, 5 + (mode == "tse"), mode) for mode in ("se", "tse")}
    legs = []
    for mode in ("se", "tse"):
        for probs in ("shipped", "forced"):
            cfg = G.config(forced=probs == "forced")
            ms, split = gpu_leg(cfg, mode, inputs[mode], args.iters, args.warmup)
            legs.append(dict(mode=mode, probabilities=probs, gpu_ms_per_batch=round(ms, 3), gpu_stage_ms=split,
                             cpu_oracle_ms_per_batch_one_thread=round(cpu_leg(cfg, mode, inputs[mode]), 1)))
    out = dict(metric="unise_simulation", batch=args.batch, cut_seconds=CUT / FS, legs=legs, card=card())
    if not args.no_train:
        out["train_step"] = train_legs(args.batch, max(2, args.iters // 2), 2, inputs)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
