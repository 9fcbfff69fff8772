"""UniSE training-data simulation, host side: the oracle against the reference-pinned fixture, the Simulator's parameter draws against
the reference's recorded generator calls, the configured parameter ranges, and the inputs Simulator.batch refuses (no GPU needed).

tests/golden/simulation_small.npz (oracle/make_golden_simulation.py) holds, per case, the seed, every call the reference's
simulate_data / process_one_sample made to `random` and `np.random`, and its outputs; the inputs are re-made from the case table."""
import json

import numpy as np
import pytest
import torch

from oracle import make_golden_simulation as G
from oracle import simulate as osim
from unified_audio_b200.simulate import Simulator

Z = np.load(G.OUT)
META = json.loads(bytes(Z["meta"]).decode())


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_oracle_reproduces_reference(name):
    p = G.recorded_params(name, META[name]["calls"])
    w = G.make_inputs(name)
    got = osim.apply(p, w["speech"], w["noise"], w["rir"], w["interf"], w["enroll"], cut=G.CUT, enroll_len=G.ENROLL, fs=G.FS)
    for k, g in zip(("enroll", "mix", "speech", "interf"), got):
        key = f"{name}/{k}"
        assert (g is None) == (key not in Z.files), key
        if g is not None:
            assert np.array_equal(g, Z[key]), key


class _Rec:
    """records [name, args, kwargs, result] of a generator's calls (random.Random.uniform is a + (b - a) random(): recorded as uniform)"""

    def __init__(self, gen, prefix, log):
        self.gen, self.prefix, self.log = gen, prefix, log

    def __getattr__(self, name):
        fn = getattr(self.gen, name)

        def call(*args, **kw):
            before = list(args[0]) if name == "shuffle" else None
            out = fn(*args, **kw)
            if name == "shuffle":
                out, args = list(args[0]), (before,)
            self.log.append([self.prefix + name, G._plain(args), G._plain(kw), G._plain(out)])
            return out
        return call


def simulator_calls(name):
    mode, seed, ckw, ls, ln, li, le, *_ = G.CASES[name]
    sim = Simulator(G.config(**ckw), seed=seed)
    log = []
    sim.rng, sim.nprng = _Rec(sim.rng, "random.", log), _Rec(sim.nprng, "np.random.", log)
    if mode == "se":
        assert sim.se_interference() == (li is not None)
    n_noise = int(ln.split(":")[1]) if isinstance(ln, str) else ln
    p = sim.draw(mode, ls, n_noise, li, le, cut=G.CUT, enroll_len=G.ENROLL)
    return log, p


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_draws_follow_reference_calls(name):
    """same seeds -> the same calls with the same results, in order, up to the normalisation draw; after it only the enrollment
    offset follows, which moves by one draw when the reference skipped its conditional uniform"""
    ref = [c[:4] for c in META[name]["calls"]]
    got, p = simulator_calls(name)
    k = next(i for i, c in enumerate(got) if c[0] == "random.random" and c[3] == p["norm_r"] and i >= len(got) - 2)
    assert got[:k] == ref[:k]
    want = G.recorded_params(name, META[name]["calls"])
    assert p["lost"] == want["lost"] and p["cut_offset"] == want["cut_offset"]
    if len(ref) > k and ref[k][0] == "random.uniform":           # the reference drew the normalisation uniform too
        assert META[name]["calls"][k][4] == p["norm_r"]           # its underlying random(), recorded by the generator
        assert got[k + 1:] == ref[k + 1:]
    else:
        assert [c[0] for c in got[k + 1:]] == [c[0] for c in ref[k:]]


def test_parameter_ranges_follow_config():
    cfg = G.config(forced=False)
    sim = Simulator(cfg, seed=5)
    seen = {"fs_new": set(), "order": set()}
    for i in range(400):
        mode = ("se", "tse", "rtse")[i % 3]
        Ls = 8000 + 37 * i
        p = sim.draw(mode, Ls, 5000 + 11 * i, 7000 + 5 * i, 9000, cut=6000, enroll_len=4000)
        sir = cfg["tse_interference" if mode != "se" else "se_interference"]["sir"]
        assert sir[0] <= p["sir"] <= sir[1] and -5.0 <= p["snr"] <= 20.0
        assert 0.0 <= p["min_q"] <= 0.1 and 0.9 <= p["max_q"] <= 1.0 and 0.05 <= p["loss_rate"] <= 0.25
        assert 0 <= p["cut_offset"] <= Ls - 6000 and 0 <= p["enroll_offset"] <= 5000 and 0.0 <= p["norm_r"] < 1.0
        assert p["interf_offset"] is None or 0 <= p["interf_offset"] < abs(Ls - (7000 + 5 * i))
        assert sorted(p["order"]) == [0, 1, 2]
        packets = Ls * 1000 // 16000 // 20
        assert all(0 <= j < packets + 9 for j in p["lost"])
        seen["fs_new"].add(p["fs_new"])
        seen["order"].add(tuple(p["order"]))
    assert seen["fs_new"] == {4000, 8000, 16000} and len(seen["order"]) == 6


def test_packet_loss_indices_match_oracle():
    for seed in range(50):
        a, b = np.random.RandomState(seed), np.random.RandomState(seed)
        from unified_audio_b200.simulate import packet_loss_indices
        L = 3000 + 1777 * seed
        assert packet_loss_indices(a, L, 16000, 20, 0.05 + 0.004 * seed, 10) == osim.packet_loss_indices(b, L, 16000, 20,
                                                                                                         0.05 + 0.004 * seed, 10)


def test_refuses_bad_inputs():
    cfg = G.config(forced=True)
    with pytest.raises(ValueError, match="fs must be 16000"):
        Simulator(cfg, fs=8000)
    bad = G.config(forced=True)
    bad["bandwidth_limitation"]["fs_new"] = [11025]
    with pytest.raises(ValueError, match="fs_new"):
        Simulator(bad)
    sim = Simulator(cfg, seed=0)
    t = torch.zeros(100)           # checks run before any device work: CPU tensors show the argument errors first
    with pytest.raises(ValueError, match="mode"):
        sim.batch("ss", [t], [t], [t])
    with pytest.raises(ValueError, match="empty batch"):
        sim.batch("se", [], [], [])
    with pytest.raises(ValueError, match="interfering"):
        sim.batch("tse", [t], [t], [t], interf=[None], enroll=[t])
    with pytest.raises(ValueError, match="enrollment"):
        sim.batch("rtse", [t], [t], [t], interf=[t])
    with pytest.raises(ValueError, match="no enrollment"):
        sim.batch("se", [t], [t], [t], enroll=[t])
    with pytest.raises(ValueError, match="entries"):
        sim.batch("se", [t, t], [t], [t, t])
    with pytest.raises(ValueError, match="CUDA"):
        sim.batch("se", [t], [t], [t])
