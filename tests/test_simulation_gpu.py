"""UniSE training-data simulation on the GPU (csrc/simulate.cu behind unified_audio_b200.Simulator).

Each kernel against oracle/simulate.py in fp64 at the bench shape (utterances of 4-12 s, RIRs up to 1.5 s) and at edge shapes: the
non-silence mask identical (the smallest |power / mean - 0.01| margin reported), RIR windows identical, quantiles and clipped samples
exact, packet-loss zeros exactly placed, cut / wrap placement exact, convolution and resampling within 1e-5 of each row's peak (with
the fp32 oracle's own gap to fp64 reported).  Then whole batches against the reference-pinned fixture and the fp64 oracle in every
mode, bit-identical repeats, independence from the lengths run before, and Model.training_step on a simulated batch."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import make_golden_simulation as G
from oracle import simulate as osim

pytestmark = pytest.mark.gpu
FS = 16000


def pack(rows, dtype=torch.float32):
    offs = torch.tensor([0] + list(np.cumsum([len(r) for r in rows])), dtype=torch.int64, device="cuda")
    buf = torch.from_numpy(np.concatenate([np.asarray(r, dtype=np.float32) for r in rows])).to("cuda", dtype)
    return buf, offs


def unpack(buf, rows):
    out, o, b = [], 0, buf.cpu().numpy()
    for r in rows:
        out.append(b[o:o + len(r)])
        o += len(r)
    return out


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def i64(v):
    return torch.tensor(v, dtype=torch.int64, device="cuda")


def f64(v):
    return torch.tensor(v, dtype=torch.float64, device="cuda")


def speech_rows(seed, lengths):
    g = np.random.default_rng(seed)
    return [G.speech_like(g, L) for L in lengths]


BENCH_LEN = [int(L) for L in np.random.default_rng(7).integers(4 * FS, 12 * FS, 8)]
EDGE_LEN = [1, 800, 1023, 1024, 1025, 1536, 2047, 5000]


def frames(L):
    return 0 if L < 1024 else (L + (-(L - 1024)) % 512 % 1024 - 1024) // 512 + 1


# ------------------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("shape", ["bench", "edge"])
def test_non_silence_and_rms_vs_fp64(lib, shape):
    from unified_audio_b200 import ops
    rows = speech_rows(1, BENCH_LEN if shape == "bench" else EDGE_LEN)
    rows.append(np.zeros(3000, dtype=np.float32))                        # all-zero row: every sample counts
    x, offs = pack(rows)
    F = [frames(len(r)) for r in rows]
    fo = i64([0] + list(np.cumsum(F)))
    rms, mask = torch.empty(len(rows), dtype=torch.float64, device="cuda"), torch.empty(x.numel(), dtype=torch.uint8, device="cuda")
    ops.sim_active_rms(x, offs, fo, len(rows), max(map(len, rows)), max(F), rms, mask)
    margin = min(osim.non_silence_margin(r[None].astype(np.float64)) for r in rows)
    print(f"non-silence: smallest |power / mean - 0.01| = {margin:.3e}")
    for r, m, got in zip(rows, unpack(mask, rows), rms.cpu().numpy()):
        want = osim.non_silence(r[None].astype(np.float64))[0]
        assert np.array_equal(m.astype(bool), want)
        ref = osim.active_rms(r[None].astype(np.float64))
        assert abs(got - ref) <= 1e-9 * max(ref, 1e-30)


def test_place_vs_oracle(lib):
    from unified_audio_b200 import ops
    from unified_audio_b200.simulate import _shift
    speech = speech_rows(2, [9000, 4000, 16000, 700])
    g = np.random.default_rng(3)
    other = [g.standard_normal(n).astype(np.float32) for n in (2500, 9000, 40000, 700)]
    offsets = [1234, 3100, 20000, None]
    x, offs = pack(speech)
    o, o_offs = pack(other)
    placed = torch.empty_like(x)
    ops.sim_place(o, o_offs, offs, i64([_shift(len(s), len(t), k) for s, t, k in zip(speech, other, offsets)]), 4, 16000, placed)
    for got, s, t, k in zip(unpack(placed, speech), speech, other, offsets):
        assert np.array_equal(got, osim.place(t[None], len(s), k)[0])


@pytest.mark.parametrize("shape", ["bench", "edge"])
def test_rir_window_and_convolution_vs_fp64(lib, shape):
    from unified_audio_b200 import ops
    g = np.random.default_rng(4)
    if shape == "bench":
        lens, rl = BENCH_LEN[:4], [int(0.3 * FS), int(0.8 * FS), int(1.0 * FS), int(1.5 * FS)]
    else:
        lens, rl = [700, 1500, 3000, 5000], [1, 2, 300, 2500]
    x_rows = speech_rows(5, lens)
    rirs = [G.rir_like(g, "delayed" if i % 2 == 0 else "no_fall", n) if n > 50 else g.standard_normal(n).astype(np.float32)
            for i, n in enumerate(rl)]
    if shape == "edge":
        rirs[0] = np.array([0.7], dtype=np.float32)                          # peak at sample 0 of a 1-tap RIR: status 1
        rirs[1] = np.array([0.5, -0.25], dtype=np.float32)
        rirs[2][[40, 90]] = 3.0                                              # a tie: the first occurrence is the peak
    x, offs = pack(x_rows)
    h, h_offs = pack(rirs)
    B = len(x_rows)
    hn, win, status = torch.empty_like(h), torch.empty(B, 2, dtype=torch.int64, device="cuda"), torch.empty(B, dtype=torch.int32,
                                                                                                             device="cuda")
    on = i32([1] * B)
    ops.sim_rir_prep(h, h_offs, B, on, hn, win, status)
    for b, (r, got_hn) in enumerate(zip(rirs, unpack(hn, rirs))):
        want = r / (np.max(np.abs(r)) + np.float32(1e-5))
        assert np.array_equal(got_hn, want)
        peak = int(np.argmax(np.abs(want)))
        assert int(status[b]) == (peak == len(r) - 1)
        if peak < len(r) - 1:
            assert tuple(win[b].tolist()) == osim.rir_window(want)
    ok = [b for b in range(B) if int(status[b]) == 0]
    worst = {"full": 0.0, "early": 0.0, "fp32_oracle_full": 0.0}
    for kind, w in (("full", None), ("early", win)):
        y = torch.empty_like(x)
        ops.sim_convolve(x, offs, B, max(lens), hn, h_offs, w, i32([int(b in ok) for b in range(B)]), y)
        for b, got in enumerate(unpack(y, x_rows)):
            hb = unpack(hn, rirs)[b].astype(np.float64)
            if b not in ok:
                assert np.array_equal(got, x_rows[b])
                continue
            if kind == "early":
                s, e = win[b].tolist()
                hb = np.concatenate([np.zeros(s), hb[s:e], np.zeros(len(hb) - e)])
            ref = osim.reverb(x_rows[b][None].astype(np.float64), hb[None])[0]
            peak = max(np.abs(ref).max(), 1e-30)
            err = np.abs(got - ref).max() / peak
            worst[kind] = max(worst[kind], err)
            assert err < 1e-5, (kind, b, err)
            if kind == "full":
                f32 = osim.reverb(x_rows[b][None], hb[None].astype(np.float32))[0]
                worst["fp32_oracle_full"] = max(worst["fp32_oracle_full"], np.abs(f32 - ref).max() / peak)
    print("convolution: max |err| / row peak vs fp64", json.dumps(worst))


@pytest.mark.parametrize("shape", ["bench", "edge"])
def test_bandwidth_vs_fp64(lib, shape):
    from unified_audio_b200 import ops
    from unified_audio_b200.simulate import Simulator
    lens = BENCH_LEN[:6] if shape == "bench" else [1, 3, 5, 700, 1025, 4001]
    rows = speech_rows(6, lens)
    fs_new = [4000, 8000, 16000, 4000, 8000, 4000]
    on = [1, 1, 1, 1, 0, 1]
    x, offs = pack(rows)
    tmp = torch.empty_like(x)
    sim = Simulator(G.config(forced=True))
    ops.sim_bandwidth(x, offs, len(rows), max(lens), i32(fs_new), i32(on), sim._resample_taps(x.device), tmp)
    worst, worst32 = 0.0, 0.0
    for r, got, f, o in zip(rows, unpack(x, rows), fs_new, on):
        if not o or f == FS:
            assert np.array_equal(got, r)
            continue
        ref = osim.bandwidth(r[None].astype(np.float64), FS, f)[0]
        peak = max(np.abs(ref).max(), 1e-30)
        worst = max(worst, np.abs(got - ref).max() / peak)
        worst32 = max(worst32, np.abs(osim.bandwidth(r[None], FS, f)[0] - ref).max() / peak)
    print(f"bandwidth: max |err| / row peak vs fp64 {worst:.2e} (fp32 oracle {worst32:.2e})")
    assert worst < 1e-5


@pytest.mark.parametrize("shape", ["bench", "edge"])
def test_clip_exact(lib, shape):
    from unified_audio_b200 import ops
    lens = BENCH_LEN[:4] if shape == "bench" else [1, 2, 3, 10, 1000, 4097]
    rows = speech_rows(8, lens)
    rows[0][::7] = 0.0                                                   # ties and signed zeros, as packet loss leaves them
    if shape == "edge":
        rows[3][:] = 0.25                                                # all equal
    q = [(0.0, 1.0), (0.05, 0.95), (0.1, 0.9), (0.0371, 0.9123), (0.1, 1.0), (0.0, 0.9)][:len(rows)]
    x, offs = pack(rows)
    stats = torch.empty(len(rows), 4, device="cuda")
    ops.sim_clip(x, offs, len(rows), max(lens), f64([v for p in q for v in p]), i32([1] * len(rows)), stats)
    for r, got, (a, b), s in zip(rows, unpack(x, rows), q, stats.cpu().numpy()):
        srt = np.sort(r)
        for k, qq in enumerate((a, b)):
            v = (len(r) - 1) * qq
            lo = min(int(math.floor(v)), len(r) - 1)
            assert s[2 * k] == srt[lo] and s[2 * k + 1] == srt[min(lo + 1, len(r) - 1)]
        want = osim.clip(r[None], a, b)[0].astype(np.float32)
        assert np.array_equal(got, want)


def test_packet_loss_exact(lib):
    from unified_audio_b200 import ops
    from unified_audio_b200.simulate import packet_loss_indices
    rows = speech_rows(9, BENCH_LEN[:3] + [900, 330])
    lost = [packet_loss_indices(np.random.RandomState(i), len(r), FS, 20, 0.25, 10) for i, r in enumerate(rows)]
    lost[3] = [0, 2, 5]                                                  # packets past the end of a short row
    flat = [(b, j) for b, l in enumerate(lost) for j in l]
    x, offs = pack(rows)
    ops.sim_packet_loss(x, offs, i64([j for _, j in flat]), i32([b for b, _ in flat]), 320)
    for r, got, l in zip(rows, unpack(x, rows), lost):
        assert np.array_equal(got, osim.packet_loss(r[None], l)[0])


# ------------------------------------------------------------------------------------------------------------------- batches
def _gpu_inputs(w_list):
    c = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return {k: [c(w[k]) for w in w_list] for k in ("speech", "noise", "rir", "interf", "enroll")}


def _close(got, want, tol):
    """max |got - want| over the row's peak, per row"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30)) <= tol


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_batch_vs_reference_fixture(lib, name):
    """the reference's own outputs (tests/golden/simulation_small.npz) from its recorded draws, through Simulator.apply"""
    from unified_audio_b200.simulate import Simulator
    z = np.load(G.OUT)
    meta = json.loads(bytes(z["meta"]).decode())
    p = G.recorded_params(name, meta[name]["calls"])
    if p["norm_r"] is None:                  # the reference's normalisation needed no draw: the device ignores it
        p["norm_r"] = 0.0
    w = G.make_inputs(name)
    sim = Simulator(G.config(**G.CASES[name][2]))
    ins = _gpu_inputs([w])
    mode, enroll, mix, speech, interf, fs, lengths, names = sim.apply(
        [p], ins["speech"], ins["noise"], ins["rir"], ins["interf"], ins["enroll"] if p["mode"] != "se" else None, G.CUT, G.ENROLL)
    assert mode == p["mode"] and int(fs[0]) == FS and int(lengths[0]) == G.CUT
    outs = {"mix": mix, "speech": speech, "interf": interf, "enroll": enroll}
    for k, t in outs.items():
        if t is None:
            assert k in ("interf", "enroll") and mode == "se"
            continue
        assert _close(t[0].cpu().numpy(), z[f"{name}/{k}"], 1e-4), (k, name)


def _random_batch(seed, mode, B, forced):
    g = np.random.default_rng(seed)
    lens = [int(L) for L in g.integers(1 * FS, 12 * FS, B)]
    w = []
    for i, L in enumerate(lens):
        rl = int(g.integers(int(0.3 * FS), int(1.5 * FS)))
        w.append({"speech": G.speech_like(g, L), "noise": (0.2 * g.standard_normal(int(g.integers(FS // 2, 14 * FS)))).astype(np.float32),
                  "rir": G.rir_like(g, "delayed", rl),
                  "interf": G.speech_like(g, int(g.integers(FS, 12 * FS))) if (mode != "se" or i % 2 == 0) else None,
                  "enroll": G.speech_like(g, int(g.integers(2 * FS, 9 * FS))) if mode != "se" else None})
    return w


@pytest.mark.parametrize("mode", ["se", "tse", "rtse"])
@pytest.mark.parametrize("forced", [True, False])
def test_batch_vs_fp64_oracle(lib, mode, forced):
    from unified_audio_b200.simulate import Simulator
    B = 6
    w = _random_batch(10 + forced, mode, B, forced)
    sim = Simulator(G.config(forced=forced), seed=3)
    ins = _gpu_inputs(w)
    out = sim.batch(mode, ins["speech"], ins["noise"], ins["rir"], ins["interf"], ins["enroll"] if mode != "se" else None,
                    cut_duration=5.0, enroll_duration=5.0)
    again = Simulator(G.config(forced=forced), seed=3)
    params = [again.draw(mode, len(x["speech"]), len(x["noise"]), None if x["interf"] is None else len(x["interf"]),
                         None if x["enroll"] is None else len(x["enroll"]), 80000, 80000) for x in w]
    for b, (x, p) in enumerate(zip(w, params)):
        e, m, s, i = osim.apply(p, x["speech"], x["noise"], x["rir"], x["interf"], x["enroll"], cut=80000, enroll_len=80000, fp64=True)
        assert _close(out[2][b].cpu().numpy(), m, 1e-4) and _close(out[3][b].cpu().numpy(), s, 1e-4), (b, p)
        if mode != "se":
            assert _close(out[4][b].cpu().numpy(), i, 1e-4) and _close(out[1][b].cpu().numpy(), e, 1e-4), (b, p)
    # the same draws on the same inputs give the same bits
    rep = again.apply(params, ins["speech"], ins["noise"], ins["rir"], ins["interf"], ins["enroll"] if mode != "se" else None, 80000, 80000)
    for a, b in zip(out[1:5], rep[1:5]):
        assert (a is None and b is None) or torch.equal(a, b)


def test_call_history_does_not_matter(lib):
    """a batch after one of other lengths equals the same batch on a fresh Simulator, bit for bit"""
    from unified_audio_b200.simulate import Simulator
    first, second = _random_batch(20, "tse", 5, True), _random_batch(21, "tse", 5, True)
    sim = Simulator(G.config(forced=True), seed=9)
    a = _gpu_inputs(first)
    sim.batch("tse", a["speech"], a["noise"], a["rir"], a["interf"], a["enroll"])
    state = (sim.rng.getstate(), sim.nprng.get_state())
    b = _gpu_inputs(second)
    got = sim.batch("tse", b["speech"], b["noise"], b["rir"], b["interf"], b["enroll"])
    fresh = Simulator(G.config(forced=True))
    fresh.rng.setstate(state[0])
    fresh.nprng.set_state(state[1])
    want = fresh.batch("tse", b["speech"], b["noise"], b["rir"], b["interf"], b["enroll"])
    for x, y in zip(got[1:5], want[1:5]):
        assert torch.equal(x, y)


def test_refuses_rir_peaking_at_its_end(lib):
    from unified_audio_b200.simulate import Simulator
    cfg = G.config(forced=True)
    sim = Simulator(cfg, seed=0)
    s = torch.from_numpy(G.speech_like(np.random.default_rng(0), 4000)).cuda()
    rir = torch.tensor([0.1, 0.2, 1.0], device="cuda")
    with pytest.raises(ValueError, match="last sample"):
        sim.batch("se", [s], [s.clone()], [rir], cut_duration=0.1)


@pytest.mark.parametrize("mode", ["se", "tse"])
def test_training_step_on_simulated_batch(lib, mode):
    from test_unise_validation_gpu import build_small
    from unified_audio_b200.simulate import Simulator
    model, z, _ = build_small()
    T = z["e2e_wav"].shape[1]
    w = _random_batch(30, mode, 2, False)
    for x in w:                                   # short utterances keep the small model's sequence lengths small
        x["speech"] = x["speech"][:2 * T]
        if x["interf"] is not None:
            x["interf"] = x["interf"][:3 * T]
    ins = _gpu_inputs(w)
    sim = Simulator(G.config(forced=False), seed=1)
    batch = sim.batch(mode, ins["speech"], ins["noise"], ins["rir"], ins["interf"], ins["enroll"] if mode != "se" else None,
                      cut_duration=T / FS, enroll_duration=4800 / FS)
    model.dnn.requires_grad_(True)
    out = model.training_step(batch, 0, dropout_seed=5)
    assert math.isfinite(float(out["loss"].detach()))
    out["loss"].backward()
