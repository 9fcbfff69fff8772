"""oracle.simulate's last stages, `finish` (peak rule, cut, normalisation) and `enroll`, against the tail `apply` ran before they were
split out of it (kept below as it was), bit for bit in float32: on the inputs every fixture case hands them and on random rows.
The float32 results must stay float32 (NEP 50: a Python float meeting a np.float32 stays fp32), since the kernel tests compare
csrc/simulate.cu's finish_kernel and enroll_kernel with these functions bit for bit."""
import json

import numpy as np
import pytest

from oracle import make_golden_simulation as G
from oracle import simulate as osim

META = json.loads(bytes(np.load(G.OUT)["meta"]).decode())


def old_tail(noisy, speech, interf, enroll, p, cut, enroll_len):
    """apply's lines after the degradations, as they were before finish / enroll existed"""
    pad_or_cut = osim.pad_or_cut
    peak = max(np.max(np.abs(noisy)), np.max(np.abs(speech)))
    if interf is not None:
        peak = max(peak, np.max(np.abs(interf)))
    if peak > 0.99:
        noisy, speech = noisy / peak * 0.99, speech / peak * 0.99
        if interf is not None:
            interf = interf / peak * 0.99
    noisy, speech = pad_or_cut(noisy, cut, p["cut_offset"]), pad_or_cut(speech, cut, p["cut_offset"])
    if interf is None:
        tgt, src = np.max(np.abs(speech)) + 1e-5, np.max(np.abs(noisy)) + 1e-5
        factor = min((0.1 + (0.99 - 0.1) * p["norm_r"]) / tgt, 0.99 / max(tgt, src))
        noisy, speech = noisy * factor, speech * factor
    else:
        interf = pad_or_cut(interf, cut, p["cut_offset"])
        a, b, c = np.max(np.abs(noisy)), np.max(np.abs(speech)), np.max(np.abs(interf))
        factor = 0.99 / (max(a, b, c) + 1e-5)
        least = min(a, b, c)
        if least * factor > 0.1:
            lo = 0.1 / (least * factor)
            factor = (lo + (1 - lo) * p["norm_r"]) * factor
        noisy, speech, interf = noisy * factor, speech * factor, interf * factor
    if enroll is not None:
        enroll = pad_or_cut(enroll, enroll_len, p["enroll_offset"])
        enroll = enroll / (np.max(np.abs(enroll)) + 1e-5) * 0.99
    return noisy, speech, interf, enroll


def _same(new, old, f32):
    assert (new is None) == (old is None)
    if new is not None:
        assert new.dtype == old.dtype and (new.dtype == np.float32 or not f32)
        assert np.array_equal(new, old)


def _check(noisy, speech, interf, enroll, p, cut, enroll_len):
    """float32 inputs must give float32 results; after clipping apply's noisy is float64 (np.quantile), as the reference's is"""
    f32 = all(x is None or x.dtype == np.float32 for x in (noisy, speech, interf))
    on, os_, oi, oe = old_tail(noisy, speech, interf, enroll, p, cut, enroll_len)
    n, s, i = osim.finish(noisy, speech, interf, cut, p["cut_offset"], p["norm_r"])
    for new, old in ((n, on), (s, os_), (i, oi)):
        _same(new, old, f32)
        assert new is None or new.shape == (1, cut)
    if enroll is not None:
        e = osim.enroll(enroll, enroll_len, p["enroll_offset"])
        _same(e, oe, enroll.dtype == np.float32)
        assert e.shape == (1, enroll_len)


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_stages_match_old_tail_on_fixture_cases(name, monkeypatch):
    """the arguments apply hands finish / enroll on each fixture case, through both the new functions and the old tail"""
    seen = {}
    real_finish, real_enroll = osim.finish, osim._enroll

    def finish(*a):
        seen["finish"] = a
        return real_finish(*a)

    def enroll(*a):
        seen["enroll"] = a
        return real_enroll(*a)
    monkeypatch.setattr(osim, "finish", finish)
    monkeypatch.setattr(osim, "_enroll", enroll)
    p = G.recorded_params(name, META[name]["calls"])
    if p["norm_r"] is None:              # the reference drew no normalisation uniform: the value is not read
        p["norm_r"] = 0.0
    w = G.make_inputs(name)
    osim.apply(p, w["speech"], w["noise"], w["rir"], w["interf"], w["enroll"], cut=G.CUT, enroll_len=G.ENROLL, fs=G.FS)
    noisy, speech, interf, cut, cut_offset, norm_r = seen["finish"]
    assert cut == G.CUT and cut_offset == p["cut_offset"] and norm_r == p["norm_r"]
    e = seen.get("enroll")
    assert (e is None) == (w["enroll"] is None)
    if e is not None:
        assert e[1] == G.ENROLL and e[2] == p["enroll_offset"]
    _check(noisy, speech, interf, None if e is None else e[0], p, G.CUT, G.ENROLL)


def test_stages_match_old_tail_on_random_rows():
    g = np.random.default_rng(17)
    for t in range(300):
        cut = int(g.choice([1, 7, 300, 1024, 4000]))
        L = int(g.choice([1, 5, cut, cut + 1, 3 * cut + 11, int(g.integers(1, 5 * cut + 2))]))
        peak = float(g.choice([0.05, 0.5, 0.99, 1.0, 3.0]))
        row = lambda: (g.standard_normal(L) * peak / 3).astype(np.float32)[None]
        noisy, speech = row(), row()
        interf = row() if t % 2 else None
        if t % 7 == 0:
            speech[:] = 0
        Le = int(g.choice([1, 9, 2000, 5000]))
        enroll = (g.standard_normal(Le) * 0.2).astype(np.float32)[None]
        if t % 11 == 0:
            enroll[:] = 0
        p = {"cut_offset": int(g.integers(0, L - cut + 1)) if L >= cut else None,
             "enroll_offset": int(g.integers(0, Le - 2000 + 1)) if Le >= 2000 else None,
             "norm_r": float(g.choice([0.0, float(np.nextafter(1.0, 0.0)), g.random()]))}
        _check(noisy, speech, interf, enroll, p, cut, 2000)
