"""The simulation's last launches exactly, and every launch of a simulated batch on the inputs it received
(csrc/simulate.cu behind unified_audio_b200.Simulator).

sim_finish and sim_enroll use only correctly rounded fp32 operations (and one double expression the oracle rounds the same way), so
they must equal oracle.simulate.finish / enroll in float32 bit for bit.  sim_mix must equal its restatement on the rms vectors the
test passes in, except where CUDA's double pow may round the fp32 scale to the other neighbour (those rows are counted and printed).
Outputs start as NaN, inside NaN guard bands that must stay NaN.  Then whole batches run with every ops.sim_* launcher wrapped, and
each recorded launch is checked against the oracle on the exact inputs it received, with its flags, offsets and order checked
against the drawn parameters."""
import inspect
import itertools
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import make_golden_simulation as G
from oracle import simulate as osim
from test_simulation_gpu import FS, f64, i32, i64, pack, unpack

pytestmark = pytest.mark.gpu
F32 = np.float32
GUARD = 37
# norm_r values for which 0.1 + (0.99 - 0.1) * norm_r rounds to another fp32 level when the multiply-add is fused: finish_kernel
# once computed it with a contracted DFMA, and the FMA rows of test_finish_bit_exact caught it (its outputs were an ulp off).
FMA_NORM_R = [float.fromhex(h) for h in ("0x1.4be241fa3f47bp-5", "0x1.d960b76a6d4dbp-1", "0x1.9d060a61cc398p-1", "0x1.62e8605c0b7f6p-9",
                                         "0x1.2f74e54228451p-2")]


def up(v, k=1):
    """k fp32 ulps above v"""
    v = F32(v)
    for _ in range(k):
        v = np.nextafter(v, F32(np.inf))
    return v


def nan_out(rows, cols):
    """(buffer, [rows, cols] view): NaN everywhere, the view GUARD samples in from each end"""
    buf = torch.full((rows * cols + 2 * GUARD,), float("nan"), device="cuda")
    return buf, buf[GUARD:GUARD + rows * cols].view(rows, cols)


def assert_guards(buf):
    b = buf.cpu().numpy()
    assert np.isnan(b[:GUARD]).all() and np.isnan(b[-GUARD:]).all()


def shaped(g, L, peak, at):
    """a speech-like fp32 row of L samples whose largest |sample| is exactly `peak`, at index `at` (every other sample at most half)"""
    x = G.speech_like(g, L).astype(np.float64)
    m = np.abs(x).max()
    x = (x / m * 0.5 * float(peak) if m > 0 else x).astype(np.float32)
    if peak != 0:
        x[at] = -F32(peak) if at % 2 else F32(peak)
    return x


def least_at(target, M=0.8):
    """(M', least): fp32 peaks with fl32(least * factor) == target, factor = fl32(0.99 / fl32(M' + 1e-5)) as normalize_mix_speech_inferf
    computes it (M' the largest peak, least the smallest)"""
    for k in range(64):
        m = up(M, k)
        fac = F32(0.99) / (m + F32(1e-5))
        first = F32(target) / fac
        for j in range(-16, 17):
            cand = up(first, j) if j >= 0 else -up(-first, -j)
            if cand * fac == F32(target):
                return m, cand
    raise AssertionError(f"no fp32 peaks give least * factor == {target}")


# ------------------------------------------------------------------------------------------------------------------- sim_finish
def finish_rows(C):
    """[(label, noisy, speech, interf or None, cut_offset or None, norm_r)] for one launch of cut C: every case of the peak rule, the
    cut and both normalisation rules"""
    g = np.random.default_rng(C)
    long_L = 192000 if C == 80000 else C + 1500          # 12 s rows at the training cut
    rows = []

    def add(label, L, off, pk, r=0.37, at=None):
        """pk: (noisy, speech, interf or None) peaks, placed at `at` (default: inside the cut window)"""
        at = (L // 2 if off is None else off + min(C, L) // 2) if at is None else at
        sig = [None if p is None else shaped(g, L, p, at if p else 0) for p in pk]
        rows.append((label, sig[0], sig[1], sig[2], off, r))

    for interf in (None, 0.45):
        i = "" if interf is None else "+interf "
        add(i + "peak exactly 0.99f", long_L, 0, (F32(0.99), 0.5, interf))
        add(i + "peak one ulp above 0.99f", long_L, long_L - C, (0.5, up(0.99), interf))
        add(i + "peak outside the cut window", long_L, 1000, (0.3, 0.7, interf))
        rows[-1][1][10] = 2.5                               # before the window [1000, 1000 + C)
        add(i + "L == cut", C, 0, (0.6, 0.4, interf))
        add(i + "wrap L = 1", 1, None, (0.3, 0.2, interf))
        add(i + "wrap L = 7", 7, None, (1.4, 0.2, interf))
        add(i + "wrap, cut not a multiple of L", C // 3 + 1, None, (0.5, 0.7, interf))
        add(i + "peak rule with a long row", long_L, (long_L - C) // 3, (1.9, 3.1, interf))
    add("+interf peak only in interf", long_L, 17, (0.8, 0.6, 1.7))
    # normalize_src_tgt: min(level / tgt, 0.99 / max(tgt, src))
    add("src_tgt level side", long_L, 5, (0.4, 0.6, None), r=0.37)
    add("src_tgt peak side", long_L, 5, (0.9, 0.05, None), r=0.9)
    add("src_tgt norm_r = 0", long_L, 0, (0.4, 0.6, None), r=0.0)
    add("src_tgt norm_r just below 1", long_L, 0, (0.3, 0.6, None), r=float(np.nextafter(1.0, 0.0)))
    add("src_tgt all-zero speech", long_L, 0, (0.3, 0, None))
    add("src_tgt all zero", C // 2, None, (0, 0, None))
    for r in FMA_NORM_R:                    # level side, level < tgt < 1: an ulp of level moves the factor
        add(f"src_tgt fma norm_r {r:.6f}", long_L, 3, (0.5, 0.98, None), r=r)
    # normalize_mix_speech_inferf: rescale when fl32(least * factor) > 0.1f.  At equality the rescale would be the identity
    # (lo = 0.1f / 0.1f = 1, so factor * (1 + 0 * norm_r) = factor): `>` and `>=` give the same bits, and the equality rows pin the
    # arithmetic around the threshold rather than the comparison.
    add("inferf least = noisy", long_L, 0, (0.3, 0.6, 0.8), r=0.61)
    add("inferf least = speech", long_L, 0, (0.6, 0.3, 0.8), r=0.61)
    add("inferf least = interf", long_L, 0, (0.8, 0.6, 0.3), r=0.61)
    add("inferf least * factor < 0.1", long_L, 0, (0.8, 0.05, 0.6), r=0.61)
    for label, target in (("exactly 0.1f", F32(0.1)), ("one ulp above 0.1f", up(0.1))):
        M, least = least_at(target)
        fac = F32(0.99) / (M + F32(1e-5))
        assert least * fac == target and (least * fac > 0.1) == (target != F32(0.1))
        add(f"inferf least * factor {label}", long_L, 0, (M, 0.5, least), r=0.73)
        add(f"inferf least * factor {label}, least = noisy", long_L, 0, (least, M, 0.5), r=0.73)
    return rows


@pytest.mark.parametrize("C", [300, 4000, 80000])
def test_finish_bit_exact(lib, C):
    """three launches of the same rows: interferer buffer and out_interf given, out_interf NULL ('se'), and the rows without an
    interferer alone with both NULL; every output equals oracle.simulate.finish in float32, bit for bit"""
    from unified_audio_b200 import ops
    for r in FMA_NORM_R:
        fused = float(Fraction(0.1) + Fraction(0.99 - 0.1) * Fraction(r))
        assert F32(0.1 + (0.99 - 0.1) * r) != F32(fused)
    rows = finish_rows(C)
    B = len(rows)
    noisy, offs = pack([r[1] for r in rows])
    speech, _ = pack([r[2] for r in rows])
    interf, _ = pack([r[3] if r[3] is not None else np.full(len(r[1]), 1e3, np.float32) for r in rows])   # read only if has_interf
    has = [int(r[3] is not None) for r in rows]
    cut_off = [-1 if r[4] is None else r[4] for r in rows]
    want = [osim.finish(r[1][None], r[2][None], None if r[3] is None else r[3][None], C, r[4], r[5]) for r in rows]
    for k, (label, *_rest) in enumerate(rows):
        assert all(w is None or (w.dtype == np.float32 and w.shape == (1, C)) for w in want[k]), label

    def launch(sel, with_interf, with_out_interf):
        ins = [noisy, speech, interf] if sel is None else [pack([rows[b][c] for b in sel])[0] for c in (1, 2)] + [None]
        o = offs if sel is None else pack([rows[b][1] for b in sel])[1]
        idx = list(range(B)) if sel is None else sel
        n = len(idx)
        bufs = [nan_out(n, C) for _ in range(3)]
        ops.sim_finish(ins[0], ins[1], ins[2] if with_interf else None, o, n, i32([has[b] for b in idx]), i64([cut_off[b] for b in idx]),
                       f64([rows[b][5] for b in idx]), C, bufs[0][1], bufs[1][1], bufs[2][1] if with_out_interf else None)
        torch.cuda.synchronize()
        for buf, _ in bufs:
            assert_guards(buf)
        outs = [v.cpu().numpy() for _, v in bufs]
        for j, b in enumerate(idx):
            label = rows[b][0]
            assert np.array_equal(outs[0][j], want[b][0][0]), ("mix", label)
            assert np.array_equal(outs[1][j], want[b][1][0]), ("speech", label)
            if has[b] and with_out_interf:
                assert np.array_equal(outs[2][j], want[b][2][0]), ("interf", label)
            else:                                            # not written
                assert np.isnan(outs[2][j]).all(), ("interf", label)
    launch(None, True, True)
    launch(None, True, False)
    launch([b for b in range(B) if not has[b]], False, False)


# ------------------------------------------------------------------------------------------------------------------- sim_enroll
@pytest.mark.parametrize("C", [2000, 80000])
def test_enroll_bit_exact(lib, C):
    from unified_audio_b200 import ops
    g = np.random.default_rng(C + 1)
    long_L = 192000 if C == 80000 else 5000
    seam = C // 3 + 1                                               # wraps, C not a multiple of it
    rows = [("offset 0", shaped(g, long_L, 0.7, 40), 0),
            ("offset L - C", shaped(g, long_L, 0.4, long_L - 3), long_L - C),
            ("offset in the middle", shaped(g, long_L, 1.3, long_L // 2), (long_L - C) // 2),
            ("L == C", shaped(g, C, 0.2, C - 1), 0),
            ("wrap L = 1", np.array([-0.3], np.float32), None),
            ("wrap L = 1, zero", np.zeros(1, np.float32), None),
            ("wrap L = 7", shaped(g, 7, 0.9, 3), None),
            ("all zero", np.zeros(long_L, np.float32), 11),
            ("peak at the seam, last sample", shaped(g, seam, 0.8, seam - 1), None),
            ("peak at the seam, first sample", shaped(g, seam, 2.0, 0), None)]
    e, offs = pack([r[1] for r in rows])
    buf, out = nan_out(len(rows), C)
    ops.sim_enroll(e, offs, len(rows), i64([-1 if r[2] is None else r[2] for r in rows]), C, out)
    torch.cuda.synchronize()
    assert_guards(buf)
    got = out.cpu().numpy()
    for (label, x, off), y in zip(rows, got):
        want = osim.enroll(x[None], C, off)
        assert want.dtype == np.float32 and np.array_equal(y, want[0]), label


# ------------------------------------------------------------------------------------------------------------------- sim_mix
def mix_candidates(x, other, snr, rms_x, rms_o):
    """[(y, diff)] of the device's arithmetic: scale = fl32(10^(-snr/20) rms_x / (rms_o + 1e-10)) in double, y = fl32(fl32(other scale) + x),
    diff = fl32(y - x).  CUDA's double pow is not correctly rounded, so where the double scale lies within 16 double ulps of an fp32
    rounding boundary both fp32 neighbours are candidates."""
    s = 10 ** (-snr / 20) * rms_x / (rms_o + 1e-10)
    scales = sorted({F32(s * (1 - 16 * 2.0 ** -52)), F32(s), F32(s * (1 + 16 * 2.0 ** -52))})
    out = []
    for sc in scales:
        y = other * sc + x
        out.append((y, y - x))
    return out


def check_mix_row(x, other, snr, rms_x, rms_o, y, diff):
    """-> True when the row was a boundary row; asserts an exact match with one candidate (diff None: not checked)"""
    cands = mix_candidates(x, other, snr, rms_x, rms_o)
    assert any(np.array_equal(y, cy) and (diff is None or np.array_equal(diff, cd)) for cy, cd in cands)
    return len(cands) > 1


def test_mix_exact(lib):
    from unified_audio_b200 import ops
    g = np.random.default_rng(41)
    lens = [12 * FS, 4 * FS + 777, 1, 1023, 1025, 2048, 5000, 9 * FS + 3, 3000, 3000, 7000, 7000]
    x_rows = [G.speech_like(g, L) for L in lens]
    o_rows = [(0.2 * g.standard_normal(L)).astype(np.float32) if k % 2 else G.speech_like(g, L) for k, L in enumerate(lens)]
    snr = [float(v) for v in g.uniform(-5, 20, len(lens))]
    on = [1] * len(lens)
    snr[1], snr[5] = -80.0, 80.0                                       # large negative / positive SNR
    o_rows[8][:] = 0                                                   # rms_o = 0: the zero-noise case, y == x
    x_rows[9][:] = 0                                                   # rms_x = 0
    on[10] = on[11] = 0                                                # x and diff untouched
    rms_x = [osim.active_rms(r[None].astype(np.float64)) for r in x_rows]
    rms_o = [osim.active_rms(r[None].astype(np.float64)) for r in o_rows]
    assert rms_o[8] == 0 and rms_x[9] == 0
    x, offs = pack(x_rows)
    other, _ = pack(o_rows)
    x2 = x.clone()
    n = x.numel()
    dbuf = torch.full((n + 2 * GUARD,), float("nan"), device="cuda")
    diff = dbuf[GUARD:GUARD + n]
    args = (offs, len(lens), max(lens), f64(snr), f64(rms_x), f64(rms_o), i32(on))
    ops.sim_mix(x, other, *args, diff)
    ops.sim_mix(x2, other, *args)                                      # diff NULL
    torch.cuda.synchronize()
    assert_guards(dbuf)
    assert torch.equal(x, x2)
    boundary, worst = 0, 0.0
    for k, (y, d) in enumerate(zip(unpack(x, x_rows), unpack(diff, x_rows))):
        if not on[k]:
            assert np.array_equal(y, x_rows[k]) and np.isnan(d).all(), k
            continue
        boundary += check_mix_row(x_rows[k], o_rows[k], snr[k], rms_x[k], rms_o[k], y, d)
        if k == 8:
            assert np.array_equal(y, x_rows[k])
        ref = osim.mix(x_rows[k][None].astype(np.float64), o_rows[k][None].astype(np.float64), snr[k], None)[0]
        err = np.abs(y - ref).max() / max(np.abs(ref).max(), 1e-30)
        worst = max(worst, err)
        assert err < 1e-6, (k, err)
    print(f"sim_mix: {boundary} of {sum(on)} rows within 16 double ulps of an fp32 rounding boundary of the scale; "
          f"max |err| / row peak vs fp64 oracle.simulate.mix {worst:.2e}")


# ------------------------------------------------------------------------------------------------------------------- batches, launch by launch
def sim_launchers():
    """the ops.sim_* functions: one per qb_sim_* entry point of include/quark_b200.h"""
    from unified_audio_b200 import _lib, ops
    names = sorted(n.removeprefix("qb_") for n in _lib.SIGNATURES if n.startswith("qb_sim_"))
    assert names == sorted(n for n in dir(ops) if n.startswith("sim_")), names
    return names


class Launch:
    def __init__(self, name, before, after):
        self.name, self.before, self.after = name, before, after

    def np(self, key, when="before"):
        return getattr(self, when)[key].cpu().numpy()


class Recorder:
    """wraps every ops.sim_* function (simulate.py looks them up at call time): each call's tensor arguments are cloned before and
    after it runs (with a synchronize), in call order.  sim_active_rms is also given a mask buffer, so its non-silence flags can be
    checked; the flags are an optional output and the rms does not depend on them."""

    def __init__(self, monkeypatch):
        from unified_audio_b200 import ops
        self.calls = []
        for name in sim_launchers():
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))

    def _wrap(self, name, real):
        sig = inspect.signature(real)

        def call(*args, **kw):
            a = sig.bind(*args, **kw)
            a.apply_defaults()
            if name == "sim_active_rms" and a.arguments["mask"] is None:
                a.arguments["mask"] = torch.empty(a.arguments["x"].numel(), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            grab = lambda: {k: v.clone() for k, v in a.arguments.items() if isinstance(v, torch.Tensor)}
            before = {**grab(), **{k: v for k, v in a.arguments.items() if not isinstance(v, torch.Tensor)}}
            real(*a.args, **a.kwargs)
            torch.cuda.synchronize()
            self.calls.append(Launch(name, before, grab()))
        return call


def rows_of(a, lens):
    o = np.concatenate([[0], np.cumsum(lens)])
    return [a[o[k]:o[k + 1]] for k in range(len(lens))]


def cum(lens):
    return [0] + list(np.cumsum(lens))


def n_frames(L):
    """frames detect_non_silence pads a row of L samples to (0 below one frame)"""
    return 0 if L < 1024 else -(-(L - 1024) // 512) + 1


def expected_shift(L, Lo, offset):
    """the index shift of mix_noise's alignment: wrap padding puts other[0] at `offset`; a cut starts at `offset`"""
    if offset is None or Lo == 0:
        return 0
    return (Lo - offset % Lo) % Lo if Lo < L else offset


class Walk:
    """the recorded launches of one batch, taken in order and checked against the drawn parameters and the oracle"""

    def __init__(self, calls, params, w):
        self.calls, self.p, self.w = list(calls), params, w
        self.B = len(params)
        self.Ls = [len(x["speech"]) for x in w]
        self.boundary = 0
        self.worst = {"convolve": 0.0, "bandwidth": 0.0}

    def take(self, name, lens=None):
        """the next launch, which must be `name` over rows of `lens` samples (default: the utterances)"""
        assert self.calls, f"no launch left, expected {name}"
        c = self.calls.pop(0)
        assert c.name == name, (c.name, name)
        assert c.np("offs").tolist() == cum(self.Ls if lens is None else lens), name
        return c

    def rows(self, c, key, when="before"):
        return rows_of(c.np(key, when), self.Ls)

    def place(self, src_key, off_key, src_list):
        c = self.take("sim_place")
        Lo = [0 if s is None else len(s) for s in src_list]
        assert c.np("src_offs").tolist() == cum(Lo) and c.before["rows"] == self.B and c.before["max_len"] == max(self.Ls)
        assert np.array_equal(c.np("src"), np.concatenate([s for s in src_list if s is not None]))
        assert c.np("shift").tolist() == [expected_shift(L, n, p[off_key]) for L, n, p in zip(self.Ls, Lo, self.p)]
        for b, got in enumerate(self.rows(c, "dst", "after")):       # a row the stage skips (offset None) is placed from 0, unused
            off = 0 if self.p[b][off_key] is None else self.p[b][off_key]
            want = np.zeros(self.Ls[b], np.float32) if src_list[b] is None else osim.place(src_list[b][None], self.Ls[b], off)[0]
            assert np.array_equal(got, want), b
        return c

    def active_rms(self, x):
        c = self.take("sim_active_rms")
        assert torch.equal(c.before["x"], x)
        F = [n_frames(L) for L in self.Ls]
        assert c.np("frame_off").tolist() == cum(F) and c.before["max_frames"] == max(F)
        for b, (r, m) in enumerate(zip(self.rows(c, "x"), self.rows(c, "mask", "after"))):
            r64 = r[None].astype(np.float64)
            assert np.array_equal(m.astype(bool), osim.non_silence(r64)[0]), b
            ref, got = osim.active_rms(r64), c.np("rms", "after")[b]
            assert abs(got - ref) <= 1e-9 * max(ref, 1e-30), b
        return c.after["rms"]

    def mix(self, x, placed, rms_x, rms_o, level_key, flags, diff):
        c = self.take("sim_mix")
        assert torch.equal(c.before["x"], x) and torch.equal(c.before["other"], placed)
        assert torch.equal(c.before["rms_x"], rms_x) and torch.equal(c.before["rms_other"], rms_o)
        assert c.np("snr").tolist() == [p[level_key] for p in self.p] and c.np("on").tolist() == flags
        assert (c.before["diff"] is None) == (not diff)
        snr, rx, ro = c.np("snr"), c.np("rms_x"), c.np("rms_other")
        xs, os_, ys = self.rows(c, "x"), self.rows(c, "other"), self.rows(c, "x", "after")
        ds = self.rows(c, "diff", "after") if diff else [None] * self.B
        d0 = self.rows(c, "diff") if diff else [None] * self.B
        for b in range(self.B):
            if not flags[b]:
                assert np.array_equal(ys[b], xs[b]) and (d0[b] is None or np.array_equal(ds[b], d0[b])), b
                continue
            self.boundary += check_mix_row(xs[b], os_[b], float(snr[b]), float(rx[b]), float(ro[b]), ys[b], ds[b])
        return c

    def convolve(self, x, hn, win, flags):
        c = self.take("sim_convolve")
        assert torch.equal(c.before["x"], x) and torch.equal(c.before["h"], hn) and c.np("on").tolist() == flags
        assert (win is None and c.before["win"] is None) or torch.equal(c.before["win"], win)
        Lr = [len(x["rir"]) for x in self.w]
        assert c.np("h_offs").tolist() == cum(Lr)
        hs, ws = rows_of(hn.cpu().numpy(), Lr), None if win is None else win.cpu().numpy()
        for b, (r, got) in enumerate(zip(self.rows(c, "x"), self.rows(c, "y", "after"))):
            if not flags[b]:
                assert np.array_equal(got, r), b
                continue
            h = hs[b].astype(np.float64)
            if ws is not None:
                s, e = ws[b]
                h = np.concatenate([np.zeros(s), h[s:e], np.zeros(len(h) - e)])
            ref = osim.reverb(r[None].astype(np.float64), h[None])[0]
            err = np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)
            self.worst["convolve"] = max(self.worst["convolve"], err)
            assert err < 1e-5, (b, err)
        return c.after["y"]

    def degradation(self, kind, x):
        """one slot's launch of one degradation kind -> (x after, rows it applied to)"""
        name = {0: "sim_bandwidth", 1: "sim_clip", 2: "sim_packet_loss"}[kind]
        c = self.take(name)
        assert torch.equal(c.before["x"], x)
        xs, ys = self.rows(c, "x"), self.rows(c, "x", "after")
        if kind == 2:
            lost, lrow = c.np("lost").tolist(), c.np("lost_row").tolist()
            assert c.before["packet"] == 320
            on = sorted(set(lrow))
        else:
            on = [b for b, f in enumerate(c.np("on").tolist()) if f]
        for b in range(self.B):
            if b not in on:
                assert np.array_equal(ys[b], xs[b]), (name, b)
            elif kind == 0:
                fs_new = int(c.np("fs_new")[b])
                assert fs_new == self.p[b]["fs_new"]
                if fs_new == FS:
                    assert np.array_equal(ys[b], xs[b])
                    continue
                ref = osim.bandwidth(xs[b][None].astype(np.float64), FS, fs_new)[0]
                err = np.abs(ys[b] - ref).max() / max(np.abs(ref).max(), 1e-30)
                self.worst["bandwidth"] = max(self.worst["bandwidth"], err)
                assert err < 1e-5, (b, err)
            elif kind == 1:
                q = c.np("q")
                assert q[2 * b] == self.p[b]["min_q"] and q[2 * b + 1] == self.p[b]["max_q"]
                assert np.array_equal(ys[b], osim.clip(xs[b][None], q[2 * b], q[2 * b + 1])[0].astype(np.float32)), b
            else:
                mine = [j for j, r in zip(lost, lrow) if r == b]
                assert mine == self.p[b]["lost"], b
                assert np.array_equal(ys[b], osim.packet_loss(xs[b][None], mine)[0]), b
        return c.after["x"], on


def batch_inputs(seed, mode, B, some_interf):
    """bench-length utterances (4-12 s), RIRs of 0.3-1.5 s, noise of 0.5-14 s; in 'se' an interferer on even rows when some_interf"""
    g = np.random.default_rng(seed)
    w = []
    for i in range(B):
        w.append({"speech": G.speech_like(g, int(g.integers(4 * FS, 12 * FS))),
                  "noise": (0.2 * g.standard_normal(int(g.integers(FS // 2, 14 * FS)))).astype(np.float32),
                  "rir": G.rir_like(g, "delayed", int(g.integers(int(0.3 * FS), int(1.5 * FS)))),
                  "interf": G.speech_like(g, int(g.integers(FS, 12 * FS))) if mode != "se" or (some_interf and i % 2 == 0) else None,
                  "enroll": G.speech_like(g, int(g.integers(2 * FS, 9 * FS))) if mode != "se" else None})
    return w


BATCHES = {          # name: (mode, forced config, rows, every slot order)
    "se_forced_some_interf": ("se", True, 6, False),
    "se_shipped": ("se", False, 6, False),
    "tse_forced": ("tse", True, 5, False),
    "tse_shipped": ("tse", False, 6, False),
    "rtse_forced": ("rtse", True, 5, False),
    "rtse_shipped": ("rtse", False, 6, False),
    "tse_every_order": ("tse", True, 6, True),
}


@pytest.mark.parametrize("name", sorted(BATCHES))
def test_batch_launch_by_launch(lib, monkeypatch, name):
    """Simulator.apply with every launcher recorded: each launch against the oracle on its own recorded inputs (teacher-forced), and
    its flags, offsets, level vectors and place in the sequence against the drawn parameters"""
    from unified_audio_b200.simulate import Simulator
    mode, forced, B, every_order = BATCHES[name]
    w = batch_inputs(sorted(BATCHES).index(name) + 50, mode, B, True)
    sim = Simulator(G.config(forced=forced), seed=7)
    cut, enroll_len = 80000, 80000
    params = [sim.draw(mode, len(x["speech"]), len(x["noise"]), None if x["interf"] is None else len(x["interf"]),
                       None if x["enroll"] is None else len(x["enroll"]), cut, enroll_len) for x in w]
    if every_order:                              # bandwidth, clipping and packet loss in each of the six slot orders
        for p, order in zip(params, itertools.permutations(range(3))):
            p["order"] = list(order)
    ins = {k: [None if x[k] is None else torch.from_numpy(x[k]).cuda() for x in w] for k in w[0]}
    rec = Recorder(monkeypatch)
    out = sim.apply(params, ins["speech"], ins["noise"], ins["rir"], ins["interf"], ins["enroll"] if mode != "se" else None, cut,
                    enroll_len)
    names = {c.name for c in rec.calls}
    if forced and mode != "se":
        assert names == set(sim_launchers()), sorted(set(sim_launchers()) - names)

    v = Walk(rec.calls, params, w)
    speech = torch.from_numpy(np.concatenate([x["speech"] for x in w])).cuda()
    noisy, x_interf = speech, None
    has_i = [int(p["interf"]) for p in params]
    assert has_i == [int(x["interf"] is not None) for x in w]
    if any(has_i):
        placed = v.place("interf", "interf_offset", [x["interf"] for x in w]).after["dst"]
        rms_x, rms_o = v.active_rms(speech), v.active_rms(placed)
        c = v.mix(noisy, placed, rms_x, rms_o, "sir", has_i, True)
        assert not c.before["diff"].any()                 # zero-filled: rows without an interferer keep interf = 0
        noisy, x_interf = c.after["x"], c.after["diff"]
    reverb = [int(p["reverb"]) for p in params]
    if any(reverb):
        Lr = [len(x["rir"]) for x in w]
        c = v.take("sim_rir_prep", Lr)
        assert c.np("on").tolist() == reverb
        hn, win = c.after["hn"], c.after["win"]
        for b, (r, got) in enumerate(zip(w, rows_of(hn.cpu().numpy(), Lr))):
            if reverb[b]:
                want = r["rir"] / (np.max(np.abs(r["rir"])) + F32(1e-5))
                assert np.array_equal(got, want) and int(c.np("status", "after")[b]) == 0, b
                assert tuple(win[b].tolist()) == osim.rir_window(want), b
        noisy = v.convolve(noisy, hn, None, reverb)
        speech = v.convolve(speech, hn, win, reverb)
        if x_interf is not None:
            x_interf = v.convolve(x_interf, hn, win, [a * b for a, b in zip(reverb, has_i)])
    noise = [int(p["noise"]) for p in params]
    if any(noise):
        placed = v.place("noise", "noise_offset", [x["noise"] for x in w]).after["dst"]
        rms_x, rms_o = v.active_rms(noisy), v.active_rms(placed)
        noisy = v.mix(noisy, placed, rms_x, rms_o, "snr", noise, False).after["x"]
    applied = [[] for _ in range(v.B)]
    for s in range(3):                                   # slot s: each row's order[s], when its coin came up
        for kind in range(3):                            # packet loss: rows with packets to drop
            rows = [b for b, p in enumerate(params) if p["order"][s] == kind and p["apply"][s] and (kind != 2 or p["lost"])]
            if rows:
                noisy, on = v.degradation(kind, noisy)
                assert on == rows, (s, kind)
                for b in on:
                    applied[b].append(kind)
    for b, p in enumerate(params):                       # each row's degradations in its shuffled order
        assert applied[b] == [k for k, a in zip(p["order"], p["apply"]) if a and (k != 2 or p["lost"])], (b, p["order"], p["apply"])
    if every_order:
        assert {tuple(p["order"]) for p in params} == set(itertools.permutations(range(3)))
        assert all(len(a) == 3 for a in applied)

    c = v.take("sim_finish")
    assert torch.equal(c.before["noisy"], noisy) and torch.equal(c.before["speech"], speech)
    assert (x_interf is None and c.before["interf"] is None) or torch.equal(c.before["interf"], x_interf)
    assert c.np("has_interf").tolist() == has_i and c.before["cut"] == cut
    assert c.np("cut_off").tolist() == [-1 if p["cut_offset"] is None else p["cut_offset"] for p in params]
    assert c.np("norm_r").tolist() == [p["norm_r"] for p in params]
    assert (c.before["out_interf"] is None) == (mode == "se")
    ns, ss = v.rows(c, "noisy"), v.rows(c, "speech")
    is_ = v.rows(c, "interf") if x_interf is not None else None
    for b, p in enumerate(params):
        want = osim.finish(ns[b][None], ss[b][None], is_[b][None] if has_i[b] else None, cut, p["cut_offset"], float(p["norm_r"]))
        assert np.array_equal(c.np("out_mix", "after")[b], want[0][0]), b
        assert np.array_equal(c.np("out_speech", "after")[b], want[1][0]), b
        if mode != "se":
            assert np.array_equal(c.np("out_interf", "after")[b], want[2][0]), b
    assert torch.equal(out[2], c.after["out_mix"]) and torch.equal(out[3], c.after["out_speech"])
    assert (out[4] is None) == (mode == "se") and (out[4] is None or torch.equal(out[4], c.after["out_interf"]))
    if mode != "se":
        Le = [len(x["enroll"]) for x in w]
        c = v.take("sim_enroll", Le)
        assert c.before["cut"] == enroll_len
        assert c.np("cut_off").tolist() == [-1 if p["enroll_offset"] is None else p["enroll_offset"] for p in params]
        for b, (x, p) in enumerate(zip(w, params)):
            want = osim.enroll(x["enroll"][None], enroll_len, p["enroll_offset"])
            assert np.array_equal(c.np("out", "after")[b], want[0]), b
        assert torch.equal(out[1], c.after["out"])
    assert not v.calls, [c.name for c in v.calls]
    print(f"{name}: {len(rec.calls)} launches {sorted(names)}; sim_mix boundary rows {v.boundary}; max |err| / row peak vs fp64",
          {k: f"{e:.2e}" for k, e in v.worst.items()})
