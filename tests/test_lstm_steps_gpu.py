"""The LSTM recurrence (csrc/lstm_tc.cu, the wgmma kernel) step by step against fp64, teacher-forced: the h the kernel
publishes for step t - 1 is exactly its fp16 output out.hi[:, t - 1], so the reference takes the gates of step t from that h
(gates = xp_t + out.hi[:, t - 1] @ W16^T in fp64), carries the cell state c in fp64 along those gates and compares
out.hi + out.lo with o * tanh(c_t) at every step.  No fp16 knife edge can send the two trajectories apart, so each element
gets a derived error bound instead of a loose trajectory tolerance:

  gate pre-activation: fp32 accumulation of H fp16 products and the xp add, (H + 8) * 2^-23 * (sum |w| |h| + |xp|) (one ulp
                       per step rather than half, in case the tensor cores truncate);
  activations:         4e-7 absolute (lt_sigmoid / lt_tanh < 3e-7), propagated through sigmoid' and tanh' (plus their
                       second-order terms);
  cell state:          the bound of c_{t-1} times f, plus the gate errors times |c_{t-1}|, |g|, i, plus three fp32 roundings;
  output:              o * tanh(c) with both errors, one rounding and the hi / lo representation (2^-22 relative, and
                       2^-25 absolute: half the smallest fp16 subnormal, the resolution of lo for outputs near zero).

Coverage: every shipped instantiation (U = 4, 8, 12), batches with partial 32-row groups and second and third 128-row
launches, T = 1 (no recurrence), 2 and 48, saturating pre-activations, the single-plane output, a sentinel batch row after the
last one, and batch invariance: a row's output does not depend on the rows launched with it."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF_SENTINEL = -1234.0          # exact in fp16, never an LSTM output (|h| < 1)
U32 = 2.0 ** -24
ACT_EPS = 4e-7

# H -> units per CTA of lstm_tc on a 132-SM H100 (H / U CTAs co-resident)
TC_UNITS = {256: 4, 512: 4, 768: 8, 1024: 8, 1536: 12}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(B, T, H, seed, xscale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = 1.0 / math.sqrt(H)
    whh = (torch.rand(4 * H, H, generator=g, device=DEV) * 2 - 1) * k
    xp = torch.randn(B, T, 4 * H, generator=g, device=DEV) * xscale
    return whh, xp


def _teacher_forced(xp, w16, hi):
    """fp64 h_t from the kernel's own published h_{t-1}, and a per-element bound on |h_kernel - h_t|"""
    B, T, H = hi.shape
    hprev = torch.zeros(B, T, H, dtype=torch.float64, device=DEV)
    hprev[:, 1:] = hi[:, :-1].double()
    x64 = xp.double()
    a = x64 + hprev @ w16.t()
    ea = (H + 8) * 2 * U32 * (hprev.abs() @ w16.abs().t() + x64.abs())
    del hprev
    sig = torch.sigmoid
    c = torch.zeros(B, H, dtype=torch.float64, device=DEV)
    dc = torch.zeros_like(c)
    want = torch.empty(B, T, H, dtype=torch.float64, device=DEV)
    bound = torch.empty_like(want)
    for t in range(T):
        ai, af, ag, ao = a[:, t].chunk(4, -1)
        ei, ef, eg, eo = ea[:, t].chunk(4, -1)
        i, f, g, o = sig(ai), sig(af), torch.tanh(ag), sig(ao)
        di = (i * (1 - i) + 0.1 * ei) * ei + ACT_EPS           # |sigmoid''| < 0.1, |tanh''| < 0.77
        df = (f * (1 - f) + 0.1 * ef) * ef + ACT_EPS
        dg = (1 - g * g + 0.77 * eg) * eg + ACT_EPS
        do = (o * (1 - o) + 0.1 * eo) * eo + ACT_EPS
        cn = f * c + i * g
        dc = (f + df) * dc + c.abs() * df + g.abs() * di + (i + di) * dg + 3 * U32 * ((f * c).abs() + (i * g).abs()) + \
            U32 * cn.abs()
        c = cn
        tc = torch.tanh(c)
        want[:, t] = o * tc
        dt = (1 - tc * tc + 0.77 * dc) * dc + ACT_EPS
        bound[:, t] = tc.abs() * do + (o + do) * dt + 6 * U32 * (o * tc).abs() + 2.0 ** -25
    return want, bound


def _sentinel_out(B, T, H, split):
    from unified_audio_b200 import ops
    buf = torch.full((2, B + 1, T, H), HALF_SENTINEL, dtype=torch.float16, device=DEV)
    return ops.Planes(buf[0, :B], buf[1, :B] if split else None), buf


def _run(xp, whh, B, T, H, split):
    from unified_audio_b200 import ops
    out, buf = _sentinel_out(B, T, H, split)
    U = TC_UNITS[H]
    ws = torch.zeros(ops.lstm_tc_workspace_bytes(B, H), dtype=torch.uint8, device=DEV)
    ops.lstm_tc(xp, ops.lstm_tc_permute(whh, U), U, B, T, H, out, ws)
    torch.cuda.synchronize()
    return out, buf


def _check(B, T, H, seed, xscale=1.0):
    whh, xp = _inputs(B, T, H, seed, xscale)
    out, buf = _run(xp, whh, B, T, H, True)
    assert bool((buf[:, B] == HALF_SENTINEL).all()), "the row after the last batch row was written"
    got = out.hi.double() + out.lo.double()
    assert bool(torch.isfinite(got).all()), "non-finite output"
    want, bound = _teacher_forced(xp, whh.half().double(), out.hi)
    err = (got - want).abs()
    ratio = err / bound
    worst = float(ratio.max())
    # outputs within ~1e-7 of zero (o ~ sigmoid(-60) when saturated) sit on the 2^-25 floor of the lo plane's subnormals, where
    # the ratio says nothing about the arithmetic; it is also reported over the outputs in fp16's normal range
    sel = ratio[want.abs() >= 2.0 ** -14]
    normal = float(sel.max()) if sel.numel() else 0.0
    print(f"[lstm_tc H{H} B{B} T{T} x{xscale:g}] max |err| {float(err.max()):.2e}, worst error / bound {worst:.3e} "
          f"(|h| >= 2^-14: {normal:.3e})")
    assert worst <= 1.0, f"error {float(err.flatten()[ratio.argmax()]):.2e} at (b, t, j) = " \
                         f"{tuple(int(v) for v in torch.unravel_index(ratio.argmax(), ratio.shape))} exceeds its bound"
    return xp, whh, out


@pytest.mark.parametrize("T", [1, 2, 48])
@pytest.mark.parametrize("B", [1, 31, 32, 33, 97, 128, 129, 257])
@pytest.mark.parametrize("H", sorted(TC_UNITS))
def test_lstm_tc_teacher_forced(lib, H, B, T):
    if H // TC_UNITS[H] > _sms():
        pytest.skip(f"H {H} / U {TC_UNITS[H]} CTAs do not fit on {_sms()} SMs")
    _check(B, T, H, seed=H + 7 * B + T)


@pytest.mark.parametrize("H,B", [(256, 33), (512, 65), (768, 97), (1024, 1), (1024, 300), (1536, 129)])
def test_lstm_saturating_and_single_plane(lib, H, B):
    """Pre-activations to about +-60 (xp x 16): finite and within the same bound; then the same call with hi only (lo None)
    gives a bit-identical hi"""
    if H // TC_UNITS[H] > _sms():
        pytest.skip("instantiation pinned for a 132-SM H100")
    T = 48
    xp, whh, out = _check(B, T, H, seed=3 * H + B, xscale=16.0)
    assert float(xp.abs().max()) > 60
    one, buf = _run(xp, whh, B, T, H, False)
    assert torch.equal(one.hi, out.hi), "hi differs when the lo plane is not written"
    assert bool((buf[1] == HALF_SENTINEL).all()) and bool((buf[0, B] == HALF_SENTINEL).all())


@pytest.mark.parametrize("H", [512, 768, 1024])
def test_lstm_tc_batch_invariant_across_launches(lib, H):
    """B = 300 runs as launches of rows 0-127, 128-255 and 256-299; rows 0-43, 128-171 and 256-299 of it are bit for bit what
    those 44 rows give as a call of their own (one launch, two 32-row groups, the second partial)"""
    if H // TC_UNITS[H] > _sms():
        pytest.skip("instantiation pinned for a 132-SM H100")
    B, T = 300, 48
    whh, xp = _inputs(B, T, H, seed=11 * H)
    full, _ = _run(xp, whh, B, T, H, True)
    for r0 in (0, 128, 256):
        part, _ = _run(xp[r0:r0 + 44].contiguous(), whh, 44, T, H, True)
        for plane in ("hi", "lo"):
            a, b = getattr(full, plane)[r0:r0 + 44], getattr(part, plane)
            assert torch.equal(a, b), f"H {H}: rows {r0}-{r0 + 43} {plane} differ from their own call " \
                                      f"({int((a != b).sum())} elements)"


def test_lstm_tc_units_on_132_sms(lib):
    from unified_audio_b200 import ops
    if _sms() != 132:
        pytest.skip(f"units per CTA depend on the SM count ({_sms()} here, 132 on an H100 SXM)")
    assert {H: ops.lstm_tc_units(H) for H in TC_UNITS} == TC_UNITS
