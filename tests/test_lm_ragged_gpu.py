"""LLM_SFT.generate with ragged conditioning prefixes (`enroll_lengths`): rows whose enrollments differ in length decode in one call,
with one position per row in the decode kernels (qb_lm_decode_layer_tc / qb_lm_head_{argmax,sample}_tc).  Reduced widths,
as tests/test_lm_kernels_gpu.py.

Every comparison holds the decode attention's keys in flight (att_unroll / lane_att_unroll) equal on both sides: 8 on a single chain
and 4 on lanes by default, which changes the online-softmax grouping in lm_decode_attn2_kernel and may legitimately flip near-tie
tokens (tests/test_llm_gpu.py::test_lm_generate_lanes_identical pins it the same way)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def build_lm():
    from oracle import llama
    from test_llm_gpu import build
    cfg = llama.lm_small()
    m, sd = build(cfg, 5, 2.0)
    m.lane_att_unroll = m.att_unroll
    return m, sd, cfg


def inputs(te_lens, T, F, seed, pad_value=float("nan")):
    """mix [B, T, F]; enrollments right-padded to the longest with `pad_value` (NaN: a frame past a row's length must never be read)"""
    g = torch.Generator().manual_seed(seed)
    B = len(te_lens)
    mix = torch.randn(B, T, F, generator=g)
    enr = torch.full((B, max(te_lens), F), pad_value)
    for b, n in enumerate(te_lens):
        enr[b, :n] = torch.randn(n, F, generator=g)
    return mix.cuda(), enr.cuda()


def test_ragged_with_equal_lengths_is_the_uniform_call(lib):
    """all lengths equal (padded 7 NaN frames wider): identical greedy tokens, and identical sampled tokens for one seed, on a single
    chain and on lanes, twice (the second call replays the captured graphs)"""
    m, _, cfg = build_lm()
    B, T, Te = 5, 20, 9
    mix, enr_pad = inputs([Te] * B + [Te + 7], T, cfg["feats_dim"], 1)
    mix, enr_pad = mix[:B], enr_pad[:B]
    enr = enr_pad[:, :Te].contiguous()
    lens = torch.full((B,), Te, dtype=torch.int32)
    for chunk, lanes in ((32, 1), (2, 3)):
        m.chunk, m.lanes = chunk, lanes
        want_g = m.generate("tse", enr, enr, mix, mix, do_sample=False)
        want_s = m.generate("tse", enr, enr, mix, mix, do_sample=True, seed=77)
        for rep in range(2):
            got_g = m.generate("tse", enr_pad, enr_pad, mix, mix, do_sample=False, enroll_lengths=lens)
            got_s = m.generate("tse", enr_pad, enr_pad, mix, mix, do_sample=True, seed=77, enroll_lengths=lens.cuda())
            for a, b in zip(got_g + got_s, want_g + want_s):
                assert torch.equal(a, b), f"ragged call with equal lengths differs (chunk {chunk}, lanes {lanes}, call {rep})"


@pytest.mark.parametrize("B", [6, 40])
def test_ragged_rows_equal_each_row_alone(lib, B):
    """rows with different enrollment lengths in one call (B = 6: one chain; B = 40: two chunks on lanes) give each row the tokens
    it gets when generated alone; against the oracle (oracle/llama.py) under the top-2-margin rule"""
    from oracle import llama
    from test_unise_gpu import check_tokens
    m, sd, cfg = build_lm()
    T = 20
    te = [1, 5, 17, 9, 30, 2] if B == 6 else [1 + (7 * b) % 31 for b in range(B)]
    mix, enr = inputs(te, T, cfg["feats_dim"], 2)
    gg, ss = m.generate("tse", enr, enr, mix, mix, do_sample=False, enroll_lengths=te)
    gs, ss_s = m.generate("tse", enr, enr, mix, mix, do_sample=True, seed=5, enroll_lengths=te)
    torch.cuda.synchronize()
    assert gg.shape == (B, 32) and ss.shape == (B, T)
    assert int(gs.min()) >= 0 and int(gs.max()) < 64 and int(ss_s.min()) >= 0 and int(ss_s.max()) < 128
    for b, n in enumerate(te):
        e = enr[b:b + 1, :n].contiguous()
        g1, s1 = m.generate("tse", e, e, mix[b:b + 1], mix[b:b + 1], do_sample=False)
        assert torch.equal(gg[b:b + 1], g1) and torch.equal(ss[b:b + 1], s1), f"row {b} (enrollment {n} frames) differs from alone"
    if B <= 32:
        for b, n in enumerate(te):
            og, os_, margins = llama.sft_generate(sd, cfg, "tse", enr[b:b + 1, :n].cpu(), mix[b:b + 1].cpu(), T, return_margins=True)
            check_tokens(f"ragged row {b}", torch.cat([gg[b:b + 1].cpu(), ss[b:b + 1].cpu()], 1), torch.cat([og, os_], 1),
                         torch.cat([margins[:, :32], margins[:, 33:]], 1))


def test_enroll_lengths_refused(lib):
    m, _, cfg = build_lm()
    mix, enr = inputs([3, 4], 6, cfg["feats_dim"], 3)
    for bad in ([3], [0, 4], [3, 5]):
        with pytest.raises(ValueError):
            m.generate("tse", enr, enr, mix, mix, do_sample=False, enroll_lengths=bad)
    with pytest.raises(ValueError):
        m.generate("se", None, None, mix, mix, do_sample=False, enroll_lengths=[3, 4])
