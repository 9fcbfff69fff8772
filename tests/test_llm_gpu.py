"""GPU parity of unified_audio_b200.LLM_SFT against the LM oracle (pinned against transformers.LlamaModel)
and the committed golden fixture tests/golden/lm_small.npz."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def build(cfg, seed, gain):
    from oracle import llama
    from unified_audio_b200.llm import LLM_SFT
    sd = llama.make_lm_state_dict(cfg, seed, gain)
    m = LLM_SFT(num_tasks=cfg["num_tasks"], task_map=cfg["task_map"], feats_dim=cfg["feats_dim"],
                llm_base_config=cfg["llm_base_config"])
    sd2 = dict(sd)
    sd2["cond_input_layer.weight"] = torch.zeros(4, 4)        # dead conformer weights of a real checkpoint
    m.load_state_dict(sd2, strict=True)
    return m.cuda(), sd


def compare_tokens(tag, got, want, margins, thr=1e-4):
    """first differing step per sequence must be a numerically unsafe decision (tiny top-2 logit margin)"""
    got, want = got.cpu(), want.cpu()
    nbad = 0
    for b in range(want.shape[0]):
        diff = (got[b] != want[b]).nonzero()
        if len(diff):
            nbad += 1
            t = int(diff[0])
            print(f"[{tag}] seq {b}: first divergence at step {t}, oracle margin {float(margins[b, t]):.2e}")
            assert float(margins[b, t]) < thr, "token differs although the oracle's decision margin is safe"
    print(f"[{tag}] sequences with a differing token: {nbad}/{want.shape[0]}")
    return nbad


def test_lm_small_golden(lib):
    z = np.load(os.path.join(GOLD, "lm_small.npz"))
    meta = json.loads(str(z["meta"]))
    cfg = meta["cfg"]
    m, sd = build(cfg, meta["seed"], meta["gain"])
    mix, enr = torch.from_numpy(z["mix"]).cuda(), torch.from_numpy(z["enroll"]).cuda()
    gids, sids = torch.from_numpy(z["gids"]).cuda(), torch.from_numpy(z["sids"]).cuda()
    loss, acc, logits = m(task_name="tse", enroll_mel=enr, enroll_feats=enr, mix_mel=mix, mix_feats=mix, global_ids=gids,
                          semantic_ids=sids, return_logits=True)
    torch.cuda.synchronize()
    e = rel(logits, torch.from_numpy(z["logits"]))
    print(f"teacher-forced logits rel {e:.2e}  loss {float(loss):.6f} vs {float(z['loss']):.6f}")
    assert e < TOL and abs(float(loss) - float(z["loss"])) < 1e-3 * abs(float(z["loss"]))
    margins = torch.from_numpy(z["gen_margins"])
    for graph in (False, True):
        gg, ss = m.generate("se", None, None, mix, mix, do_sample=False, use_cuda_graph=graph)
        torch.cuda.synchronize()
        allt = torch.cat([gg.cpu() , torch.zeros(gg.shape[0], 1, dtype=torch.long), ss.cpu()], 1)
        want = torch.cat([torch.from_numpy(z["gen_global"]), torch.zeros(gg.shape[0], 1, dtype=torch.long),
                          torch.from_numpy(z["gen_semantic"])], 1)
        margins2 = margins.clone(); margins2[:, 32] = 1.0      # the 33rd step's token is discarded by the reference
        compare_tokens(f"small generate graph={graph}", allt, want, margins2)


def test_lm_full_config_vs_oracle(lib):
    """Shipped UniSE LM (12 x 512, vocab 12291): prefill + cached decode hidden states, then greedy generation."""
    from oracle import llama
    cfg = llama.LM_FULL
    m, sd = build(cfg, 7, 2.0)
    g = torch.Generator().manual_seed(11)
    B, T = 4, 24
    x = torch.randn(B, 70, 512, generator=g)
    ref_full, _ = llama.llm_forward(sd, cfg, x)
    out = m.llm_forward(x[:, :66].cuda(), use_cache=True)
    hs = [out.last_hidden_state]
    cache = out.past_key_values
    for i in range(66, 70):
        o = m.llm_forward(x[:, i:i + 1].cuda(), past_key_values=cache, use_cache=True)
        hs.append(o.last_hidden_state)
    torch.cuda.synchronize()
    got = torch.cat(hs, 1)
    e_pre, e_dec = rel(got[:, :66], ref_full[:, :66]), rel(got[:, 66:], ref_full[:, 66:])
    print(f"llm_forward: prefill rel {e_pre:.2e}  cached decode rel {e_dec:.2e}")
    assert e_pre < TOL and e_dec < TOL
    mix = torch.randn(B, T, 768, generator=g)
    enr = torch.randn(B, 30, 768, generator=g)
    og, os_, margins = llama.sft_generate(sd, cfg, "tse", enr, mix, T, return_margins=True)
    gg, ss = m.generate("tse", enr.cuda(), enr.cuda(), mix.cuda(), mix.cuda(), do_sample=False)
    torch.cuda.synchronize()
    margins[:, 32] = 1.0
    zero = torch.zeros(B, 1, dtype=torch.long)
    compare_tokens("full generate", torch.cat([gg.cpu(), zero, ss.cpu()], 1), torch.cat([og, zero, os_], 1), margins)
    print("min oracle margin", float(margins.min()))


@pytest.mark.parametrize("B", [1, 5, 32])
def test_lm_decode_step_vs_oracle(lib, B):
    """The decode step (packed fp16-split weights, mma.sync, programmatic dependent launch) against the oracle: cached
    single-token hidden states after a 40-token prefill."""
    from oracle import llama
    cfg = llama.LM_FULL
    m, sd = build(cfg, 3, 2.0)
    g = torch.Generator().manual_seed(100 + B)
    x = torch.randn(B, 46, 512, generator=g)
    ref, _ = llama.llm_forward(sd, cfg, x)
    out = m.llm_forward(x[:, :40].cuda(), use_cache=True)
    cache = out.past_key_values
    hs = []
    for i in range(40, 46):
        hs.append(m.llm_forward(x[:, i:i + 1].cuda(), past_key_values=cache, use_cache=True).last_hidden_state)
    torch.cuda.synchronize()
    e_tc = rel(torch.cat(hs, 1), ref[:, 40:])
    print(f"B={B}: decode rel vs oracle {e_tc:.2e}")
    assert e_tc < TOL


def test_lm_prefill_continuation_vs_oracle(lib):
    """A prefill that continues a filled cache (lm_qkv_prep + lm_flash_attn at pos0 > 0), then cached decodes, against the oracle's
    one-shot forward over all positions"""
    from oracle import llama
    cfg = llama.LM_FULL
    m, sd = build(cfg, 5, 2.0)
    g = torch.Generator().manual_seed(17)
    B = 3
    x = torch.randn(B, 74, 512, generator=g)
    ref, _ = llama.llm_forward(sd, cfg, x)
    out = m.llm_forward(x[:, :40].cuda(), use_cache=True)
    cache = out.past_key_values
    hs = [out.last_hidden_state, m.llm_forward(x[:, 40:70].cuda(), past_key_values=cache, use_cache=True).last_hidden_state]
    assert cache.length == 70
    for i in range(70, 74):
        hs.append(m.llm_forward(x[:, i:i + 1].cuda(), past_key_values=cache, use_cache=True).last_hidden_state)
    torch.cuda.synchronize()
    got = torch.cat(hs, 1)
    e_first, e_cont, e_dec = rel(got[:, :40], ref[:, :40]), rel(got[:, 40:70], ref[:, 40:70]), rel(got[:, 70:], ref[:, 70:])
    print(f"prefill rel {e_first:.2e}, continuation prefill rel {e_cont:.2e}, decode after it rel {e_dec:.2e}")
    assert e_first < TOL and e_cont < TOL and e_dec < TOL


@pytest.mark.parametrize("ssize", [100, 128])
def test_lm_generate_ranges_not_multiple_of_16(lib, ssize):
    """Token ranges whose width is not a multiple of 16 (global 40; semantic 100 or 128): greedy tokens match the oracle under the
    margin rule, and greedy and sampled tokens stay inside their ranges (the head's last CTA owns fewer than 16 columns)"""
    from oracle import llama
    cfg = llama.lm_small(gsize=40, ssize=ssize)
    m, sd = build(cfg, 9, 2.0)
    g = torch.Generator().manual_seed(ssize)
    B, T = 5, 20
    mix = torch.randn(B, T, cfg["feats_dim"], generator=g)
    og, os_, margins = llama.sft_generate(sd, cfg, "se", None, mix, T, return_margins=True)
    for graph in (False, True):
        gg, ss = m.generate("se", None, None, mix.cuda(), mix.cuda(), do_sample=False, use_cuda_graph=graph)
        torch.cuda.synchronize()
        gg, ss = gg.cpu(), ss.cpu()
        assert int(gg.min()) >= 0 and int(gg.max()) < 40 and int(ss.min()) >= 0 and int(ss.max()) < ssize
        margins[:, 32] = 1.0
        zero = torch.zeros(B, 1, dtype=torch.long)
        compare_tokens(f"gsize 40 ssize {ssize} graph={graph}", torch.cat([gg, zero, ss], 1), torch.cat([og, zero, os_], 1), margins)
    for seed in (1, 2, 3):
        gs_, ss_ = m.generate("se", None, None, mix.cuda(), mix.cuda(), do_sample=True, seed=seed, top_k=1024, top_p=1.0,
                              temperature=1.0)
        torch.cuda.synchronize()
        assert int(gs_.min()) >= 0 and int(gs_.max()) < 40 and int(ss_.min()) >= 0 and int(ss_.max()) < ssize


def test_lm_sampled_generate_vs_oracle(lib):
    """do_sample=True with the reference's default arguments (temperature 0.8, top_k 50, top_p 0.95; llm_sft.py:93-107).
    The device sampler's tokens are replayed on the oracle along the device's own token path: at every step the token must
    lie in the reference's filtered support (top-k -> top-p restated verbatim in oracle.llama.sample_filter) and must be the
    inverse-CDF pick at the same Philox uniform, except where the uniform lands within 1e-5 of a CDF boundary."""
    from oracle import llama
    cfg = llama.LM_FULL
    m, sd = build(cfg, 7, 2.0)
    g = torch.Generator().manual_seed(21)
    B, T, seed = 3, 12, 123456789012345
    mix = torch.randn(B, T, 768, generator=g)
    for use_graph in (False, True):
        gg, ss = m.generate("se", None, None, mix.cuda(), mix.cuda(), use_cuda_graph=use_graph, seed=seed)   # do_sample default True
        torch.cuda.synchronize()
        gg, ss = gg.cpu(), ss.cpu()
        assert gg.shape == (B, 32) and ss.shape == (B, T)
        assert int(gg.min()) >= 0 and int(gg.max()) < 4096 and int(ss.min()) >= 0 and int(ss.max()) < 8192
        if use_graph:
            assert torch.equal(gg, first[0]) and torch.equal(ss, first[1]), "graph replay must reproduce the eager sampled tokens"
        first = (gg, ss)
    # replay on the oracle (teacher-forced along the device's tokens)
    goff, soff = 3, 3 + 4096
    st = m._gen_state[next(iter(m._gen_state))]
    all_ids = st["out_ids"].cpu()                                   # [B, 33 + T] raw ids incl. the discarded 33rd global step
    hs, cache = llama.llm_forward(sd, cfg, llama._prefix(sd, cfg, "se", None, mix))
    ids = torch.zeros(B, 1, dtype=torch.long)
    n_in_support = n_same = n_close = 0
    total = 33 + T
    for step in range(total):
        if step == 33:
            ids = torch.ones(B, 1, dtype=torch.long)
        lo, hi = (goff, goff + 4096) if step < 33 else (soff, soff + 8192)
        h, cache = llama.llm_forward(sd, cfg, sd["codec_embedding.weight"][ids], cache)
        logits = torch.nn.functional.linear(h[:, 0], sd["output_head.weight"])[:, lo:hi]
        probs = llama.sample_filter(logits, 0.8, 50, 0.95)
        for b in range(B):
            tok = int(all_ids[b, step]) - lo
            assert 0 <= tok < hi - lo
            n_in_support += int(probs[b, tok] > 0)
            want, near = llama.inverse_cdf_pick(probs[b], llama.sample_uniform(seed, 0, step, b))
            if want == tok:
                n_same += 1
            elif near < 1e-4 or float(probs[b, tok]) < 1e-4:
                n_close += 1            # uniform on a CDF boundary / support edge at the float tolerance
            else:
                raise AssertionError(f"step {step} row {b}: device token {tok} (p={float(probs[b, tok]):.3e}) vs "
                                     f"inverse-CDF pick {want} (p={float(probs[b, want]):.3e}), boundary distance {near:.2e}")
        ids = all_ids[:, step:step + 1]
    print(f"sampled generate: {n_same}/{B * total} tokens identical to the oracle's inverse-CDF pick at the same uniform, "
          f"{n_close} on a boundary, {n_in_support}/{B * total} inside the reference's filtered support")
    assert n_in_support >= B * total - n_close and n_same >= 0.95 * B * total
    # different seed -> different draw; temperature bound is the reference's assert
    g2, s2 = m.generate("se", None, None, mix.cuda(), mix.cuda(), seed=seed + 1)
    assert not (torch.equal(g2.cpu(), gg) and torch.equal(s2.cpu(), ss))
    with pytest.raises(AssertionError):
        m.generate("se", None, None, mix.cuda(), mix.cuda(), temperature=1.5)


def test_lm_rope_table_grows_and_nan_safe(lib):
    """ADVICE r01: positions beyond max_position_embeddings (the reference's rotary embedding has no table limit), a cache
    that outgrows its capacity, a cache built for another batch, and an all-NaN logit row."""
    from oracle import llama
    cfg = llama.lm_small(hidden=128, layers=2, heads=2, gsize=64, ssize=128, feats=64)
    cfg["llm_base_config"]["max_position_embeddings"] = 96
    m, sd = build(cfg, 3, 2.0)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 140, 128, generator=g)
    ref, _ = llama.llm_forward(sd, cfg, x)
    out = m.llm_forward(x[:, :100].cuda(), use_cache=True, max_new_tokens=8)     # 100 > max_pos 96: table must grow
    cache = out.past_key_values
    hs = [out.last_hidden_state]
    for i in range(100, 140):                                                    # 40 > 8: the cache must grow
        hs.append(m.llm_forward(x[:, i:i + 1].cuda(), past_key_values=cache, use_cache=True).last_hidden_state)
    torch.cuda.synchronize()
    e = rel(torch.cat(hs, 1), ref)
    print(f"positions past max_position_embeddings + cache growth: rel {e:.2e}, cache capacity {cache.Lmax}")
    assert e < TOL and cache.length == 140
    with pytest.raises(ValueError):
        m.llm_forward(x[:1, :4].cuda(), past_key_values=cache, use_cache=True)   # batch mismatch
    mix = torch.full((2, 6, 64), float("nan"))
    gg, ss = m.generate("se", None, None, mix.cuda(), mix.cuda(), do_sample=False)
    torch.cuda.synchronize()                                                     # no illegal address; ids inside the range
    assert int(gg.min()) >= 0 and int(gg.max()) < 64 and int(ss.min()) >= 0 and int(ss.max()) < 128


@pytest.mark.parametrize("task", ["se", "tse"])
def test_lm_generate_lanes_identical(lib, task):
    """generate() over concurrent lanes (QB_LM_LANES / QB_LM_CHUNK: chunks of the batch on their own streams, KV caches and captured
    graphs) returns exactly the tokens of the serial chunk walk - greedy and sampled (same seed), ragged last chunk included -
    and keeps doing so when the lanes' cached state is reused by a second call."""
    from oracle import llama
    cfg = llama.lm_small()
    m, _ = build(cfg, 5, 2.0)
    g = torch.Generator().manual_seed(21)
    B, T = 7, 6
    mix = torch.randn(B, T, cfg["feats_dim"], generator=g).cuda()
    enr = torch.randn(B, T, cfg["feats_dim"], generator=g).cuda() if task == "tse" else None
    m.lane_att_unroll = m.att_unroll          # same fp32 summation order of the decode attention on every lane: bit-equal tokens
    m.chunk, m.lanes = 2, 1
    ref_g = m.generate(task, enr, enr, mix, mix, do_sample=False)
    ref_s = m.generate(task, enr, enr, mix, mix, do_sample=True, seed=77)
    whole = None
    if B <= 32:
        m.chunk = 32
        whole = m.generate(task, enr, enr, mix, mix, do_sample=False)       # rows are independent of how the batch is cut
    m.chunk, m.lanes = 2, 3
    for rep in range(2):
        got_g = m.generate(task, enr, enr, mix, mix, do_sample=False)
        got_s = m.generate(task, enr, enr, mix, mix, do_sample=True, seed=77)
        torch.cuda.synchronize()
        for a, b in zip(got_g + got_s, ref_g + ref_s):
            assert torch.equal(a, b), f"lanes changed the tokens (call {rep})"
    for a, b in zip(whole, ref_g):
        assert torch.equal(a, b), "chunk size changed the greedy tokens"
