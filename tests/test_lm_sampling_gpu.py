"""Sampled decoding for every top_k / top_p the reference accepts, and one random stream per row (qb_lm_head_sample_tc /
qb_lm_head_sample_rows_tc, LLM_SFT.generate(row_seeds=), Model.enhance(utterance_seed=) / enhance_batch(utterance_seeds=)).

The head kernels run on the planted logits of tests/golden/lm_sampling.npz (the reference's own sample_logits,
oracle/make_golden_lm_sampling.py) at the shipped range widths (4096 / 8192 columns of max_cols 8192); every kept set and every
drawn token is judged by the fp64 oracle.  The device sums in another order than the reference's torch.cumsum, so a kept count may
differ where the fp64 cumulative probability lies within MARGIN of top_p, and a token where the draw's target lies within MARGIN
of a CDF boundary; those rows are printed, and no other difference is accepted."""
import os
import random

import numpy as np
import pytest
import torch

from test_lm_kernels_gpu import DEV, HK, SENT, _onehot_x, _planted_head, _rnd

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MARGIN = 1e-5
V, MAX_COLS = 12291, 8192
RANGES = {"global": (3, 4096), "semantic": (4099, 8192)}
SEED, CALL, SLOT0 = 987654321012345, 3, 7


def _fixture():
    return np.load(os.path.join(GOLD, "lm_sampling.npz"))


class Head:
    """the sampled head over planted logits: row b of the range [lo, lo + width) is vals[:, b] (times one common RMSNorm factor)"""

    def __init__(self, lo, width, vals):
        B = vals.shape[1]
        w = torch.zeros(V + 16, B, device=DEV)
        w[lo:lo + width] = vals.to(DEV)
        w[lo + width:lo + width + 16] = 1e4                       # just past the range: never drawn
        w[lo - 1] = 1e4
        self.B, self.lo, self.width = B, lo, width
        self.wp = _planted_head(V, 16, w)
        self.x = _onehot_x(B, list(range(B)))
        self.rng = torch.tensor([lo, lo + width], dtype=torch.int32, device=DEV)
        self.emb = _rnd((V + 16, HK), 5)

    def draw(self, temperature, top_k, top_p, keys=None):
        """one step at slot SLOT0; keys: one 64-bit key per row (qb_lm_head_sample_rows_tc), else the call's seed.  -> (token ids
        relative to lo, debug [B, 4], the range logits the head wrote)"""
        from unified_audio_b200 import ops
        B = self.B
        out_ids = torch.full((B, 16), -7, dtype=torch.int64, device=DEV)
        x_next = torch.empty(B, HK, device=DEV)
        pos = torch.full((B,), 11, dtype=torch.int32, device=DEV)
        slot = torch.tensor([SLOT0, 0], dtype=torch.int32, device=DEV)
        pv = torch.zeros(MAX_COLS // 16 + 1, 32, device=DEV)
        pi = torch.zeros(MAX_COLS // 16 + 1, 32, dtype=torch.int32, device=DEV)
        logits = torch.full((B, MAX_COLS), SENT, device=DEV)
        dbg = torch.zeros(B, 4, device=DEV)
        args = (self.x, B, HK, self.wp, self.rng, MAX_COLS, self.emb, x_next, out_ids, 16, pos, slot, pv, pi, logits, temperature,
                top_k, top_p)
        if keys is not None:
            ops.lm_head_sample_rows_tc(*args, ops.row_keys_words(keys).to(DEV), dbg)
        else:
            to_i32 = lambda v: v - (1 << 32) if v >= (1 << 31) else v
            sd = torch.tensor([to_i32(SEED & 0xFFFFFFFF), to_i32(SEED >> 32), CALL, 0], dtype=torch.int32, device=DEV)
            ops.lm_head_sample_tc(*args, sd, dbg)
        torch.cuda.synchronize()
        ids = out_ids[:, SLOT0].cpu()
        assert bool((out_ids[:, :SLOT0] == -7).all()) and bool((out_ids[:, SLOT0 + 1:] == -7).all()), "out_ids column"
        assert bool((logits[:, self.width:] == SENT).all()), "logits written past the range"
        assert torch.equal(x_next, self.emb[out_ids[:, SLOT0]]), "x_next must be emb[token]"
        assert pos.tolist() == [12] * B and slot.tolist() == [SLOT0 + 1, 0]
        return ids - self.lo, dbg.cpu(), logits[:, :self.width].cpu()


def check_vs_fp64(tag, ids, dbg, logits, temperature, top_k, top_p, uniforms):
    """kept sets and tokens against the fp64 oracle; returns the near-tie rows"""
    from oracle import lm_sampling
    near_rows = []
    for b in range(logits.shape[0]):
        row = logits[b]
        assert float(dbg[b, 0]) == uniforms[b], f"{tag} row {b}: uniform {float(dbg[b, 0])} vs {uniforms[b]}"
        kk = row.numel() if top_k <= 0 else min(top_k, row.numel())
        n_surv = int((row >= torch.topk(row, kk)[0][-1]).sum())
        assert int(dbg[b, 1]) == n_surv, f"{tag} row {b}: survivors {int(dbg[b, 1])} vs {n_surv}"
        probs = lm_sampling.sample_filter(row[None], temperature, top_k, top_p, dtype=torch.float64)[0]
        dist = lm_sampling.top_p_distance(row, top_k, top_p)
        kept = int((probs > 0).sum())
        want, near = lm_sampling.inverse_cdf_pick(probs, uniforms[b])
        tok = int(ids[b])
        if int(dbg[b, 2]) != kept or tok != want:
            assert dist < MARGIN or (int(dbg[b, 2]) == kept and near < MARGIN), (
                f"{tag} row {b}: kept {int(dbg[b, 2])} vs {kept}, token {tok} vs {want} (top-p distance {dist:.2e}, draw {near:.2e})")
            near_rows.append((b, int(dbg[b, 2]) - kept, tok, want, dist, near))
        assert bool(probs[tok] > 0) or dist < MARGIN, f"{tag} row {b}: token {tok} outside the fp64 support"
    if near_rows:
        print(f"{tag}: near-tie rows (row, kept - fp64 kept, token, fp64 token, top-p distance, draw distance): {near_rows}")
    return near_rows


@pytest.mark.parametrize("rng", list(RANGES))
@pytest.mark.parametrize("top_k", [0, 1024, 1025, 4096, 8192, 12291])
def test_sampler_fixture_cases_vs_fp64(lib, rng, top_k):
    """every case of the reference fixture, on the call's stream and on per-row keys: survivors, kept set and token"""
    from oracle import lm_sampling
    z = _fixture()
    lo, width = RANGES[rng]
    rows = torch.from_numpy(z[f"{rng}.logits"])
    head = Head(lo, width, rows.t().contiguous())
    keys = [random.Random(top_k * 7 + b).getrandbits(64) for b in range(rows.shape[0])]
    for top_p in (0.95, 1.0):
        for temperature in (0.8, 0.3):
            ids, dbg, lg = head.draw(temperature, top_k, top_p)
            check_vs_fp64(f"{rng} k{top_k} p{top_p} t{temperature}", ids, dbg, lg, temperature, top_k, top_p,
                          [lm_sampling.sample_uniform(SEED, CALL, SLOT0, b) for b in range(rows.shape[0])])
            ids_r, dbg_r, lg_r = head.draw(temperature, top_k, top_p, keys=keys)
            assert torch.equal(lg_r, lg)
            check_vs_fp64(f"{rng} k{top_k} p{top_p} t{temperature} rows", ids_r, dbg_r, lg_r, temperature, top_k, top_p,
                          [lm_sampling.sample_uniform_row(k, SLOT0) for k in keys])
            again = head.draw(temperature, top_k, top_p, keys=keys)[0]
            assert torch.equal(again, ids_r), "the draw changed between identical calls"


def test_sampler_top_k_1_is_argmax(lib):
    z = _fixture()
    for rng, (lo, width) in RANGES.items():
        rows = torch.from_numpy(z[f"{rng}.logits"])
        head = Head(lo, width, rows.t().contiguous())
        for keys in (None, [11, 12, 13, 14, 15]):
            ids, _, lg = head.draw(1.0, 1, 1.0, keys=keys)
            uniq = (lg == lg.max(1, keepdim=True).values).sum(1) == 1
            assert int(uniq.sum()) >= 2 and torch.equal(ids[uniq], lg.argmax(1)[uniq]), f"{rng}: top_k = 1 must be the arg-max"


@pytest.mark.parametrize("top_k", [0, 50, 1024, 2000])
def test_row_keyed_draws_follow_their_rows(lib, top_k):
    """permuting the rows and their keys together permutes the tokens; a row alone draws what it draws in the batch"""
    z = _fixture()
    lo, width = RANGES["semantic"]
    rows = torch.from_numpy(z["semantic.logits"])
    rows = torch.cat([rows, rows[:2]], 0)                         # two rows twice: equal logits, different keys
    keys = [random.Random(100 + b).getrandbits(64) for b in range(rows.shape[0])]
    ids = Head(lo, width, rows.t().contiguous()).draw(0.8, top_k, 0.99, keys=keys)[0]
    perm = torch.randperm(rows.shape[0], generator=torch.Generator().manual_seed(top_k))
    ids_p = Head(lo, width, rows[perm].t().contiguous()).draw(0.8, top_k, 0.99, keys=[keys[i] for i in perm.tolist()])[0]
    assert torch.equal(ids_p, ids[perm]), f"top_k {top_k}: {ids_p.tolist()} vs {ids[perm].tolist()}"
    for b in (0, 3, 5):
        alone = Head(lo, width, rows[b:b + 1].t().contiguous()).draw(0.8, top_k, 0.99, keys=[keys[b]])[0]
        assert int(alone[0]) == int(ids[b]), f"top_k {top_k} row {b}: alone {int(alone[0])} vs {int(ids[b])}"


def test_uniform_path_tokens_unchanged(lib):
    """top_k <= 1024 on the call's stream: the tokens the uniform kernel drew before full-range sampling and per-row streams
    existed (tests/golden/lm_sampling_uniform_tokens.npz, recorded on an H100 from the kernel of the previous revision)"""
    z = _fixture()
    t = np.load(os.path.join(GOLD, "lm_sampling_uniform_tokens.npz"))
    n = 0
    for rng, (lo, width) in RANGES.items():
        head = Head(lo, width, torch.from_numpy(z[f"{rng}.logits"]).t().contiguous())
        for top_k in (1, 50, 1024):
            for top_p in (0.95, 1.0):
                for temperature in (0.8, 0.3):
                    ids = head.draw(temperature, top_k, top_p)[0]
                    want = torch.from_numpy(t[f"{rng}.k{top_k}.p{top_p}.t{temperature}"])
                    assert torch.equal(ids, want), f"{rng} k{top_k} p{top_p} t{temperature}: {ids.tolist()} vs {want.tolist()}"
                    n += 1
    assert n == 24


# ---------------------------------------------------------------------------------------------- LLM_SFT.generate(row_seeds=)
def _lm(cfg, seed=3, gain=2.0):
    from oracle import llama
    from unified_audio_b200.llm import LLM_SFT
    m = LLM_SFT(num_tasks=cfg["num_tasks"], task_map=cfg["task_map"], feats_dim=cfg["feats_dim"], llm_base_config=cfg["llm_base_config"])
    m.load_state_dict(llama.make_lm_state_dict(cfg, seed, gain))
    m = m.cuda()
    m.lane_att_unroll = m.att_unroll          # same decode-attention summation order on lanes and on one chain
    return m


@pytest.mark.parametrize("task", ["se", "tse"])
@pytest.mark.parametrize("top_k", [50, 0])
def test_generate_row_seeds_independent_of_the_batch(lib, task, top_k):
    """40 rows (two chunks of <= 32, run on two lanes), the same rows shuffled, and each row alone give every row the same global
    and semantic tokens; 'tse' with ragged enrollments"""
    from oracle import llama
    cfg = llama.lm_small()
    m = _lm(cfg)
    g = torch.Generator().manual_seed(21)
    B, T, Te = 40, 9, 6
    mix = torch.randn(B, T, cfg["feats_dim"], generator=g).cuda()
    enr = torch.randn(B, Te, cfg["feats_dim"], generator=g).cuda() if task == "tse" else None
    te = torch.randint(1, Te + 1, (B,), generator=g).tolist() if task == "tse" else None
    seeds = [random.Random(b).getrandbits(63) - (1 << 62) for b in range(B)]
    kw = dict(do_sample=True, top_k=top_k, top_p=0.97, temperature=0.9)

    def gen(rows):
        r = torch.tensor(rows)
        return m.generate(task, enr[r] if enr is not None else None, enr[r] if enr is not None else None, mix[r], mix[r],
                          enroll_lengths=[te[i] for i in rows] if te else None, row_seeds=[seeds[i] for i in rows], **kw)

    gg, ss = gen(list(range(B)))
    assert gg.shape == (B, 32) and ss.shape == (B, T)
    assert bool(((gg >= 0) & (gg < cfg["llm_base_config"]["global_size"])).all())
    assert bool(((ss >= 0) & (ss < cfg["llm_base_config"]["semantic_size"])).all())
    perm = torch.randperm(B, generator=g).tolist()
    gp, sp = gen(perm)
    assert torch.equal(gp, gg[perm]) and torch.equal(sp, ss[perm]), "shuffled rows drew other tokens"
    for b in (0, 17, 33, 39):
        g1, s1 = gen([b])
        assert torch.equal(g1[0], gg[b]) and torch.equal(s1[0], ss[b]), f"row {b} alone drew other tokens"
    g2, s2 = gen(list(range(B)))
    assert torch.equal(g2, gg) and torch.equal(s2, ss), "a repeated call drew other tokens"
    n_diff = int((gg[:, None] != gg[None]).any(-1).sum())
    assert n_diff > 0, "rows with different keys drew the same tokens everywhere"


def test_generate_full_range_at_shipped_widths(lib):
    """top_k = 0 (no filter) over the shipped 4096 / 8192-token ranges with per-row keys and with the call's seed; a row keyed k
    draws what row 0 of a one-row call with seed k draws"""
    from oracle import llama
    cfg = llama.LM_FULL
    m = _lm(cfg, 7, 2.0)
    g = torch.Generator().manual_seed(5)
    mix = torch.randn(3, 8, cfg["feats_dim"], generator=g).cuda()
    gg, ss = m.generate("se", None, None, mix, mix, top_k=0, top_p=1.0, row_seeds=[1, 2, 3])
    assert bool(((gg >= 0) & (gg < 4096)).all()) and bool(((ss >= 0) & (ss < 8192)).all())
    g1, s1 = m.generate("se", None, None, mix[1:2], mix[1:2], top_k=0, top_p=1.0, seed=2)
    assert torch.equal(g1[0], gg[1]) and torch.equal(s1[0], ss[1])
    for top_k, top_p in ((0, 0.95), (12291, 0.9), (5000, 1.0)):
        a = m.generate("se", None, None, mix, mix, top_k=top_k, top_p=top_p, seed=9)
        b = m.generate("se", None, None, mix, mix, top_k=top_k, top_p=top_p, seed=9)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    with pytest.raises(RuntimeError, match="out of range"):
        m.generate("se", None, None, mix, mix, top_k=12292)


# ---------------------------------------------------------------------------------------------- Model.enhance / enhance_batch
@pytest.fixture(scope="module")
def unise_model(lib):
    from test_unise_gpu import build
    model, _ = build()
    model.dnn.lane_att_unroll = model.dnn.att_unroll
    return model


@pytest.mark.parametrize("mode", ["se", "tse", "ss"])
def test_enhance_batch_sampled_equals_enhance_alone(unise_model, mode):
    from test_unise_batch_gpu import as_tuple, utterances
    model = unise_model
    srcs, enrolls = utterances(41)
    srcs, enrolls = [s.cuda() for s in srcs], [e.cuda() for e in enrolls]
    seeds = [1000 + 17 * u for u in range(len(srcs))]
    ef = enrolls if mode == "tse" else None
    want = [model.enhance(mode, e if mode == "tse" else None, s, do_sample=True, utterance_seed=sd, return_ids=True)
            for s, e, sd in zip(srcs, enrolls, seeds)]
    for max_segments in (128, 4):
        got = model.enhance_batch(mode, ef, srcs, do_sample=True, utterance_seeds=seeds, return_ids=True, max_segments=max_segments)
        for u, (g, w) in enumerate(zip(got, want)):
            for a, b in zip(as_tuple(g), as_tuple(w)):
                assert a.shape == b.shape and torch.equal(a, b), f"{mode} utterance {u} differs (max_segments {max_segments})"
    again = model.enhance_batch(mode, ef, srcs, do_sample=True, utterance_seeds=seeds, return_ids=True)
    for g, w in zip(again, want):
        assert all(torch.equal(a, b) for a, b in zip(as_tuple(g), as_tuple(w))), "a repeated call differs"
    greedy = model.enhance(mode, ef[0] if ef else None, srcs[0], return_ids=True)
    assert any(not torch.equal(a, b) for a, b in zip(as_tuple(greedy), as_tuple(want[0]))), "sampled output equals greedy"
