"""Sampled decoding without a GPU: oracle.lm_sampling.sample_filter against the reference's own sample_logits for every top_k / top_p it
accepts (tests/golden/lm_sampling.npz, oracle/make_golden_lm_sampling.py), the per-row random streams' key derivation and packing,
and the argument checks of LLM_SFT.generate(row_seeds=, top_k=) and Model.enhance_batch(utterance_seeds=)."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_oracle_matches_reference_sample_logits():
    """support bit for bit (where the cut falls inside a run of equal logits the reference's unstable sort keeps another subset
    of the run: outside it the supports agree and both keep as many of it) and probabilities to 1e-5"""
    from oracle import lm_sampling
    z = np.load(os.path.join(GOLD, "lm_sampling.npz"))
    meta = json.loads(str(z["meta"]))
    n_cases = n_tied = 0
    for rng, (lo, width) in meta["ranges"].items():
        rows = torch.from_numpy(z[f"{rng}.logits"])
        for top_k in meta["top_k"]:
            for top_p in meta["top_p"]:
                for temp in meta["temperatures"]:
                    name = f"{rng}.k{top_k}.p{top_p}.t{temp}"
                    probs = lm_sampling.sample_filter(rows, temp, top_k, top_p)
                    sup_r = torch.from_numpy(np.unpackbits(z[f"{name}.support"], axis=1)[:, :width].astype(bool))
                    tied = set(z[f"{name}.tied_cut"].tolist())
                    for b in range(rows.shape[0]):
                        sup_o = probs[b] > 0
                        if b in tied:
                            run = rows[b] == rows[b][sup_o].min()
                            assert torch.equal(sup_o & ~run, sup_r[b] & ~run), f"{name} row {b}"
                            assert int((sup_o & run).sum()) == int((sup_r[b] & run).sum()) < int(run.sum()), f"{name} row {b}"
                            n_tied += 1
                        else:
                            assert torch.equal(sup_o, sup_r[b]), f"{name} row {b}: support"
                            assert np.allclose(probs[b, z[f"{name}.top_ids"][b]].numpy(), z[f"{name}.top_probs"][b], rtol=1e-5,
                                               atol=1e-7), f"{name} row {b}: probabilities"
                    top = torch.topk(probs, 32, -1).values.numpy()
                    assert np.allclose(top, z[f"{name}.top_probs"], rtol=1e-5, atol=1e-7), f"{name}: probabilities"
                    assert np.allclose(probs.max(-1).values.numpy(), z[f"{name}.probs_max"], rtol=1e-5, atol=1e-7)
                    n_cases += 1
    assert n_cases == 48 and n_tied > 0


def test_oracle_filter_edges():
    """top_k <= 0 and top_p >= 1 filter nothing; top_k >= the width keeps every token; fp64 agrees with fp32 on the support"""
    from oracle import lm_sampling
    row = torch.randn(2, 300, generator=torch.Generator().manual_seed(1)).half().float() * 2
    every = torch.softmax(row / 0.7, -1)
    for top_k in (0, -3, 300, 301, 12291):
        assert torch.allclose(lm_sampling.sample_filter(row, 0.7, top_k, 1.0), every)
    p32 = lm_sampling.sample_filter(row, 0.7, 40, 0.9)
    p64 = lm_sampling.sample_filter(row, 0.7, 40, 0.9, dtype=torch.float64)
    assert p64.dtype == torch.float64 and torch.equal(p32 > 0, p64 > 0) and int((p32[0] > 0).sum()) <= 40
    assert lm_sampling.top_p_distance(row[0], 0, 1.0) == float("inf") and lm_sampling.top_p_distance(row[0], 40, 0.9) > 0


def test_row_uniform_and_key_words():
    """a row keyed k draws row 0 / call 0 of the call stream seeded k; keys pack as {low, high} int32 words, mod 2^64"""
    from oracle import lm_sampling
    from unified_audio_b200 import ops
    for key in (0, 1, 987654321012345, (1 << 64) - 1):
        for step in (0, 5, 282):
            assert lm_sampling.sample_uniform_row(key, step) == lm_sampling.sample_uniform(key, 0, step, 0)
    assert lm_sampling.sample_uniform_row(-1, 3) == lm_sampling.sample_uniform_row((1 << 64) - 1, 3)
    assert lm_sampling.sample_uniform_row(5, 3) != lm_sampling.sample_uniform_row(6, 3)
    w = ops.row_keys_words([0x0123456789ABCDEF, -1, 7])
    assert w.dtype == torch.int32 and w.shape == (3, 2)
    assert w.tolist() == [[0x89ABCDEF - (1 << 32), 0x01234567], [-1, -1], [7, 0]]


def test_segment_key_is_a_pure_function():
    from unified_audio_b200.unise import GENERATE_PASSES, segment_key
    m64 = (1 << 64) - 1

    def mix(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m64
        return z ^ (z >> 31)

    def restated(seed, p, seg):
        g = 0x9E3779B97F4A7C15
        h = mix((seed + g) & m64)
        h = mix(((h ^ GENERATE_PASSES.index(p)) + g) & m64)
        return mix(((h ^ seg) + g) & m64)

    keys = {}
    for seed in (0, 1, 12345, -7, (1 << 63) + 5):
        for p in GENERATE_PASSES:
            for seg in (0, 1, 2, 31, 1000):
                k = segment_key(seed, p, seg)
                assert k == segment_key(seed, p, seg) == restated(seed, p, seg) and 0 <= k <= m64
                keys.setdefault(k, (seed, p, seg))
    assert len(keys) == 5 * 3 * 5, "distinct (seed, pass, segment) share a key"
    with pytest.raises(ValueError):
        segment_key(1, "ss", 0)
    with pytest.raises(ValueError):
        segment_key(1, "se", -1)


def _lm(cfg):
    from unified_audio_b200.llm import LLM_SFT
    return LLM_SFT(num_tasks=cfg["num_tasks"], task_map=cfg["task_map"], feats_dim=cfg["feats_dim"], llm_base_config=cfg["llm_base_config"])


def test_generate_argument_checks():
    """refused before any device work: row_seeds with seed, row_seeds of the wrong length or type, a top_k above the vocabulary"""
    from oracle import llama
    m = _lm(llama.LM_FULL)
    mix = torch.zeros(3, 4, llama.LM_FULL["feats_dim"])
    gen = lambda **kw: m.generate("se", None, None, mix, mix, **kw)
    with pytest.raises(ValueError, match="not both"):
        gen(row_seeds=[1, 2, 3], seed=4)
    for bad in ([1, 2], [1, 2, 3, 4], torch.tensor([1, 2]), []):
        with pytest.raises(ValueError, match="3 keys"):
            gen(row_seeds=bad)
    for bad in ([1.5, 2, 3], torch.tensor([1.0, 2.0, 3.0])):
        with pytest.raises(ValueError, match="integers"):
            gen(row_seeds=bad)
    with pytest.raises(RuntimeError, match="out of range"):
        gen(top_k=12292)
    with pytest.raises(AssertionError):
        gen(temperature=0.0)


def test_enhance_batch_seed_checks():
    from unified_audio_b200.unise import Model
    model = Model.__new__(Model)
    srcs = [torch.zeros(1, 100), torch.zeros(1, 200)]
    with pytest.raises(ValueError, match="3 utterance_seeds for 2 utterances"):
        model._enhance_batch("se", None, srcs, True, False, 32, [1, 2, 3])
    with pytest.raises(ValueError, match="1 utterance_seeds for 2 utterances"):
        model._enhance_batch("se", None, srcs, True, False, 32, [1])
    with pytest.raises(ValueError, match="cannot be combined"):
        model._enhance_batch("se", None, srcs, True, False, 32, [1, 2], seed=3)
    with pytest.raises(ValueError, match="cannot be combined"):
        Model._check_seed_args(dict(row_seeds=[1]), "utterance_seed")
