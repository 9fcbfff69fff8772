"""CPU checks of the UniSE LM training path's edges: the split-K slicing of weight gradients covers every token with no empty slice,
the dropout threshold is float32(p) * 2^24 rounded half-to-even (the value the library receives is a C float), and the planted
(seed, b, h, i, j, layer) tuples that tests/test_lm_train_edges_gpu.py reads back from the kernels sit exactly on the threshold."""
import numpy as np
import pytest

from oracle import llama, llama_train
from unified_audio_b200 import ops

# (n_out, n_in) of every weight gradient the LM computes at the shipped widths: QKV, o_proj, gate/up, down, head, adapter
LM_WEIGHT_SHAPES = [(1536, 512), (512, 512), (4096, 512), (512, 2048), (12291, 512), (512, 768)]

# Philox words on the threshold, found by a search over seeds above 2^32 with the NumPy Philox (B = 3, heads = 8, i < 96):
# (p, word, (seed, b, h, i, j, layer)).  The device keeps the key whose word equals thr and drops the one at thr - 1.  At p = 0.09,
# float32(p) * 2^24 = 1509949.56 rounds to 1509950 while the double p * 2^24 = 1509949.44 rounds to 1509949: the word 1509949 is the
# key that a threshold rounded from the double would keep.
HEADS = 8
EDGE = [
    (0.1, 1677722, (4295035691, 1, 7, 78, 35, 11)),
    (0.1, 1677722, (4295135345, 0, 6, 77, 20, 11)),
    (0.1, 1677721, (4294996611, 1, 0, 58, 46, 11)),
    (0.1, 1677721, (4295072817, 2, 5, 50, 41, 11)),
    (0.09, 1509950, (4295234022, 1, 7, 63, 42, 11)),
    (0.09, 1509950, (4295482180, 2, 2, 88, 60, 11)),
    (0.09, 1509949, (4295316090, 1, 3, 27, 0, 11)),
    (0.09, 1509949, (4295405974, 0, 6, 70, 30, 11)),
]


def edge_word(seed, b, h, i, j, layer):
    """the 24-bit word of key j of query i (include/quark_b200.h), from the scalar Philox of oracle/llama.py"""
    return llama.philox4x32_10((seed & 0xFFFFFFFF, seed >> 32), (i, j >> 2, b * HEADS + h, layer))[j & 3] >> 8


@pytest.mark.parametrize("n_out,n_in", LM_WEIGHT_SHAPES)
def test_grad_slice_covers_every_token(n_out, n_in):
    for tokens in range(1, 30001):
        ks = ops.grad_slice(tokens, n_out, n_in)
        S = -(-tokens // ks)
        assert ks >= 64 and ks % 64 == 0, (tokens, ks)
        assert (S - 1) * ks < tokens <= S * ks, (tokens, ks)           # every token in a slice, the last slice not empty


def test_grad_slice_at_the_training_batch():
    """the slice counts the GPU weight-gradient tests rely on: B = 32 x 5 s splits the QKV and o_proj gradients into many slices, the
    head stays one slice of B * Lt tokens"""
    S = lambda T, n_out, n_in: -(-T // ops.grad_slice(T, n_out, n_in))
    assert S(17120, 1536, 512) == 6 and S(17120, 512, 512) == 17
    assert S(9056, 12291, 512) == 1 and S(786, 1536, 512) <= 2


def test_dropout_threshold_is_float32_half_even():
    assert llama_train.dropout_threshold(0.1) == 1677722
    assert llama_train.dropout_threshold(0.09) == 1509950 and round(0.09 * 2 ** 24) == 1509949
    assert llama_train.dropout_threshold(0.0) == 0 and llama_train.dropout_threshold(0.5) == 2 ** 23
    # ties go to even: p = 3 / 2^25 and 5 / 2^25 are floats with p * 2^24 = 1.5 and 2.5
    assert llama_train.dropout_threshold(3 * 2.0 ** -25) == 2 and llama_train.dropout_threshold(5 * 2.0 ** -25) == 2
    differ = [k for k in range(1, 1000) if llama_train.dropout_threshold(k / 1000) != round(k / 1000 * 2 ** 24)]
    for k in range(1, 1000):
        assert llama_train.dropout_threshold(k / 1000) == int(np.rint(float(np.float32(k / 1000)) * 2 ** 24))
    assert {58, 90, 160} <= set(differ) and len(differ) == 81
    assert all(abs(llama_train.dropout_threshold(k / 1000) - round(k / 1000 * 2 ** 24)) == 1 for k in differ)


def test_dropout_keep_thresholds_float32_p():
    """dropout_keep(p) is words >= dropout_threshold(p) at a p where float32 and double roundings differ"""
    seed, layer, B, L = 2 ** 40 + 3, 4, 2, 40
    words = llama_train.dropout_words(seed, layer, B, HEADS, L)
    keep = llama_train.dropout_keep(seed, layer, B, HEADS, L, 0.09)
    assert np.array_equal(keep, words >= 1509950)
    assert words.max() < 2 ** 24


@pytest.mark.parametrize("p,word,t", EDGE)
def test_threshold_edge_tuples_recompute(p, word, t):
    seed, b, h, i, j, layer = t
    assert seed >= 2 ** 32 and j <= i < 96 and b < 3 and h < HEADS
    assert edge_word(*t) == word
    thr = llama_train.dropout_threshold(p)
    assert word in (thr, thr - 1)
    B, L = 3, i + 1
    assert bool(llama_train.dropout_keep(seed, layer, B, HEADS, L, p)[b, h, i, j]) == (word == thr)
