"""CPU restatement of the UniSE LM's sampled decoding for every top_k / top_p the reference accepts, and of the per-row random
streams of the device sampler.

TEST INFRASTRUCTURE - see oracle/__init__.py.  Extends oracle/llama.py's sampled-decoding helpers (`sample_filter`, `sample_uniform`,
`inverse_cdf_pick`), which cover 1 <= top_k <= the range width in fp32:
  sample_filter       top_k <= 0 (no filter) and top_k >= the range width, and an fp64 mode - the oracle near-ties are judged by
  sample_uniform_row  the uniform of a row keyed by its own 64-bit key (qb_lm_head_sample_rows_tc)
  top_p_distance      how close a row's top-p cut lies to a near-tie
Pinned against the reference's own `sample_logits` (QuarkAudio-UniSE/model/llm/llm.py:253-289) by oracle/make_golden_lm_sampling.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.llama import inverse_cdf_pick, philox4x32_10, sample_uniform  # noqa: F401  (the draw helpers, re-exported)


def sample_filter(logits, temperature=0.8, top_k=50, top_p=0.95, dtype=torch.float32):
    """The reference's sample_logits up to (not including) the multinomial draw on range rows [B, V']: returns the final
    probabilities (zeros where a token was filtered out).  Steps, in the reference's order: top-k by threshold value
    (`logits < topk[-1]` removed, ties at the k-th value stay) -> top-p on the descending sort of the survivors (a token goes when
    the cumulative softmax BEFORE it exceeds top_p; the first always stays) -> / temperature -> softmax.
    top_k <= 0: no top-k filter; top_k >= V' keeps every token (the reference's torch.topk runs over the range-masked vocabulary
    row, whose masked entries are -inf); top_p >= 1: no top-p filter.  The sort is stable: where the cut falls inside a run of
    equal logits the lowest ids are kept, the order the device sampler defines (the reference's unstable sort keeps an arbitrary
    subset of the run).  dtype float64 is the fp64 oracle the device sampler's near-ties are judged by."""
    logits = logits.clone().to(dtype)
    if top_k > 0:
        kth = torch.topk(logits, min(top_k, logits.shape[-1]))[0][..., -1, None]
        logits[logits < kth] = float("-inf")
    if top_p < 1.0:
        sorted_logits, sorted_indices = torch.sort(logits, descending=True, stable=True)
        cum = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
        rem = cum > top_p
        rem[..., 1:] = rem[..., :-1].clone()
        rem[..., 0] = 0
        logits[rem.scatter(-1, sorted_indices, rem)] = float("-inf")
    assert 0 < temperature <= 1.0
    return F.softmax(logits / temperature, dim=-1)


def sample_uniform_row(key, step):
    """The uniform of a row keyed `key` (64-bit, taken mod 2^64) at decode step `step` (qb_lm_head_sample_rows_tc): 24 high bits
    of Philox4x32-10(key split lo/hi, counter = {step, 0, 0, 0}).x - a function of (key, step) only."""
    key &= 0xFFFFFFFFFFFFFFFF
    r = philox4x32_10((key & 0xFFFFFFFF, key >> 32), (step, 0, 0, 0))[0]
    return (r >> 8) / 16777216.0


def top_p_distance(logits_row, top_k, top_p):
    """fp64 distance of the top-p cut from a near-tie: min over the survivors of top-k, sorted descending, of
    |cumulative softmax - top_p| (inf when top_p >= 1).  A sampler that sums in another order than torch.cumsum may put the
    token after such a boundary on the other side of it."""
    if top_p >= 1.0:
        return float("inf")
    row = logits_row.double()
    if top_k > 0:
        row = row[row >= torch.topk(row, min(top_k, row.numel()))[0][-1]]
    cum = torch.cumsum(torch.softmax(torch.sort(row, descending=True).values, 0), 0)
    return float((cum - top_p).abs().min())
