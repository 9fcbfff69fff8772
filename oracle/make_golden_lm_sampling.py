"""Pin oracle.lm_sampling.sample_filter against the REFERENCE'S OWN `sample_logits` (QuarkAudio-UniSE/model/llm/llm.py:253-289) for every
top_k / top_p the reference accepts, at the shipped range widths.

TEST INFRASTRUCTURE.  Run in the build container only:  python -m oracle.make_golden_lm_sampling

The reference is imported as oracle/make_golden_lm_reference.py imports it (same shims, none touching its files).  `sample_logits`
runs unmodified on vocabulary rows of the shipped size (12 291) that are -inf outside one token range, as its `generate` masks them
(llm_sft.py:155-161,184-190): the global range (4096 columns from id 3) and the semantic range (8192 columns from id 4099).  Cases:
top_k in {0, 1024, 1025, 4096, 8192, 12291} x top_p in {0.95, 1.0} x temperature in {0.8, 0.3}, on five rows per range:
  0  N(0, 3)                       1  N(0, 0.05): a flat row, the top-p cut falls thousands of tokens deep
  2  integers in [-4, 4): ties at every k-th value and at the top-p cut
  3  30 equal logits far above the rest: the top-p cut falls inside the tied run
  4  1100 equal logits behind 20 larger ones: the 1024th / 1025th values are tied
Every logit is exactly representable in fp16 (the device tests plant them into an fp16-split head).  Where the top-p cut falls
inside a run of equal logits (rows 2 and 3), the reference's unstable sort keeps an arbitrary subset of the run; the oracle keeps
the lowest ids.  Such rows are listed per case (`tied_cut`): the two supports agree outside the run and keep as many of it.  Writes
tests/golden/lm_sampling.npz: the range rows and, per case, the reference's support (bit-packed), its probability maximum and its
32 most probable tokens with their probabilities; tests/test_lm_sampling_host.py re-checks the oracle against it.
"""
import json
import os

import numpy as np
import torch

from oracle import llama, lm_sampling
from oracle.make_golden_lm_reference import GOLD, build_reference

V = 12291
RANGES = {"global": (3, 4096), "semantic": (4099, 8192)}
TOP_K = (0, 1024, 1025, 4096, 8192, 12291)
TOP_P = (0.95, 1.0)
TEMPS = (0.8, 0.3)


def range_rows(width, seed):
    g = torch.Generator().manual_seed(seed)
    rows = torch.empty(5, width)
    rows[0] = torch.randn(width, generator=g) * 3.0
    rows[1] = torch.randn(width, generator=g) * 0.05
    rows[2] = torch.randint(-4, 4, (width,), generator=g).float()
    rows[3] = torch.randn(width, generator=g) * 0.5 - 6.0
    rows[3, torch.randperm(width, generator=g)[:30]] = 4.0
    rows[4] = torch.randn(width, generator=g) * 0.5 - 4.0
    perm = torch.randperm(width, generator=g)
    rows[4, perm[:20]] = torch.arange(20, dtype=torch.float32) * 0.25 + 3.0
    rows[4, perm[20:1120]] = 2.0
    return rows.half().float()


def tied_cut_rows(rows, sup_r, sup_o):
    """Rows whose top-p cut falls inside a run of equal logits and where the reference's unstable torch.sort kept another subset
    of that run than the oracle (which keeps the lowest ids, the order the device sampler defines): every token above the run's
    value is kept by both, none below it, and both keep as many of the run."""
    out = []
    for b in range(rows.shape[0]):
        if torch.equal(sup_r[b], sup_o[b]):
            continue
        v = float(rows[b][sup_o[b]].min())
        run = rows[b] == v
        assert torch.equal(sup_r[b] & ~run, sup_o[b] & ~run) and int((sup_r[b] & run).sum()) == int((sup_o[b] & run).sum()), b
        assert int(run.sum()) > int((sup_o[b] & run).sum()), b
        out.append(b)
    return out


def case_name(rng, top_k, top_p, temp):
    return f"{rng}.k{top_k}.p{top_p}.t{temp}"


def main():
    cfg = llama.lm_small()
    ref = build_reference(cfg, llama.make_lm_state_dict(cfg, 5, 4.0))
    out, report = {}, {}
    for ri, (rng, (lo, width)) in enumerate(RANGES.items()):
        rows = range_rows(width, 100 + ri)
        out[f"{rng}.logits"] = rows.numpy()
        full = torch.full((rows.shape[0], V), float("-inf"))
        full[:, lo:lo + width] = rows
        for top_k in TOP_K:
            for top_p in TOP_P:
                for temp in TEMPS:
                    work = full.clone()
                    with torch.no_grad():
                        ref.sample_logits(work, temperature=temp, top_k=top_k, top_p=top_p, do_sample=False)   # filters in place
                    probs_r = torch.softmax(work / temp, -1)[:, lo:lo + width]          # what torch.multinomial draws from
                    sup_r = torch.isfinite(work[:, lo:lo + width])
                    assert not torch.isfinite(work[:, :lo]).any() and not torch.isfinite(work[:, lo + width:]).any()
                    probs_o = lm_sampling.sample_filter(rows, temp, top_k, top_p)
                    tied = tied_cut_rows(rows, sup_r, probs_o > 0)
                    same = [bool(torch.equal(sup_r[b], probs_o[b] > 0)) for b in range(rows.shape[0])]
                    err = float((probs_r.sort(-1).values - probs_o.sort(-1).values).abs().max())
                    dist = [lm_sampling.top_p_distance(r, top_k, top_p) for r in rows]
                    name = case_name(rng, top_k, top_p, temp)
                    report[name] = dict(support=sup_r.sum(1).tolist(), support_identical=same, tied_cut_rows=tied,
                                        sorted_probs_max_abs_diff=err, top_p_boundary_distance=dist)
                    print(name, report[name])
                    assert all(same[b] or b in tied for b in range(rows.shape[0])) and err < 1e-6, name
                    out[f"{name}.tied_cut"] = np.array(tied, dtype=np.int32)
                    top = torch.topk(probs_r, 32, -1)
                    out[f"{name}.support"] = np.packbits(sup_r.numpy(), axis=1)
                    out[f"{name}.probs_max"] = probs_r.max(-1).values.numpy()
                    out[f"{name}.top_ids"] = top.indices.numpy().astype(np.int32)
                    out[f"{name}.top_probs"] = top.values.numpy()
    meta = dict(vocab=V, ranges=RANGES, top_k=TOP_K, top_p=TOP_P, temperatures=TEMPS,
                reference="QuarkAudio-UniSE/model/llm/llm.py:253-289 sample_logits (unmodified)")
    np.savez_compressed(os.path.join(GOLD, "lm_sampling.npz"), meta=np.array(json.dumps(meta)), **out)
    json.dump(report, open(os.path.join(GOLD, "lm_sampling_pinning_report.json"), "w"), indent=1)
    print("wrote lm_sampling.npz", os.path.getsize(os.path.join(GOLD, "lm_sampling.npz")), "bytes")


if __name__ == "__main__":
    main()
