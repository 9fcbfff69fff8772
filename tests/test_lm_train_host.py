"""CPU checks of the training oracle: its fp64 autograd reproduces the gradients of the reference's own LLM_SFT.forward
(tests/golden/lm_reference_grads.npz, written by oracle/make_golden_lm_grads.py: small gradients whole, large ones as seeded Gaussian
projections), and the NumPy restatement of the attention dropout mask is the documented Philox function, deterministic, and keeps
1 - p of the entries."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import llama, llama_train

GOLD = os.path.join(os.path.dirname(__file__), "golden", "lm_reference_grads.npz")


@pytest.mark.parametrize("task", ["se", "tse"])
def test_oracle_grads_match_reference_fixture(task):
    z = np.load(GOLD)
    meta = json.loads(str(z["meta"]))
    cfg = meta["cfg"]
    sd = {k: v.double().requires_grad_(True) for k, v in llama.make_lm_state_dict(cfg, meta["seed"], meta["gain"]).items()}
    enroll = torch.from_numpy(z["enroll"]) if task == "tse" else None
    loss, _ = llama_train.sft_forward(sd, cfg, task, enroll, torch.from_numpy(z["mix"]), torch.from_numpy(z["gids"]),
                                      torch.from_numpy(z["sids"]))
    loss.backward()
    # the reference computes its loss from fp32 logits (llm.py:88): agreement to fp32 rounding
    assert abs(float(loss) - float(z[f"{task}.loss"])) < 1e-6 * abs(float(z[f"{task}.loss"]))
    keys = [k for k in z.files if k.startswith(f"{task}.grad.")]
    assert len(keys) == len(sd) - (1 if task == "se" else 0)          # 'se' never reads enroll_sos_embedding
    for k in keys:              # small gradients whole, large ones as seeded projections (llama_train.grad_sketch)
        name = k[len(f"{task}.grad."):]
        ref = torch.from_numpy(z[k])
        err = float((llama_train.grad_sketch(name, sd[name].grad) - ref).norm() / ref.norm())
        assert err < 1e-4, (name, err)


def test_dropout_mask_is_the_documented_philox():
    seed, layer, B, heads, L, p = 0x1234_5678_9ABC_DEF0, 3, 2, 2, 37, 0.1
    keep = llama_train.dropout_keep(seed, layer, B, heads, L, p)
    thr = round(p * 2 ** 24)
    for b, h, i, j in ((0, 0, 0, 0), (1, 1, 36, 36), (0, 1, 5, 17), (1, 0, 20, 3), (1, 1, 9, 30)):
        r = llama.philox4x32_10((seed & 0xFFFFFFFF, seed >> 32), (i, j >> 2, b * heads + h, layer))[j & 3]
        assert bool(keep[b, h, i, j]) == ((r >> 8) >= thr)


def test_dropout_mask_deterministic_and_binomial():
    B, heads, L, p = 2, 4, 200, 0.1
    a = llama_train.dropout_keep(7, 0, B, heads, L, p)
    assert np.array_equal(a, llama_train.dropout_keep(7, 0, B, heads, L, p))
    assert not np.array_equal(a, llama_train.dropout_keep(8, 0, B, heads, L, p))
    assert not np.array_equal(a, llama_train.dropout_keep(7, 1, B, heads, L, p))
    n = a.size
    sd = (n * p * (1 - p)) ** 0.5
    assert abs(int(a.sum()) - n * (1 - p)) < 5 * sd
    assert llama_train.dropout_keep(7, 0, B, heads, L, 0.0).all()
