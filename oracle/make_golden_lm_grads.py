"""Pin oracle/llama_train.py's gradients against the REFERENCE'S OWN `LLM_SFT.forward` + `loss.backward()`.

TEST INFRASTRUCTURE.  Run in the build container only:  python -m oracle.make_golden_lm_grads

The reference's classes run unmodified through the shims of oracle/make_golden_lm_reference.py, at the small config, in eval mode (no
attention dropout), for 'se' and 'tse', in fp64 (its loss_function casts the logits to fp32, llm.py:88, so the pin holds to fp32
rounding).  Every parameter's gradient goes to tests/golden/lm_reference_grads.npz as `llama_train.grad_sketch` keeps it (small tensors
whole, large ones as 256 seeded Gaussian projections), with a pinning report (relative Frobenius difference of the full gradients to the
oracle's fp64 autograd); tests/test_lm_train_host.py re-checks the oracle against the fixture without the reference.
"""
import json
import os

import numpy as np
import torch

from oracle import llama, llama_train
from oracle.make_golden_lm_reference import GOLD, build_reference

SEED, GAIN = 5, 4.0
B, T, TE = 2, 12, 7


def inputs(cfg):
    b = cfg["llm_base_config"]
    g = torch.Generator().manual_seed(21)
    return dict(mix=torch.randn(B, T, cfg["feats_dim"], generator=g, dtype=torch.float64),
                enroll=torch.randn(B, TE, cfg["feats_dim"], generator=g, dtype=torch.float64),
                gids=torch.randint(0, b["global_size"], (B, 32), generator=g),
                sids=torch.randint(0, b["semantic_size"], (B, T), generator=g))


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def main():
    cfg = llama.lm_small()
    sd = {k: v.double() for k, v in llama.make_lm_state_dict(cfg, SEED, GAIN).items()}
    ref = build_reference(cfg, sd).double().eval()
    x = inputs(cfg)
    out, report = {k: v.numpy() for k, v in x.items()}, {}
    for task in ("se", "tse"):
        e_feats = x["enroll"] if task == "tse" else None
        e_mel = torch.zeros(B, TE, 80) if task == "tse" else None
        ref.zero_grad(set_to_none=True)
        loss_r, _ = ref(task, e_mel, e_feats, torch.zeros(B, T, 80), x["mix"], x["gids"], x["sids"])
        loss_r.backward()
        grads = {n: p.grad.detach().clone() for n, p in ref.named_parameters() if p.grad is not None and n in sd}
        osd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        loss_o, _ = llama_train.sft_forward(osd, cfg, task, e_feats, x["mix"], x["gids"], x["sids"])
        loss_o.backward()
        rep = dict(loss_reference=float(loss_r.detach()), loss_oracle=float(loss_o), grads={})
        for n, gr in grads.items():
            rep["grads"][n] = rel(osd[n].grad, gr)
            out[f"{task}.grad.{n}"] = llama_train.grad_sketch(n, gr).numpy()
        missing = sorted(n for n in sd if n not in grads)
        rep["no_grad"] = missing
        rep["max_rel"] = max(rep["grads"].values())
        print(task, float(loss_r), "max rel grad diff", rep["max_rel"], "no grad:", missing)
        # the reference's loss_function casts the logits to fp32 (llm.py:88): its loss and gradients carry fp32 rounding
        assert abs(float(loss_r) - float(loss_o)) < 1e-6 * abs(float(loss_r)) and rep["max_rel"] < 1e-4
        out[f"{task}.loss"] = np.float64(loss_r)
        report[task] = rep
    meta = dict(cfg=cfg, seed=SEED, gain=GAIN, B=B, T=T, Te=TE, dtype="float64", mode="eval (no attention dropout)",
                reference="QuarkAudio-UniSE/model/llm/llm_sft.py:37-89, llm.py:87-104 (unmodified) + loss.backward()",
                shims="oracle/make_golden_lm_reference.py")
    np.savez_compressed(os.path.join(GOLD, "lm_reference_grads.npz"), meta=np.array(json.dumps(meta)), **out)
    json.dump(report, open(os.path.join(GOLD, "lm_reference_grads_pinning_report.json"), "w"), indent=1)
    print("wrote lm_reference_grads.npz", os.path.getsize(os.path.join(GOLD, "lm_reference_grads.npz")), "bytes")


if __name__ == "__main__":
    main()
