"""Deterministic stand-ins for the components `Model.validation_step` glues together (TEST INFRASTRUCTURE).

Used twice with identical arithmetic: by oracle/make_golden_unise_validation.py under the REFERENCE's unmodified `validation_step`
(QuarkAudio-UniSE/model/model.py:134-160) and by tests/test_unise_validation_host.py under
`unified_audio_b200.unise.Model._validation_step`.  The semantic model is `oracle.unise_stubs.HFSemanticModel` / `SemanticModel`.
Every float that reaches an output is first quantised to an integer (floor of a scaled fp64 value), so the recorded values do not
depend on the last bits of a CPU's fp32 matmul or summation order.
"""
import torch

from oracle.unise_stubs import TASKS


def _q(x: torch.Tensor, scale: float) -> torch.Tensor:
    return torch.floor(x.double() * scale).long()


class Tokenizer:
    """tokenize(wav [B, L]) -> (global int32 [B, 1, 32], semantic int64 [B, T']), T' = (L - 400) // 320 + 1: wav2vec2's unpadded
    frame count (80 000 samples -> 249), so T' differs from the WavLM frame count of the same length.  The semantic ids follow
    the energy of each frame, the global ids the whole waveform."""

    def tokenize(self, wav):
        B, L = wav.shape
        frames = wav.double().unfold(-1, 400, 320)
        T = frames.shape[1]
        semantic = (_q(frames.pow(2).sum(-1), 1e4) + 7 * torch.arange(T)) % 8192
        key = _q(wav.double().abs().sum(-1), 1e3)
        glob = (key[:, None] + 13 * torch.arange(32)) % 4096
        return glob.to(torch.int32)[:, None, :], semantic


class Dnn(torch.nn.Module):
    """`LLM_SFT.forward`'s signature -> (loss, acc), fp32 0-d tensors that depend on every argument it reads: the task, whether the
    enrollment mel is None (llm_sft.py:69), the enrollment and mix features, both id tensors, and the mix mel's batch size (its only
    use of `mix_mel`, llm_sft.py:60).  Each call is recorded in `calls` as JSON-ready values."""

    def __init__(self):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.zeros(()), requires_grad=False)    # where the LM's weights live (validation_epoch)
        self.calls = []

    def forward(self, task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, global_ids, semantic_ids):
        B = mix_mel.size(0)
        assert global_ids.dtype == torch.int32 and tuple(global_ids.shape) == (B, 32)
        assert semantic_ids.dtype == torch.int64 and semantic_ids.size(0) == B and mix_feats.size(0) == B
        enroll = enroll_feats if enroll_mel is not None else None
        rows = lambda x: (_q(x.double().sum(-1), 1e3) *(1 + torch.arange(x.size(1)))).sum(1)     # per clip, order-sensitive
        mix_key = rows(mix_feats)
        enroll_key = rows(enroll) if enroll is not None else torch.zeros(B, dtype=torch.long)
        g_key = (global_ids.long() * (1 + torch.arange(32))).sum(1)
        s_key = (semantic_ids * (1 + torch.arange(semantic_ids.size(1)))).sum(1)
        key = (7 * TASKS[task_name] + 11 * int(enroll is not None) + mix_key + 3 * enroll_key + 5 * g_key + 13 * s_key
               + 17 * semantic_ids.size(1) + 19 * mix_feats.size(1))
        loss = (1.0 + 8.0 * (key % 100003).double() / 100003).mean().float()
        acc = ((key // 7) % 1000).double().div(1000).mean().float()
        self.calls.append(dict(task=task_name, enroll=enroll is not None, B=int(B), mix_frames=int(mix_feats.size(1)),
                               enroll_frames=None if enroll is None else int(enroll.size(1)), mix_key=mix_key.tolist(),
                               enroll_key=enroll_key.tolist(), global_ids=global_ids.tolist(), semantic_ids=semantic_ids.tolist()))
        return loss, acc
