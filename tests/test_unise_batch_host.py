"""CPU: `unise.Model._enhance_batch` (the body of `enhance_batch`) with the deterministic stand-ins of oracle/unise_stubs.py.  Every
utterance of a batch must come out exactly as the reference's own `test_step` made it (tests/golden/unise_glue.npz) and as
`_enhance` makes it alone, whatever else is in the batch: wrap padding, the 'se' peak normalisation, the enrollment of each
utterance, the se -> tse -> rtse chain of 'ss' and the trimming all stay per utterance.  (The device kernel behind wrap_segments is
replaced by the NumPy expression it implements, as in tests/test_host.py.)"""
import json
import math
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")
SEG = 5 * 16000


class RaggedDnn:
    """the stub LM, honouring generate's `enroll_lengths` row by row: row b sees only its first enroll_lengths[b] enrollment frames"""

    def __init__(self):
        from oracle import unise_stubs as st
        self.inner = st.Dnn()

    @property
    def calls(self):
        return self.inner.calls

    @calls.setter
    def calls(self, v):
        self.inner.calls = v

    def generate(self, task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, do_sample=True, enroll_lengths=None, **kw):
        if enroll_lengths is None:
            return self.inner.generate(task_name, enroll_mel, enroll_feats, mix_mel, mix_feats, do_sample=do_sample, **kw)
        assert len(enroll_lengths) == mix_feats.size(0) and max(enroll_lengths) <= enroll_feats.size(1)
        outs = [self.inner.generate(task_name, enroll_mel[b:b + 1], enroll_feats[b:b + 1, :n], mix_mel[b:b + 1], mix_feats[b:b + 1],
                                    do_sample=do_sample, **kw) for b, n in enumerate(enroll_lengths)]
        return torch.cat([o[0] for o in outs], 0), torch.cat([o[1] for o in outs], 0)


@pytest.fixture
def model(monkeypatch):
    from oracle import unise_stubs as st
    from unified_audio_b200 import unise

    def wrap_np(src, seg_len):
        pad = math.ceil(src.shape[-1] / seg_len) * seg_len - src.shape[-1]
        return torch.from_numpy(np.pad(src.numpy(), [(0, 0), (0, pad)], "wrap")).reshape(-1, seg_len)
    monkeypatch.setattr(unise, "wrap_segments", wrap_np)
    return unise.Model(None, tokenizer=st.Tokenizer(), dnn=RaggedDnn(), semantic_model=st.SemanticModel())


def extra_utterances(seed):
    """sources of 1, 2 and 3 segments, exactly one segment and shorter than one; enrollments of other lengths than the fixture's"""
    g = torch.Generator().manual_seed(seed)
    srcs = [0.1 * torch.randn(1, n, generator=g) for n in (SEG - 999, 2 * SEG + 17, 3 * SEG - 5000, SEG, 12345)]
    enrolls = [0.1 * torch.randn(1, n, generator=g) for n in (16000, 47000, 9000, 30000, 64000)]
    return srcs, enrolls


def outputs(out):
    return out if isinstance(out, tuple) else (out,)


@pytest.mark.parametrize("max_segments", [128, 2])
def test_enhance_batch_reproduces_reference_fixture(model, max_segments):
    """each fixture case alone and in the middle of a batch of other lengths; max_segments=2 cuts utterances across calls"""
    from oracle.make_golden_unise import digest, make_cases
    z = np.load(os.path.join(GOLD, "unise_glue.npz"))
    extra_src, extra_enr = extra_utterances(7)
    for name, (enroll, src) in make_cases().items():
        mode = name.split("_")[0]
        enr = enroll if enroll is not None else 0.1 * torch.randn(1, 20000, generator=torch.Generator().manual_seed(3))
        for srcs, enrolls, at in (([src], [enr], 0), (extra_src[:2] + [src] + extra_src[2:], extra_enr[:2] + [enr] + extra_enr[2:], 2)):
            with torch.no_grad():
                outs = model._enhance_batch(mode, enrolls if mode == "tse" else None, srcs, max_segments=max_segments)
            assert len(outs) == len(srcs)
            for i, o in enumerate(outputs(outs[at])):
                got, want = digest(o.numpy()), z[f"{name}.est{i}"]
                assert got.shape == want.shape and np.array_equal(got, want), f"{name} output {i} (batch of {len(srcs)}) differs"


@pytest.mark.parametrize("mode", ["se", "tse", "ss"])
def test_enhance_batch_equals_enhance_per_utterance(model, mode):
    """every utterance of a mixed-length batch (and its ids) equals `_enhance` of that utterance alone, bit for bit"""
    srcs, enrolls = extra_utterances(11)
    with torch.no_grad():
        for max_segments in (128, 3):
            outs = model._enhance_batch(mode, enrolls if mode == "tse" else None, srcs, return_ids=True, max_segments=max_segments)
            for u, (src, enr) in enumerate(zip(srcs, enrolls)):
                want = model._enhance(mode, enr if mode == "tse" else None, src, return_ids=True)
                got = outs[u]
                assert len(got) == len(want)
                for a, b in zip(got, want):
                    assert a.shape == b.shape and torch.equal(a, b), f"{mode} utterance {u} (max_segments {max_segments})"
                assert outputs(got)[0].shape == (src.size(-1),)


def test_ragged_lm_prefix_layout():
    """LLM_SFT._ragged_prefix: row b of the uniform prefix [task, enroll_sos, enroll (Te_max), mix_sos, mix] becomes
    [task, enroll_sos, enroll[:n_b], mix_sos, mix] followed by zero rows up to the padded width"""
    from unified_audio_b200.llm import LLM_SFT
    te_max, T, H = 6, 4, 3
    lens = [6, 1, 3]
    B, P = len(lens), 3 + te_max + T
    prefix = torch.randn(B, P, H, generator=torch.Generator().manual_seed(1))
    got = LLM_SFT._ragged_prefix(prefix, lens, te_max)
    for b, n in enumerate(lens):
        want = torch.cat([prefix[b, :2 + n], prefix[b, 2 + te_max:], torch.zeros(te_max - n, H)], 0)
        assert torch.equal(got[b], want), b


def test_enhance_batch_refuses_bad_input(model):
    src = torch.zeros(1, SEG)
    with pytest.raises(ValueError):
        model._enhance_batch("se", None, [])                              # no utterance
    with pytest.raises(ValueError):
        model._enhance_batch("tse", [src], [src, src])                    # enrollment count != utterance count
    with pytest.raises(ValueError):
        model._enhance_batch("tse", None, [src])                          # 'tse' without enrollments
    with pytest.raises(ValueError):
        model._enhance_batch("rtse", None, [src])                         # unknown mode (test_step has no 'rtse')
    with pytest.raises(ValueError):
        model._enhance_batch("se", None, [torch.zeros(2, SEG)])           # one utterance per src
    with pytest.raises(ValueError):
        model._enhance_batch("se", None, [src], max_segments=0)
    with pytest.raises(RuntimeError):
        model.enhance_batch("se", None, [src])                            # CPU tensors: no fallback
    assert json.dumps(model.dnn.calls) == "[]"                            # nothing reached the LM
