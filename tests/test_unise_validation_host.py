"""UniSE's validation surface without a GPU: `unise.Model._validation_step` against what the REFERENCE'S OWN `validation_step`
(U/model/model.py:134-160, run unmodified by oracle/make_golden_unise_validation.py) logs with the same stand-ins, the refusals of
`validation_step`, and `validation_epoch`'s cross-rank batch-size-weighted mean (gloo, 2 processes)."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "unise_validation_glue.npz")


def stand_in_model():
    from oracle import unise_stubs as st
    from oracle import unise_validation_stubs as vs
    from unified_audio_b200.unise import Model
    return Model(None, tokenizer=vs.Tokenizer(), dnn=vs.Dnn(), semantic_model=st.SemanticModel())


def test_validation_step_control_flow_matches_reference_fixture():
    from oracle.make_golden_unise_validation import make_cases
    z = np.load(FIXTURE)
    cases = make_cases()
    assert json.loads(str(z["meta"]))["cases"] == list(cases)
    model = stand_in_model()
    for name, batch in cases.items():
        model.dnn.calls = []
        out = model._validation_step(batch)
        assert sorted(out) == ["valid_acc", "valid_loss"]
        for k in ("valid_loss", "valid_acc"):
            v = out[k]
            assert v.dtype == torch.float32 and v.dim() == 0, (name, k)
            assert np.array_equal(v.numpy(), z[f"{name}.{k}"]), (name, k, float(v), float(z[f"{name}.{k}"]))
        assert len(model.dnn.calls) == 1
        assert json.dumps(model.dnn.calls[0], sort_keys=True) == str(z[f"{name}.call"]), name
        assert json.loads(str(z[f"{name}.log_kwargs"])) == dict(on_step=False, on_epoch=True, sync_dist=True)
    # the cases the fixture must tell apart: interf ignored by 'se', interf tokenized by 'rtse', enrollment in the prefix
    call = lambda n: json.loads(str(z[f"{n}.call"]))
    assert call("se") == call("se_interf") and call("tse")["semantic_ids"] == call("se")["semantic_ids"]
    assert call("rtse")["semantic_ids"] != call("tse")["semantic_ids"] and call("tse")["enroll"] and not call("tse_no_enroll")["enroll"]
    unequal = call("se_unequal")
    assert len(unequal["semantic_ids"][0]) != unequal["mix_frames"]


@pytest.mark.skipif(not os.path.isdir("/root/reference/QuarkAudio-UniSE/model"), reason="the reference tree is not on this machine")
def test_generator_reproduces_committed_fixture(tmp_path):
    out = tmp_path / "unise_validation_glue.npz"
    subprocess.run([sys.executable, "-m", "oracle.make_golden_unise_validation", "--out", str(out)], cwd=ROOT, check=True,
                   capture_output=True)
    a, b = np.load(out), np.load(FIXTURE)
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert np.array_equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------------- refusals
def small_tokenizer(feature_extractor=True, semantic_tokens=True):
    from oracle.make_golden_bicodec_semantic import e2e_wav2vec2_config, small_config
    from unified_audio_b200.bicodec import BiCodec
    from unified_audio_b200.ssl import SSLFrontEnd
    from unified_audio_b200.unise import BiCodecTokenizer
    codec = BiCodec(small_config(), global_tokens=True, semantic_tokens=semantic_tokens)
    w2v = SSLFrontEnd(dict(e2e_wav2vec2_config(), kind="wav2vec2", do_normalize=True), in_rate=16000) if feature_extractor else None
    return BiCodecTokenizer(codec, ref_segment_length=9600, feature_extractor=w2v)


def batch(mode="se", B=2, enroll=False, interf=False, Bs=None, Be=None, Bi=None):
    g = torch.Generator().manual_seed(3)
    w = lambda b: 0.1 * torch.randn(b, 6400, generator=g)
    return (mode, w(Be or B) if enroll else None, w(B), w(Bs or B), w(Bi or B) if interf else None, torch.full((B,), 16000),
            torch.full((B,), 6400), ["x"] * B)


def test_validation_step_refusals():
    from oracle import unise_stubs as st
    from oracle import unise_validation_stubs as vs
    from unified_audio_b200.unise import Model
    model = lambda tok: Model(None, tokenizer=tok, dnn=vs.Dnn(), semantic_model=st.SemanticModel())
    # a tokenizer that cannot tokenize: its own NotImplementedError, before the device check (these tensors are on the CPU)
    detok_only = model(small_tokenizer(feature_extractor=False, semantic_tokens=False))
    with pytest.raises(NotImplementedError, match=r"feature_extractor.*semantic_tokens=True"):
        detok_only.validation_step(batch())
    with pytest.raises(NotImplementedError, match=r"semantic_tokens=True") as e:
        model(small_tokenizer(semantic_tokens=False)).validation_step(batch())
    assert "feature_extractor" not in str(e.value)
    with pytest.raises(NotImplementedError, match=r"feature_extractor"):
        model(small_tokenizer(feature_extractor=False)).validation_step(batch())
    # inputs the reference would only fail on later
    m = model(small_tokenizer())
    with pytest.raises(ValueError, match="unknown mode 'ss'"):
        m.validation_step(batch("ss"))
    with pytest.raises(ValueError, match="tokenizes `interf`, which is None"):
        m.validation_step(batch("rtse", enroll=True))
    with pytest.raises(ValueError, match="batch sizes differ"):
        m.validation_step(batch("se", Bs=3))
    with pytest.raises(ValueError, match="batch sizes differ"):
        m.validation_step(batch("tse", enroll=True, Be=1))
    with pytest.raises(ValueError, match="batch sizes differ"):
        m.validation_step(batch("rtse", enroll=True, interf=True, Bi=3))
    with pytest.raises(RuntimeError, match="CUDA only"):       # 'rtse' does not tokenize `speech`, so its size is not checked
        m.validation_step(batch("rtse", interf=True, Bs=3))
    # a valid batch on the CPU: no fallback
    for b in (batch("se"), batch("tse", enroll=True, interf=True), batch("rtse", enroll=True, interf=True)):
        with pytest.raises(RuntimeError, match="CUDA only"):
            m.validation_step(b)
    # the glue does not need an enrollment in any mode
    glue = stand_in_model()
    for mode in ("se", "tse", "rtse"):
        out = glue._validation_step(batch(mode, interf=True))
        assert not glue.dnn.calls[-1]["enroll"] and torch.isfinite(out["valid_loss"])


# ---------------------------------------------------------------------------------------------------------------- cross-rank mean
def epoch_batches():
    """two ranks with unequal batch counts and sizes: rank 0 gets batches of 1, 3 and 2 clips, rank 1 one batch of 4"""
    g = torch.Generator().manual_seed(40)
    out = []
    for i, B in enumerate((1, 3, 2, 4)):
        mode = ("se", "tse", "rtse", "tse")[i]
        w = lambda L: 0.1 * torch.randn(B, L, generator=g)
        out.append((mode, w(9000) if mode != "se" else None, w(12800), w(12800), w(12800), torch.full((B,), 16000),
                    torch.full((B,), 12800), ["x"] * B))
    return [out[:3], out[3:]]


def host_model():
    """a stand-in Model whose validation_step is the device-agnostic glue, so validation_epoch runs on the CPU"""
    from oracle import unise_stubs as st
    from oracle import unise_validation_stubs as vs
    from unified_audio_b200.unise import Model

    class HostModel(Model):
        def validation_step(self, batch, batch_idx=0):
            return self._validation_step(batch)
    return HostModel(None, tokenizer=vs.Tokenizer(), dnn=vs.Dnn(), semantic_model=st.SemanticModel())


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _epoch_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ret[rank] = host_model().validation_epoch(epoch_batches()[rank])
    dist.destroy_process_group()


def test_validation_epoch_cross_rank_weighted_mean_gloo():
    shards = epoch_batches()
    one = host_model()
    single = one.validation_epoch(shards[0] + shards[1])
    # the rule: Σ B·x / Σ B over every batch, from the steps' own fp32 values
    steps = [(b[2].shape[0], one.validation_step(b)) for b in shards[0] + shards[1]]
    n = sum(B for B, _ in steps)
    for k in ("valid_loss", "valid_acc"):
        want = sum(B * float(o[k]) for B, o in steps) / n
        assert abs(single[k] - want) <= 1e-12 * abs(want), k
    assert abs(single["valid_loss"] - np.mean([float(o["valid_loss"]) for _, o in steps])) > 1e-6     # not the unweighted mean
    ret = mp.Manager().dict()
    mp.spawn(_epoch_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    for r in range(2):
        for k in ("valid_loss", "valid_acc"):
            assert abs(ret[r][k] - single[k]) <= 1e-12 * abs(single[k]), (r, k, ret[r][k], single[k])
    with pytest.raises(ValueError, match="no batch"):
        one.validation_epoch([])
