"""UniSE batched inference on the GPU: `Model.enhance_batch` over utterances (and 'tse' enrollments) of different lengths equals
`enhance` of each utterance alone - identical tokens, bit-identical waveforms - and `test_epoch` returns and writes what `test_step`
does per batch.  'tse' against the chain of oracles.  Reduced widths (tests/test_unise_gpu.py::build)."""
import os

import numpy as np
import pytest
import torch

from test_unise_gpu import SEG, TOL, build, check_tokens, ref_segments, rel

pytestmark = pytest.mark.gpu


def utterances(seed):
    """1, 2 and 3 segments, exactly one segment, shorter than one; enrollments of 0.6 to 4 s"""
    g = torch.Generator().manual_seed(seed)
    srcs = [0.1 * torch.randn(1, n, generator=g) for n in (SEG - 999, 2 * SEG + 17, 3 * SEG - 5000, SEG, 12345)]
    enrolls = [0.1 * torch.randn(1, n, generator=g) for n in (16000, 47000, 9000, 30000, 64000)]
    return srcs, enrolls


def as_tuple(out):
    return out if isinstance(out, tuple) else (out,)


@pytest.fixture(scope="module")
def built(lib):
    model, o = build()
    model.dnn.lane_att_unroll = model.dnn.att_unroll      # same decode-attention summation order on every side of a comparison
    return model, o


@pytest.mark.parametrize("mode", ["se", "tse", "ss"])
def test_enhance_batch_equals_enhance_alone(built, mode):
    model, _ = built
    srcs, enrolls = utterances(41)
    srcs, enrolls = [s.cuda() for s in srcs], [e.cuda() for e in enrolls]
    want = [model.enhance(mode, e if mode == "tse" else None, s, return_ids=True) for s, e in zip(srcs, enrolls)]
    for max_segments in (128, 4):
        got = model.enhance_batch(mode, enrolls if mode == "tse" else None, srcs, return_ids=True, max_segments=max_segments)
        torch.cuda.synchronize()
        assert len(got) == len(srcs)
        for u, (g, w) in enumerate(zip(got, want)):
            assert len(g) == len(w) and as_tuple(g)[0].shape == (srcs[u].size(-1),)
            for a, b in zip(g, w):
                assert a.shape == b.shape and torch.equal(a, b), f"{mode} utterance {u} differs (max_segments {max_segments})"


def test_enhance_batch_tse_vs_oracle_chain(built):
    """ragged 'tse' prefixes against the reference's path on the oracles: wrap-pad + segment (NumPy) -> WavLM (oracle/hubert.py) of
    each enrollment alone, repeated per segment -> LLM_SFT.generate (oracle/llama.py) -> BiCodec.detokenize (oracle/bicodec.py)"""
    from oracle import bicodec as ob
    from oracle import hubert as oh
    from oracle import llama
    model, o = built
    srcs, enrolls = utterances(43)
    srcs, enrolls = srcs[:3], [enrolls[1], enrolls[2], enrolls[0]]
    got = model.enhance_batch("tse", [e.cuda() for e in enrolls], [s.cuda() for s in srcs], return_ids=True)
    torch.cuda.synchronize()
    for u, (src, enr) in enumerate(zip(srcs, enrolls)):
        est, gids, sids = got[u]
        seg = ref_segments(src, normalise=False)
        feats = oh.extract_semantic_features(o["wsd"], o["c"], seg)
        efeats = torch.cat([oh.extract_semantic_features(o["wsd"], o["c"], enr)] * seg.size(0), 0)
        og, os_, margins = llama.sft_generate(o["lsd"], o["lcfg"], "tse", efeats, feats, SEG // 320, return_margins=True)
        check_tokens(f"tse utterance {u}", torch.cat([gids.cpu(), sids.cpu()], 1), torch.cat([og, os_], 1),
                     torch.cat([margins[:, :32], margins[:, 33:]], 1))
        wav = ob.detokenize(o["bsd"], o["bc"], sids.cpu(), gids.cpu()[:, None, :]).squeeze(1).reshape(-1)[:src.size(-1)]
        e_wav = rel(est, wav)
        print(f"[enhance_batch tse utterance {u}] {seg.size(0)} segments, enrollment {enr.size(-1)} samples, waveform rel {e_wav:.2e}")
        assert e_wav < TOL


def test_test_epoch_equals_test_step(built, tmp_path):
    """consecutive batches of one mode are enhanced together; returns and written files equal test_step's, batch by batch"""
    model, _ = built
    srcs, enrolls = utterances(47)
    modes = ["se", "se", "tse", "tse", "ss", "se"]
    batches = [(m, enrolls[i % 5].cuda() if m == "tse" else None, srcs[i % 5].cuda(), None, [16000], None, [f"utt{i}"])
               for i, m in enumerate(modes)]
    model.config["save_enhanced"] = str(tmp_path / "epoch")
    os.makedirs(model.config["save_enhanced"])
    try:
        got = model.test_epoch(batches, max_segments=5)          # 5: the first two 'se' batches (4 segments) share one call
        model.config["save_enhanced"] = str(tmp_path / "step")
        os.makedirs(model.config["save_enhanced"])
        want = [model.test_step(b, i) for i, b in enumerate(batches)]
    finally:
        model.config.pop("save_enhanced")
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        g, w = (g, w) if modes[i] == "ss" else ([g], [w])
        assert len(g) == len(w) and all(isinstance(a, np.ndarray) and np.array_equal(a, b) for a, b in zip(g, w)), f"batch {i}"
    files = sorted(os.listdir(tmp_path / "step"))
    assert files == sorted(os.listdir(tmp_path / "epoch")) and len(files) == 7
    for f in files:
        assert (tmp_path / "step" / f).read_bytes() == (tmp_path / "epoch" / f).read_bytes(), f
