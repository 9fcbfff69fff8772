"""H-Codec-1.5 adaptive frame-rate primitives on the device (SURVEY 8f.4) against the oracle (oracle/adaptive.py, pinned exact
against the reference's FlexiCodec static methods by tests/golden/adaptive_alignment.npz).  The grouping is checked by running the
oracle's scan (oracle.adaptive.segments_from_sim) on the kernel's own similarities, so it must agree exactly even where a similarity
lies within float error of the threshold; the kernels one by one are in tests/test_adaptive_kernels_gpu.py."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _assert_own_grouping(a, s, n, lens, thr, cap):
    """alignment / groups per clip / token lengths of ga.similarity_alignment == the oracle's scan of the kernel's own sim"""
    from oracle import adaptive as oa
    seg, lengths, ng = oa.segments_from_sim(s.cpu(), thr, cap)
    G = int(ng.max())
    assert torch.equal(n.cpu(), ng)
    assert torch.equal(a.cpu(), F.one_hot(seg, G).transpose(1, 2).float())
    assert torch.equal(lens.cpu(), lengths[:, :G])


def test_similarity_alignment_and_length_packing(lib):
    from oracle import adaptive as oa
    from unified_audio_b200 import adaptive as ga
    g = torch.Generator().manual_seed(3)
    for B, T, D, thr, cap in ((3, 50, 64, 0.6, 8), (2, 200, 512, 0.3, 4), (1, 2, 16, 0.9, 8), (4, 33, 128, -2.0, 3), (2, 40, 32, 2.0, 8)):
        base = torch.randn(B, T, D, generator=g)
        h = base.clone()
        for t in range(1, T):                                 # correlated frames so that both outcomes occur
            h[:, t] = 0.7 * h[:, t - 1] + 0.7 * base[:, t]
        align_o, sim, _ = oa.similarity_alignment(h, thr, cap)
        a2, s2, n2, lens = ga.similarity_alignment(h.cuda(), thr, cap)
        torch.cuda.synchronize()
        assert float((s2.cpu() - sim).abs().max()) < 1e-5
        _assert_own_grouping(a2, s2, n2, lens, thr, cap)
        assert torch.equal(a2.cpu(), align_o)                 # these cases keep every similarity >= 6e-4 from the threshold
        align, ng = a2.cpu(), n2.cpu()
        G = align.shape[1]
        codes = torch.randint(0, 1024, (B, 4, G), generator=g)
        ol = oa.token_lengths(align)                           # 0 in the padded groups: negative packed codes
        packed = ga.inject_lengths(codes.cuda(), ol.cuda(), 1024)
        assert torch.equal(packed.cpu(), oa.inject_lengths(codes, ol, 1024))
        plain, ln = ga.extract_lengths(packed, 1024)
        op, oln = oa.extract_lengths(oa.inject_lengths(codes, ol, 1024), 1024)
        assert torch.equal(plain.cpu(), op) and torch.equal(ln.cpu(), oln) and torch.equal(plain.cpu(), codes)
        assert torch.equal(ln.cpu(), ol)
        feats = torch.randn(B, 24, G, generator=g)
        tl = oa.token_lengths(align)
        assert torch.equal(ga.deaggregate_by_lengths(feats.cuda(), tl.cuda()).cpu(), oa.deaggregate_by_lengths(feats, tl))
        assert torch.equal(ga.deaggregate_by_lengths(codes.cuda(), tl.cuda()).cpu(), oa.deaggregate_by_lengths(codes, tl))
        assert torch.equal(ga.deaggregate(feats.cuda(), align.cuda()).cpu(), oa.deaggregate(feats, align))
        margin = float((sim - thr).abs().min())
        print(f"[adaptive B={B} T={T} thr={thr} cap={cap}] tokens per clip {ng.tolist()}, compression {T / float(ng.float().mean()):.2f}x, "
              f"closest similarity to the threshold {margin:.2e}")


def test_alignment_against_reference_fixture(lib):
    """the committed fixture holds the alignment matrices of the reference's own FlexiCodec._perform_similarity_alignment_vectorized;
    its closest similarity to a threshold is 7.9e-5 away, farther than the 1e-5 similarity bound, so the grouping must match it"""
    from oracle import adaptive as oa
    from unified_audio_b200 import adaptive as ga
    z = np.load(os.path.join(GOLD, "adaptive_alignment.npz"))
    h = torch.from_numpy(z["h"])
    for thr in (0.6, 0.85):
        a, s, n, lens = ga.similarity_alignment(h.cuda(), thr, 8)
        torch.cuda.synchronize()
        _, sim, _ = oa.similarity_alignment(h, thr, 8)
        assert float((s.cpu() - sim).abs().max()) < 1e-5
        _assert_own_grouping(a, s, n, lens, thr, 8)
        print(f"[adaptive fixture thr={thr}] closest similarity to the threshold {float((sim - thr).abs().min()):.2e}")
        assert torch.equal(a.cpu(), torch.from_numpy(z[f"align_{thr}"]))
        assert int(lens.max()) <= 8 and bool((lens.sum(1) == h.shape[1]).all())
