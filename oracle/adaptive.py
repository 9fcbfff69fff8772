"""CPU restatement of the data-dependent primitives of H-Codec-1.5's adaptive frame-rate path (SURVEY.md 8f.4) - groundwork.

TEST INFRASTRUCTURE - see oracle/__init__.py.  Paths relative to /root/reference/QuarkAudio-HCodec/HCodec-1.5/.
H-Codec-1.5 = the H-Codec-1.0 encoder / RVQ / decoder (already built: unified_audio_b200/codec_h1.py) plus
  * similarity alignment: consecutive 50 Hz frames whose semantic embeddings have cosine similarity > threshold are merged into
    one token, at most `max_tokens_per_group` frames per token (adaptive/modeling_flexicodec_new.py:828-921);
  * query-token aggregators + a bottleneck transformer (mimi `ProjectedTransformer`, adaptive/model_blocks/mimi/transformer.py)
    - NOT restated here;
  * token lengths packed into the code indices, index = (length - 1) * codebook_size + code (vq/codec_adaptive.py:68-80);
  * de-aggregation by length: every token repeated `length` times (modeling_flexicodec_new.py:1007-1041).
Pinned by oracle/make_golden_adaptive.py against the reference's own static methods (exact: these are index computations).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def similarity_alignment(h: torch.Tensor, threshold: float, max_tokens_per_group: int = 8):
    """h [B,T,D] (all frames valid) -> (alignment [B,G,T] float 0/1, sim [B,T-1], groups per item [B])"""
    B, T, _ = h.shape
    if T <= 1:
        return torch.ones(B, 1, T), torch.ones(B, max(T - 1, 0)), torch.ones(B, dtype=torch.long)
    sim = F.cosine_similarity(h[:, :-1], h[:, 1:], dim=2)
    seg, _, n_groups = segments_from_sim(sim, threshold, max_tokens_per_group)
    G = int(n_groups.max())
    align = torch.zeros(B, G, T)
    align[torch.arange(B)[:, None].expand(B, T), seg, torch.arange(T)[None].expand(B, T)] = 1.0
    return align, sim, n_groups


def segments_from_sim(sim: torch.Tensor, threshold: float, max_tokens_per_group: int = 8):
    """the grouping scan of similarity_alignment on given similarities sim [B,T-1] -> (frame -> token seg [B,T] int64,
    frames per token lengths [B,T] int64 (0 past each clip's last token), n_groups [B] int64).  A frame opens a token when its
    similarity to the previous frame is <= threshold or when the open token already holds max_tokens_per_group frames;
    max_tokens_per_group <= 0 means no cap."""
    B, T = sim.shape[0], sim.shape[1] + 1
    new_group = torch.cat([torch.ones(B, 1, dtype=torch.bool), sim <= threshold], 1)
    ar = torch.arange(T)[None]
    start = torch.cummax(ar * new_group.long(), dim=1).values               # index of the frame that opened the segment
    if max_tokens_per_group > 0:
        split = ((ar - start) % max_tokens_per_group) == 0                  # similarity boundary or length cap
    else:
        split = new_group
    seg = torch.cumsum(split.long(), 1) - 1                                 # frame -> token
    n_groups = seg[:, -1] + 1
    lengths = torch.zeros(B, T, dtype=torch.long).scatter_add_(1, seg, torch.ones_like(seg))
    return seg, lengths, n_groups


def token_lengths(align: torch.Tensor) -> torch.Tensor:
    """vq/codec_adaptive.py:181 - frames per token [B,G] (0 for padded groups)"""
    return align.sum(2).long()


def inject_lengths(codes: torch.Tensor, lengths: torch.Tensor, codebook_size: int) -> torch.Tensor:
    """codec_adaptive.py:68-73: codes [B,nq,G], lengths [B,G]"""
    return (lengths[:, None].to(codes.dtype) - 1) * codebook_size + codes


def extract_lengths(codes: torch.Tensor, codebook_size: int):
    """codec_adaptive.py:75-80 -> (plain codes, lengths from the first quantiser row)"""
    lid = torch.div(codes, codebook_size, rounding_mode="floor") + 1
    return codes % codebook_size, lid[:, 0]


def deaggregate(grouped: torch.Tensor, align: torch.Tensor) -> torch.Tensor:
    """modeling_flexicodec_new.py:970-1004 (channel-first): [B,D,G] x [B,G,T] -> [B,D,T]"""
    return torch.einsum("bdg,bgt->bdt", grouped, align)


def deaggregate_by_lengths(grouped: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """modeling_flexicodec_new.py:1007-1041: [B,D,G], lengths [B,G] -> [B,D,max T] zero padded"""
    outs = [torch.repeat_interleave(grouped[b].t(), lengths[b], dim=0) for b in range(grouped.shape[0])]
    T = max(o.shape[0] for o in outs)
    return torch.stack([F.pad(o, (0, 0, 0, T - o.shape[0])) for o in outs], 0).transpose(1, 2)
