"""Data-dependent primitives of H-Codec-1.5's adaptive frame-rate path on the device (SURVEY.md 8f.4), with the reference's
call shapes:

    similarity_alignment(h [B,T,D], threshold, max_tokens_per_group) -> (alignment [B,G,T] 0/1, sim [B,T-1], groups per item [B])
        FlexiCodec._perform_similarity_alignment_vectorized   HCodec-1.5/adaptive/modeling_flexicodec_new.py:828-921
    inject_lengths(codes [B,nq,G], lengths [B,G], codebook_size) / extract_lengths(codes, codebook_size)
        Codec._inject_length_to_codes_index / _extract_length_from_codes_index   HCodec-1.5/vq/codec_adaptive.py:68-80
    deaggregate_by_lengths(grouped [B,C,G], lengths [B,G]) -> [B,C,max T]
        FlexiCodec._deaggregate_features_from_token_lengths   modeling_flexicodec_new.py:1007-1041
    deaggregate(grouped [B,D,G], alignment [B,G,T]) -> [B,D,T]                       modeling_flexicodec_new.py:970-1004

The codec that uses them (query-token aggregators, bottleneck transformer, H-Codec-1.0 blocks) is `codec_h15.CodecH15`.
No PyTorch / CPU fallback."""
from __future__ import annotations


import torch

from . import _lib
from .ops import _p, _stream


def similarity_alignment(h: torch.Tensor, threshold: float, max_tokens_per_group: int = 8, want_matrix: bool = True):
    """-> (alignment [B,G,T] float (or the frame -> token map [B,T] int32 if not want_matrix), sim [B,T-1], n_groups [B] int64,
    token lengths [B,G] int64)"""
    if h.device.type != "cuda":
        raise RuntimeError("unified_audio_b200.adaptive runs on CUDA only (no CPU fallback)")
    B, T, D = h.shape
    h = h.float().contiguous()
    if T <= 1:      # modeling_flexicodec_new.py:848-852: one token holding the one frame
        sim, ng = torch.ones(B, max(T - 1, 0), device=h.device), torch.ones(B, dtype=torch.long, device=h.device)
        lens = torch.ones(B, 1, dtype=torch.long, device=h.device)
        if not want_matrix:
            return torch.zeros(B, T, dtype=torch.int32, device=h.device), sim, ng, lens
        return torch.ones(B, 1, T, device=h.device), sim, ng, lens
    sim = torch.empty(B, T - 1, device=h.device)
    seg = torch.empty(B, T, dtype=torch.int32, device=h.device)
    lengths = torch.empty(B, T, dtype=torch.int32, device=h.device)
    ng = torch.empty(B, dtype=torch.int32, device=h.device)
    _lib.check(_lib.load().qb_similarity_alignment(_p(h), B, T, D, float(threshold), int(max_tokens_per_group or 0), _p(sim), _p(seg),
                                                   _p(lengths), _p(ng), _stream()))
    G = int(ng.max())                                           # the one host read the reference also does (max_segments, :905)
    lens = lengths[:, :G].long()
    if not want_matrix:
        return seg, sim, ng.long(), lens
    align = torch.empty(B, G, T, device=h.device)
    _lib.check(_lib.load().qb_alignment_matrix(_p(seg), B, T, G, _p(align), _stream()))
    return align, sim, ng.long(), lens


def inject_lengths(codes: torch.Tensor, lengths: torch.Tensor, codebook_size: int) -> torch.Tensor:
    B, nq, G = codes.shape
    codes = codes.long().contiguous()
    ln = lengths.to(torch.int32).contiguous()
    out = torch.empty_like(codes)
    _lib.check(_lib.load().qb_pack_lengths(_p(codes), _p(ln), B, nq, G, int(codebook_size), _p(out), _stream()))
    return out


def extract_lengths(codes: torch.Tensor, codebook_size: int):
    B, nq, G = codes.shape
    codes = codes.long().contiguous()
    plain = torch.empty_like(codes)
    ln = torch.empty(B, G, dtype=torch.int32, device=codes.device)
    _lib.check(_lib.load().qb_unpack_lengths(_p(codes), B, nq, G, int(codebook_size), _p(plain), _p(ln), _stream()))
    return plain, ln.long()


def deaggregate_by_lengths(grouped: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """[B,C,G] (fp32 features or int64 codes), lengths [B,G] -> [B,C,max_b sum(lengths)] zero padded"""
    B, Cc, G = grouped.shape
    if grouped.dtype not in (torch.float32, torch.int64):
        grouped = grouped.float()
    grouped = grouped.contiguous()
    ln = lengths.to(torch.int32).contiguous()
    off = torch.empty(B, G, dtype=torch.int32, device=grouped.device)
    tot = torch.empty(B, dtype=torch.int32, device=grouped.device)
    lib = _lib.load()
    _lib.check(lib.qb_length_offsets(_p(ln), B, G, _p(off), _p(tot), _stream()))
    T_out = int(tot.max())                                       # output length is data dependent (pad_sequence in the reference)
    out = torch.empty(B, Cc, T_out, dtype=grouped.dtype, device=grouped.device)
    _lib.check(lib.qb_deaggregate(_p(grouped), grouped.element_size(), _p(ln), _p(off), B, Cc, G, T_out, _p(out), _stream()))
    return out


def deaggregate(grouped: torch.Tensor, alignment: torch.Tensor) -> torch.Tensor:
    """[B,D,G] x one-hot alignment [B,G,T] -> [B,D,T]: every frame takes its token's vector (== einsum('bdg,bgt->bdt'))"""
    return deaggregate_by_lengths(grouped, alignment.sum(2).long())[..., :alignment.shape[2]]
