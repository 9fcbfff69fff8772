"""Torch-tensor front ends of the C-ABI ops.  PyTorch here is device memory + streams only: every
function hands raw device pointers to libquark_b200 on the current CUDA stream."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from ._lib import ACT_ELU, ACT_GELU, ACT_NONE, ACT_RELU, ACT_SNAKE, ACT_SWIGLU, ACT_TANH, GemmDesc, RowMap  # noqa: F401


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "libquark_b200 needs contiguous CUDA tensors"
    return C.c_void_p(t.data_ptr())


@dataclass
class Planes:
    """fp16 hi (+ optional lo) planes of a channel-last activation / weight."""
    hi: torch.Tensor
    lo: Optional[torch.Tensor] = None

    @staticmethod
    def zeros(shape, split: bool, device):
        hi = torch.zeros(shape, dtype=torch.float16, device=device)
        return Planes(hi, torch.zeros(shape, dtype=torch.float16, device=device) if split else None)

    @staticmethod
    def from_f32(x: torch.Tensor, split: bool = True):
        """Load-time helper (weights): hi = rn_fp16(x) saturated, lo = rn_fp16(x - hi)."""
        x = x.float().clamp(-65504.0, 65504.0)
        hi = x.half()
        lo = (x - hi.float()).half() if split else None
        return Planes(hi.contiguous(), lo.contiguous() if lo is not None else None)

    def float(self):
        return self.hi.float() + (self.lo.float() if self.lo is not None else 0.0)


def conv_planes(w: torch.Tensor, split: bool = True) -> Planes:
    """Conv1d weight [Cout, Cin, k] -> planes [Cout, k * pad64(Cin)], the convolution weight of qb_gemm_desc: tap-major K,
    input channels zero-padded to a multiple of 64."""
    co, ci, k = w.shape
    out = w.new_zeros(co, k, (ci + 63) // 64 * 64)
    out[:, :, :ci] = w.permute(0, 2, 1)
    return Planes.from_f32(out.reshape(co, -1), split)


def convt_planes(w: torch.Tensor, s: int, split: bool = True):
    """ConvTranspose1d weight [Cin, Cout, k], stride s -> (planes [s * Cout, J * pad64(Cin)], J = ceil(k / s)): the weight of a
    J-tap GEMM over the input zero-padded by J - 1 rows on both sides whose output row q holds all s phases of output frames
    q*s .. q*s + s - 1 of the uncropped transposed conv (a ConvTranspose1d with padding p is rows shifted by p).
    Row (r, co), GEMM tap t multiplies x[q + t - (J-1)] with w[:, co, r + (J-1-t) * s]."""
    ci, co, k = w.shape
    J = -(-k // s)
    cp = (ci + 63) // 64 * 64
    wp = w.new_zeros(ci, co, J * s)
    wp[:, :, :k] = w
    wp = wp.reshape(ci, co, J, s)                              # [ci, co, j, r]
    out = w.new_zeros(s, co, J, cp)
    out[:, :, :, :ci] = wp.permute(3, 1, 2, 0).flip(2)         # tap t <-> j = J-1-t
    return Planes.from_f32(out.reshape(s * co, J * cp), split), J


def pad_k_planes(w: torch.Tensor, kp: int, split: bool = True) -> Planes:
    """Dense weight [N, K] -> planes [N, kp], columns K..kp zero (K padded to the GEMM's multiple of 64)."""
    out = w.new_zeros(w.shape[0], kp)
    out[:, :w.shape[1]] = w
    return Planes.from_f32(out, split)


def rope_tables(T: int, D: int, device):
    """RoPE cos / sin [T, D] in the rotate-half layout: columns j and j + D/2 hold position * 10000^(-2j / D)."""
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
    fr = torch.arange(T).float()[:, None] * inv[None, :]
    emb = torch.cat((fr, fr), -1)
    return emb.cos().to(device).contiguous(), emb.sin().to(device).contiguous()


def rowmap(t: Optional[torch.Tensor], ld=0, rows_per_batch=0, row_off=0) -> RowMap:
    return RowMap(_p(t), ld, rows_per_batch, row_off)


def gemm(a: Planes, w: Planes, n: int, *, a_batch: int, a_rows_per_batch: int, a_ld: int, m_per_batch: int,
         taps: int = 1, stride: int = 1, bias=None, gamma=None, residual: Optional[RowMap] = None, act=ACT_NONE,
         act2=ACT_NONE, out_f32: Optional[RowMap] = None, out_planes: Optional[Planes] = None,
         out_planes_map=(0, 0, 0), simt: bool = False, dilation: int = 1, act_param=None, act2_param=None, a_cols: int = 0,
         a_col_off: int = 0):
    """One dense contraction (see qb_gemm_desc).  Split mode iff both a.lo and w.lo are given."""
    split = a.lo is not None and w.lo is not None
    d = GemmDesc()
    d.a_hi, d.a_lo = _p(a.hi), (_p(a.lo) if split else None)
    if a_col_off:       # grouped convolution: contract channels [a_col_off, a_col_off + a_cols) of every row
        d.a_hi = C.c_void_p(a.hi.data_ptr() + 2 * a_col_off)
        d.a_lo = C.c_void_p(a.lo.data_ptr() + 2 * a_col_off) if split else None
    d.a_cols = a_cols
    d.a_batch, d.a_rows_per_batch, d.a_ld = a_batch, a_rows_per_batch, a_ld
    d.taps, d.stride, d.m_per_batch, d.dilation = taps, stride, m_per_batch, dilation
    d.w_hi, d.w_lo, d.n = _p(w.hi), (_p(w.lo) if split else None), n
    d.bias, d.gamma = _p(bias), _p(gamma)
    d.residual = residual if residual is not None else RowMap(None, 0, 0, 0)
    d.act, d.act2 = act, act2
    d.act_param, d.act2_param = _p(act_param), _p(act2_param)
    d.out_f32 = out_f32 if out_f32 is not None else RowMap(None, 0, 0, 0)
    if out_planes is not None:
        ld, rpb, off = out_planes_map
        d.out_hi = RowMap(_p(out_planes.hi), ld, rpb, off)
        d.out_lo = RowMap(_p(out_planes.lo), ld, rpb, off) if out_planes.lo is not None else RowMap(None, 0, 0, 0)
    else:
        d.out_hi = RowMap(None, 0, 0, 0)
        d.out_lo = RowMap(None, 0, 0, 0)
    lib = _lib.load()
    _lib.check((lib.qb_gemm_simt if simt else lib.qb_gemm)(C.byref(d), _stream()))


def gemm_kernel_name(m_per_batch: int, n: int, split: bool) -> str:
    return _lib.load().qb_gemm_kernel_name(m_per_batch, n, int(split)).decode()


def split_f16(x: torch.Tensor, out: Planes):
    _lib.check(_lib.load().qb_split_f16(_p(x), _p(out.hi), _p(out.lo), x.numel(), _stream()))


def rows_to_planes(x, B, rows, Cc, out: Planes, ld, rows_per_batch, row_off, repeat=1, act=ACT_NONE):
    _lib.check(_lib.load().qb_rows_to_planes(_p(x), B, rows, Cc, repeat, act, _p(out.hi), _p(out.lo), ld,
                                             rows_per_batch, row_off, _stream()))


def bct_to_planes(x, out: Planes, ld, rows_per_batch, row_off):
    B, Cc, T = x.shape
    _lib.check(_lib.load().qb_bct_to_planes(_p(x), B, Cc, T, _p(out.hi), _p(out.lo), ld, rows_per_batch, row_off,
                                            _stream()))


def layernorm(x, w, b, B, rows, Cc, eps=1e-6, out_f32=None, out: Optional[Planes] = None, ld=0, rows_per_batch=0,
              row_off=0):
    hi = out.hi if out is not None else None
    lo = out.lo if out is not None else None
    if out is not None and ld == 0:
        ld, rows_per_batch, row_off = Cc, rows, 0
    _lib.check(_lib.load().qb_layernorm(_p(x), _p(w), _p(b), eps, B, rows, Cc, _p(out_f32), _p(hi), _p(lo), ld,
                                        rows_per_batch, row_off, _stream()))


def layernorm_act(x, w, b, B, rows, Cc, act, eps=1e-5, out_f32=None, out: Optional[Planes] = None, ld=0, rows_per_batch=0,
                  row_off=0):
    """layernorm followed by `act` (ACT_NONE / ACT_GELU)"""
    hi = out.hi if out is not None else None
    lo = out.lo if out is not None else None
    if out is not None and ld == 0:
        ld, rows_per_batch, row_off = Cc, rows, 0
    _lib.check(_lib.load().qb_layernorm_act(_p(x), _p(w), _p(b), eps, B, rows, Cc, act, _p(out_f32), _p(hi), _p(lo), ld,
                                            rows_per_batch, row_off, _stream()))


def rmsnorm(x, w, rows, Cc, out: Optional[Planes] = None, eps=1e-6, out_f32=None):
    hi = out.hi if out is not None else None
    lo = out.lo if out is not None else None
    _lib.check(_lib.load().qb_rmsnorm(_p(x), _p(w), eps, rows, Cc, _p(out_f32), _p(hi), _p(lo), _stream()))


def dwconv7_ln(x, dw_w, dw_b, ln_w, ln_b, B, T, Cc, out: Planes):
    _lib.check(_lib.load().qb_dwconv7_ln(_p(x), _p(dw_w), _p(dw_b), _p(ln_w), _p(ln_b), B, T, Cc, _p(out.hi), _p(out.lo),
                                         _stream()))


def dwconv7_adaln(x, dw_w, dw_b, scale, shift, cond_stride, B, T, Cc, out: Planes):
    _lib.check(_lib.load().qb_dwconv7_adaln(_p(x), _p(dw_w), _p(dw_b), _p(scale), _p(shift), cond_stride, B, T, Cc, _p(out.hi),
                                            _p(out.lo), _stream()))


def adalayernorm(x, scale, shift, cond_stride, B, rows, Cc, eps=1e-6, out_f32=None, out: Optional[Planes] = None, ld=0,
                 rows_per_batch=0, row_off=0):
    hi = out.hi if out is not None else None
    lo = out.lo if out is not None else None
    if out is not None and ld == 0:
        ld, rows_per_batch, row_off = Cc, rows, 0
    _lib.check(_lib.load().qb_adalayernorm(_p(x), _p(scale), _p(shift), cond_stride, eps, B, rows, Cc, _p(out_f32), _p(hi),
                                           _p(lo), ld, rows_per_batch, row_off, _stream()))


def snake_planes(x, x_batch_stride, alpha, B, T, Cc, out: Planes, ld, rows_per_batch, row_off):
    _lib.check(_lib.load().qb_snake_planes(_p(x), x_batch_stride, _p(alpha), B, T, Cc, _p(out.hi), _p(out.lo), ld,
                                           rows_per_batch, row_off, _stream()))


def elu_planes(x, x_batch_stride, B, T, Cc, out: Planes, ld, rows_per_batch, row_off):
    _lib.check(_lib.load().qb_elu_planes(_p(x), x_batch_stride, B, T, Cc, _p(out.hi), _p(out.lo), ld, rows_per_batch, row_off,
                                         _stream()))


def addvec_planes(x, vec, B, T, Cc, out: Planes, ld, rows_per_batch, row_off):
    _lib.check(_lib.load().qb_addvec_planes(_p(x), _p(vec), B, T, Cc, _p(out.hi), _p(out.lo), ld, rows_per_batch, row_off,
                                            _stream()))


def groupnorm_stats(x, B, T, Cc, stats, groups=32, eps=1e-6):
    _lib.check(_lib.load().qb_groupnorm_stats(_p(x), B, T, Cc, groups, eps, _p(stats), _stream()))


def groupnorm_apply(x, stats, w, b, B, T, Cc, swish, out_f32=None, out: Optional[Planes] = None, ld=0,
                    rows_per_batch=0, row_off=0, groups=32):
    hi = out.hi if out is not None else None
    lo = out.lo if out is not None else None
    _lib.check(_lib.load().qb_groupnorm_apply(_p(x), _p(stats), _p(w), _p(b), B, T, Cc, groups, int(swish), _p(out_f32),
                                              _p(hi), _p(lo), ld, rows_per_batch, row_off, _stream()))


def stft_gather(wav, hop, n_fft, P, Q, window, out: Planes):
    B, T = wav.shape
    _lib.check(_lib.load().qb_stft_gather(_p(wav), B, T, hop, n_fft, P, Q, _p(window), _p(out.hi), _p(out.lo), _stream()))


def stft_twiddle(Y, ldY, frames_total, P, Q, twiddle, out: Planes):
    _lib.check(_lib.load().qb_stft_twiddle(_p(Y), ldY, frames_total, P, Q, _p(twiddle), _p(out.hi), _p(out.lo), _stream()))


def stft_post2(X, ldX, B, frames, nf, P, out: Planes, ld, rows_per_batch, row_off):
    _lib.check(_lib.load().qb_stft_post2(_p(X), ldX, B, frames, nf, P, _p(out.hi), _p(out.lo), ld, rows_per_batch, row_off, _stream()))


def istft_pre(head, ld_in, M, nf, out: Planes, ld):
    _lib.check(_lib.load().qb_istft_pre(_p(head), ld_in, M, nf, _p(out.hi), _p(out.lo), ld, _stream()))


def istft_ola(frames, window, B, F, n_fft, wav, hop=None):
    _lib.check(_lib.load().qb_istft_ola(_p(frames), _p(window), B, F, n_fft, hop if hop is not None else n_fft // 2, _p(wav),
                                        _stream()))


def reflect_pad_rows(buf: Planes, B, rows_per_batch, ld, T, row_off, pad_l, pad_r):
    _lib.check(_lib.load().qb_reflect_pad_rows(_p(buf.hi), _p(buf.lo), B, rows_per_batch, ld, T, row_off, pad_l, pad_r,
                                               _stream()))


def dwconv(x, w, bias, B, T, Cc, k, out):
    _lib.check(_lib.load().qb_dwconv(_p(x), _p(w), _p(bias), B, T, Cc, k, _p(out), _stream()))


def attention_hd(qkv, B, T, heads, head_dim, rope_cos, rope_sin, out: Planes):
    _lib.check(_lib.load().qb_attention_hd(_p(qkv), B, T, heads, head_dim, _p(rope_cos), _p(rope_sin), _p(out.hi), _p(out.lo),
                                           _stream()))


def attention_umma_workspace_bytes(B, L, heads, head_dim, split):
    return int(_lib.load().qb_attention_umma_workspace_bytes(B, L, heads, head_dim, int(bool(split))))


def attention_umma(qkv, B, L, heads, head_dim, rope_cos, rope_sin, out: Planes, workspace, split=None, causal=False):
    """wgmma attention (head_dim 64 / 128); split defaults to whether `out` carries a lo plane"""
    split = (out.lo is not None) if split is None else split
    _lib.check(_lib.load().qb_attention_umma(_p(qkv), B, L, heads, head_dim, _p(rope_cos), _p(rope_sin), _p(out.hi), _p(out.lo),
                                             int(bool(split)), int(bool(causal)), _p(workspace), _stream()))


def self_attention_workspace_bytes(B, L, heads, head_dim, split):
    """workspace of `self_attention`: the wgmma kernel's operand planes at head_dim 64 / 128, nothing for the SIMT kernel"""
    return attention_umma_workspace_bytes(B, L, heads, head_dim, split) if head_dim in (64, 128) else 0


def self_attention(qkv, B, L, heads, head_dim, rope_cos, rope_sin, out: Planes, workspace, split):
    """Non-causal self-attention with RoPE: the wgmma kernel at head_dim 64 / 128 (split: fp16 hi + lo operands), the fp32 SIMT
    kernel at any other head_dim.  The kernels are looked up in this module at each call, so a wrapper assigned to
    `ops.attention_umma` / `ops.attention_hd` (bench.py counts attention FLOPs that way) sees every call."""
    if head_dim in (64, 128):
        attention_umma(qkv, B, L, heads, head_dim, rope_cos, rope_sin, out, workspace, split=split)
    else:
        attention_hd(qkv, B, L, heads, head_dim, rope_cos, rope_sin, out)


# bench.py's H-Codec-1.5 FLOP counter wraps this name; it is the single-pass wgmma attention at head_dim 64, and no model calls it
def attention_tc_workspace_bytes(B, T, heads):
    return attention_umma_workspace_bytes(B, T, heads, 64, False)


def attention_tc(qkv, B, T, heads, rope_cos, rope_sin, out: Planes, workspace):
    attention_umma(qkv, B, T, heads, 64, rope_cos, rope_sin, out, workspace, split=False)


def lstm_tc_units(H):
    return int(_lib.load().qb_lstm_tc_units(H))


def lstm_tc_workspace_bytes(B, H):
    return int(_lib.load().qb_lstm_tc_workspace_bytes(B, H))


def lstm_tc_permute(whh: torch.Tensor, U: int) -> torch.Tensor:
    """[4H,H] (gate-major i|f|g|o) -> fp16 [H/U][4U][H], row 4j+g of slice c = gate g of unit c*U+j."""
    H = whh.shape[1]
    rows = (torch.arange(4, device=whh.device)[None, None, :] * H +
            torch.arange(H, device=whh.device).reshape(H // U, U)[:, :, None]).reshape(-1)
    return whh.float().clamp(-65504.0, 65504.0)[rows].half().contiguous()


def lstm_tc(xp, whh_perm, U, B, T, H, out: Planes, workspace):
    _lib.check(_lib.load().qb_lstm_tc(_p(xp), _p(whh_perm), U, B, T, H, _p(out.hi), _p(out.lo), _p(workspace), _stream()))


def rvq_workspace_bytes(M, D, K):
    return int(_lib.load().qb_rvq_workspace_bytes(M, D, K))


def rvq_encode(x, codebooks, cb: Planes, neg_half_e2, e2max, M, D, K, nq, idx, quantized, workspace):
    _lib.check(_lib.load().qb_rvq_encode(_p(x), _p(codebooks), _p(cb.hi), _p(cb.lo), _p(neg_half_e2), float(e2max), M, D,
                                         K, nq, _p(idx), _p(quantized), _p(workspace), _stream()))


def rvq_decode(idx, codebooks, M, D, K, nq, out, out_ld, col_off):
    _lib.check(_lib.load().qb_rvq_decode(_p(idx), _p(codebooks), M, D, K, nq, _p(out), out_ld, col_off, _stream()))


def fvq_tokenize(z, M, D_in, w_in, b_in, codebook_n, K, cdim, idx, z_e=None):
    """z [M, D_in] fp32 -> idx [M] int64 (+ z_e [M, cdim] fp32); codebook_n is the fp64 normalised codebook [K, cdim]"""
    assert codebook_n.dtype == torch.float64 and idx.dtype == torch.int64
    _lib.check(_lib.load().qb_fvq_tokenize(_p(z), M, D_in, _p(w_in), _p(b_in), _p(codebook_n), K, cdim, _p(idx), _p(z_e), _stream()))


def fvq_usage(idx, K, counts, perplexity, active):
    """idx int64 [n] -> perplexity and active-code count (0-d fp32 device tensors); counts: int32 [K] scratch"""
    _lib.check(_lib.load().qb_fvq_usage(_p(idx), idx.numel(), K, _p(counts), _p(perplexity), _p(active), _stream()))


def lm_qkv_prep(qkv, B, L, heads, pos0, cos, sin, q16, kc, vc, Lmax):
    _lib.check(_lib.load().qb_lm_qkv_prep(_p(qkv), B, L, heads, pos0, _p(cos), _p(sin), _p(q16), _p(kc), _p(vc), Lmax,
                                          _stream()))


def lm_flash_attn(q16, kc, vc, B, L, heads, pos0, Lmax, out: Planes):
    _lib.check(_lib.load().qb_lm_flash_attn(_p(q16), _p(kc), _p(vc), B, L, heads, pos0, Lmax, _p(out.hi), _p(out.lo),
                                            _stream()))


def lm_pack_weight(w: torch.Tensor) -> torch.Tensor:
    """fp32 [n,k] -> fp16 [n,2k] groups of {hi[4], lo[4]} (decode B-fragment layout, include/quark_b200.h)."""
    w = w.float().contiguous()
    n, k = w.shape
    out = torch.empty(n, 2 * k, dtype=torch.float16, device=w.device)
    _lib.check(_lib.load().qb_lm_pack_weight(_p(w), n, k, _p(out), _stream()))
    return out


def lm_set_att_unroll(keys_per_lane: int):
    _lib.check(_lib.load().qb_lm_set_att_unroll(int(keys_per_lane)))


def _check_pos(pos, B):
    """the decode step reads (and the head bumps) one position per row: pos[b]"""
    if pos.dtype != torch.int32 or pos.numel() < B or not pos.is_contiguous():
        raise ValueError(f"per-row positions must be a contiguous int32 tensor of >= {B} elements, got {pos.dtype} {tuple(pos.shape)}")


def lm_decode_layer_tc(x, B, hidden, heads, inter, L, kc, vc, Lmax, pos, cos, sin, q_buf, attn_buf, mlp_buf):
    _check_pos(pos, B)
    _lib.check(_lib.load().qb_lm_decode_layer_tc(_p(x), B, hidden, heads, inter, _p(L["wqkv_p"]), _p(L["wo_p"]), _p(L["wg_p"]),
                                                 _p(L["wu_p"]), _p(L["wd_p"]), _p(kc), _p(vc), Lmax, _p(pos), _p(cos), _p(sin),
                                                 _p(q_buf), _p(attn_buf), _p(mlp_buf), _stream()))


def lm_head_argmax_tc(x, B, hidden, w_head_p, rng, max_cols, emb, x_next, out_ids, out_stride, pos, slot, pv, pi):
    _check_pos(pos, B)
    _lib.check(_lib.load().qb_lm_head_argmax_tc(_p(x), B, hidden, _p(w_head_p), _p(rng), max_cols, _p(emb), _p(x_next),
                                                _p(out_ids), out_stride, _p(pos), _p(slot), _p(pv), _p(pi), _stream()))


def lm_head_sample_tc(x, B, hidden, w_head_p, rng, max_cols, emb, x_next, out_ids, out_stride, pos, slot, pv, pi, logits,
                      temperature, top_k, top_p, seed, debug=None):
    _check_pos(pos, B)
    _lib.check(_lib.load().qb_lm_head_sample_tc(_p(x), B, hidden, _p(w_head_p), _p(rng), max_cols, _p(emb), _p(x_next),
                                                _p(out_ids), out_stride, _p(pos), _p(slot), _p(pv), _p(pi), _p(logits),
                                                float(temperature), int(top_k), float(top_p), _p(seed), _p(debug), _stream()))


def lm_head_sample_rows_tc(x, B, hidden, w_head_p, rng, max_cols, emb, x_next, out_ids, out_stride, pos, slot, pv, pi, logits,
                           temperature, top_k, top_p, row_keys, debug=None):
    """lm_head_sample_tc with one random stream per row: row_keys = contiguous int32 [>= B, 2] device tensor, {lo, hi} 32-bit
    words of row b's 64-bit key (row_keys_words)"""
    _check_pos(pos, B)
    if row_keys.dtype != torch.int32 or row_keys.numel() < 2 * B or not row_keys.is_contiguous():
        raise ValueError(f"row_keys must be a contiguous int32 tensor of >= {2 * B} elements, got {row_keys.dtype} {tuple(row_keys.shape)}")
    _lib.check(_lib.load().qb_lm_head_sample_rows_tc(_p(x), B, hidden, _p(w_head_p), _p(rng), max_cols, _p(emb), _p(x_next),
                                                     _p(out_ids), out_stride, _p(pos), _p(slot), _p(pv), _p(pi), _p(logits),
                                                     float(temperature), int(top_k), float(top_p), _p(row_keys), _p(debug), _stream()))


def row_keys_words(keys) -> torch.Tensor:
    """64-bit row keys (Python ints, any sign: taken mod 2^64) -> host int32 [n, 2] = {low word, high word} per key, the layout
    qb_lm_head_sample_rows_tc reads"""
    to_i32 = lambda v: v - (1 << 32) if v >= (1 << 31) else v
    words = [(to_i32(k & 0xFFFFFFFF), to_i32((k >> 32) & 0xFFFFFFFF)) for k in (int(k) & 0xFFFFFFFFFFFFFFFF for k in keys)]
    return torch.tensor(words, dtype=torch.int32).reshape(-1, 2)


def ssl_conv0_gn_gelu(x, w, gn_w, gn_b, eps, k, stride, out: Planes, ld, rows_per_batch, row_off, y_scratch, workspace):
    B, T_in = x.shape
    _lib.check(_lib.load().qb_ssl_conv0_gn_gelu(_p(x), B, T_in, _p(w), w.shape[0], k, stride, _p(gn_w), _p(gn_b), float(eps), _p(y_scratch),
                                                _p(workspace), _p(out.hi), _p(out.lo), ld, rows_per_batch, row_off, _stream()))


def ssl_conv0_workspace_bytes(B, T0, Cc):
    return int(_lib.load().qb_ssl_conv0_workspace_bytes(B, T0, Cc))


def ssl_conv0_bias(x, w, bias, k, stride, y):
    """x [B, T_in] -> y [B, T0, C] = Conv1d(1, C, k, stride)(x) + bias, channel-last"""
    B, T_in = x.shape
    _lib.check(_lib.load().qb_ssl_conv0_bias(_p(x), B, T_in, _p(w), _p(bias), w.shape[0], k, stride, _p(y), _stream()))


def wav_normalize(x, eps, out):
    """per row: (x - mean) / sqrt(var + eps) (Wav2Vec2FeatureExtractor, do_normalize=True)"""
    B, T = x.shape
    _lib.check(_lib.load().qb_wav_normalize(_p(x), B, T, float(eps), _p(out), _stream()))


def wavlm_gate(x, B, T, heads, head_dim, w, bias, cst, gate):
    _lib.check(_lib.load().qb_wavlm_gate(_p(x), B, T, heads, head_dim, _p(w), _p(bias), _p(cst), _p(gate), _stream()))


def attention_relbias(qkv, B, T, heads, head_dim, rel_table, gate, out: Planes):
    _lib.check(_lib.load().qb_attention_relbias(_p(qkv), B, T, heads, head_dim, _p(rel_table), _p(gate), _p(out.hi), _p(out.lo), _stream()))


def axpy(x, scale, out, accumulate=True):
    _lib.check(_lib.load().qb_axpy(_p(x), float(scale), x.numel(), int(accumulate), _p(out), _stream()))


def ssl_compress(x, B, T, Cc, power, channel_first, out):
    _lib.check(_lib.load().qb_ssl_compress(_p(x), B, T, Cc, float(power), int(channel_first), _p(out), _stream()))


def pad_wav(x, left, T_out, wrap=False):
    """[B, T] fp32 -> [B, T_out]: out[b, i] = x[b, i - left], zero (or wrapped) outside"""
    x = x.float().contiguous()
    B, T = x.shape
    out = torch.empty(B, T_out, device=x.device)
    _lib.check(_lib.load().qb_pad_wav(_p(x), B, T, left, T_out, int(wrap), _p(out), _stream()))
    return out


def mel_gather(wav, hop, n_fft, P, Q, window, out: Planes):
    B, L = wav.shape
    _lib.check(_lib.load().qb_mel_gather(_p(wav), B, L, hop, n_fft, P, Q, _p(window), _p(out.hi), _p(out.lo), _stream()))


def spec_magnitude(X, ldX, M, nf, P, out: Planes, ld):
    _lib.check(_lib.load().qb_spec_magnitude(_p(X), ldX, M, nf, P, _p(out.hi), _p(out.lo), ld, _stream()))


def add_planes(x, ldx, y, ldy, B, T, Cc, out: Planes, ld, rows_per_batch, row_off):
    """x (+ y) over Cc channels of rows with pitches ldx / ldy -> planes of a padded buffer (y may be None)"""
    _lib.check(_lib.load().qb_add_planes(_p(x), ldx, _p(y), ldy, B, T, Cc, _p(out.hi), _p(out.lo), ld, rows_per_batch, row_off,
                                         _stream()))


def se_gate(z, B, T, Cc, w1, b1, w2, b2, s):
    _lib.check(_lib.load().qb_se_gate(_p(z), B, T, Cc, _p(w1), _p(b1), w1.shape[0], _p(w2), _p(b2), _p(s), _stream()))


def se_apply(z, s, x, B, T, Cc, out=None, planes: Optional[Planes] = None, ld=0, col_off=0):
    hi = planes.hi if planes is not None else None
    lo = planes.lo if planes is not None else None
    _lib.check(_lib.load().qb_se_apply(_p(z), _p(s), _p(x), B, T, Cc, _p(out), _p(hi), _p(lo), ld, col_off, _stream()))


def geglu_planes(h, rows, inner, out: Planes, ld):
    """h [rows, 2 * inner] (value | gate) -> planes [rows, ld] = gelu(gate) * value"""
    _lib.check(_lib.load().qb_geglu_planes(_p(h), rows, inner, _p(out.hi), _p(out.lo), ld, _stream()))


def cross_attention(q, kv, B, Nq, Nk, heads, out: Planes):
    _lib.check(_lib.load().qb_cross_attention(_p(q), _p(kv), B, Nq, Nk, heads, _p(out.hi), _p(out.lo), _stream()))


def fsq_tokenize(x, rows, dim, gamma, w_in, b_in, levels, num_quantizers, idx, z=None, xn=None):
    lv = (C.c_int32 * len(levels))(*levels)
    _lib.check(_lib.load().qb_fsq_tokenize(_p(x), rows, dim, _p(gamma), _p(w_in), _p(b_in), len(levels), lv, num_quantizers, _p(idx),
                                           _p(z), _p(xn), _stream()))


def asp_context(x, B, T, Cc, out, planes: Planes, ld):
    """latent [B*T, Cc] -> [mean | unbiased std + 1e-7] fp32 [B, 2 Cc] and planes [B, ld]"""
    _lib.check(_lib.load().qb_asp_context(_p(x), B, T, Cc, _p(out), _p(planes.hi), _p(planes.lo), ld, _stream()))


def asp_tanh_planes(h, row, B, T, N, out: Planes, ld):
    """tanh(h [B*T, N] + row [B, N] per clip) -> planes [B*T, ld]"""
    _lib.check(_lib.load().qb_asp_tanh_planes(_p(h), _p(row), B, T, N, _p(out.hi), _p(out.lo), ld, _stream()))


def asp_pool(x, logits, B, T, Cc, out, planes: Planes, ld):
    """softmax-over-T attentive [mean | std] of x [B*T, Cc] -> fp32 [B, 2 Cc] and planes [B, ld]"""
    _lib.check(_lib.load().qb_asp_pool(_p(x), _p(logits), B, T, Cc, _p(out), _p(planes.hi), _p(planes.lo), ld, _stream()))


def lm_loss(logits, ld, M, V, targets, label_smoothing):
    """-> float32 [2] = {label-smoothed KL (batchmean), arg-max accuracy}"""
    ws = torch.empty(2 * M, device=logits.device)
    out = torch.empty(2, device=logits.device)
    _lib.check(_lib.load().qb_lm_loss(_p(logits), ld, M, V, _p(targets), float(label_smoothing), _p(ws), _p(out), _stream()))
    return out


# ------------------------------------------------------------------ training (csrc/lm_train.cu): gradients of the LM's loss
def _seed64(seed: int) -> int:
    return int(seed) & 0xFFFFFFFFFFFFFFFF


def lm_attn_train_fwd(qkv, B, L, heads, cos, sin, dropout_p, seed, layer, qs, kr, v, out, lse):
    _lib.check(_lib.load().qb_lm_attn_train_fwd(_p(qkv), B, L, heads, _p(cos), _p(sin), float(dropout_p), _seed64(seed), int(layer),
                                                _p(qs), _p(kr), _p(v), _p(out), _p(lse), _stream()))


def lm_attn_train_bwd(qs, kr, v, out, dout, lse, B, L, heads, cos, sin, dropout_p, seed, layer, dqkv, workspace):
    _lib.check(_lib.load().qb_lm_attn_train_bwd(_p(qs), _p(kr), _p(v), _p(out), _p(dout), _p(lse), B, L, heads, _p(cos), _p(sin),
                                                float(dropout_p), _seed64(seed), int(layer), _p(dqkv), _p(workspace), _stream()))


def lm_loss_scale(V: int) -> float:
    """qb_lm_loss_bwd's output scale: the power of two >= V, at most 2^14"""
    return float(2 ** min(14, (V - 1).bit_length()))


def lm_loss_bwd(logits, ld, M, V, targets, label_smoothing, grad_loss, out, planes: Planes, ld_out, scale):
    _lib.check(_lib.load().qb_lm_loss_bwd(_p(logits), ld, M, V, _p(targets), float(label_smoothing), _p(grad_loss), float(scale), _p(out),
                                          _p(planes.hi), _p(planes.lo), ld_out, _stream()))


def rmsnorm_bwd(x, w, dy, rows, Cc, dx, gw, accumulate, eps=1e-6):
    _lib.check(_lib.load().qb_rmsnorm_bwd(_p(x), _p(w), _p(dy), eps, rows, Cc, _p(dx), int(accumulate), _p(gw), _stream()))


def col_sum(x, rows, Cc, ld, out, accumulate=False, scale=1.0):
    """out[c] (+)= scale * sum_r x[r * ld + c], rows in order, fp64 partials"""
    ws = torch.empty(int(_lib.load().qb_col_sum_workspace_bytes(rows, Cc)), dtype=torch.uint8, device=x.device)
    _lib.check(_lib.load().qb_col_sum(_p(x), rows, Cc, ld, float(scale), _p(ws), _p(out), int(accumulate), _stream()))


def swiglu(gu, M, inter, h, planes: Planes):
    _lib.check(_lib.load().qb_swiglu(_p(gu), M, inter, _p(h), _p(planes.hi), _p(planes.lo), _stream()))


def swiglu_bwd(gu, dh, M, inter, dgu, planes: Planes):
    _lib.check(_lib.load().qb_swiglu_bwd(_p(gu), _p(dh), M, inter, _p(dgu), _p(planes.hi), _p(planes.lo), _stream()))


def transpose_split(x, rows, cols, ks, ldx=None) -> Planes:
    """x [rows, cols] fp32 -> planes [S, cols, ks] (S = ceil(rows / ks)): slice s holds rows s*ks .. s*ks + ks - 1 transposed"""
    S = -(-rows // ks)
    out = Planes(torch.empty(S, cols, ks, dtype=torch.float16, device=x.device), torch.empty(S, cols, ks, dtype=torch.float16, device=x.device))
    _lib.check(_lib.load().qb_transpose_split(_p(x), rows, cols, cols if ldx is None else ldx, ks, _p(out.hi), _p(out.lo), _stream()))
    return out


def embedding_bwd(dx, ids, n, Lt, L, P, H, V, out, accumulate=False, scale=1.0):
    _lib.check(_lib.load().qb_embedding_bwd(_p(dx), _p(ids), n, Lt, L, P, H, V, float(scale), _p(out), int(accumulate), _stream()))


def grad_slice(tokens: int, n_out: int, n_in: int, sms: int = 132) -> int:
    """Tokens per split-K slice of a weight gradient [n_out, n_in] contracted over `tokens`: enough slices that the persistent GEMM's
    128 x 128-ish tiles fill every SM about twice, no slice shorter than 512 tokens (a multiple of 64)."""
    tiles = -(-n_out // 128) * -(-n_in // 128)
    slices = max(1, min(-(-2 * sms // tiles), -(-tokens // 512)))
    per_slice = -(-tokens // slices)
    return -(-per_slice // 64) * 64


def weight_grad(dy, x, tokens, n_out, n_in, out, ks=None, dy_ld=None, scale=1.0):
    """out [n_out, n_in] = scale * dy^T x over `tokens` rows (dy [tokens, n_out] with row pitch dy_ld, x [tokens, n_in] fp32): the transposed
    operands cut into slices of ks tokens, one 3-term-split qb_gemm per slice into fp32 partials, the partials summed in slice order
    in fp64."""
    ks = grad_slice(tokens, n_out, n_in) if ks is None else ks
    a, w = transpose_split(dy, tokens, n_out, ks, dy_ld), transpose_split(x, tokens, n_in, ks)
    S = a.hi.shape[0]
    part = torch.empty(S, n_out, n_in, device=dy.device)
    for s in range(S):
        gemm(Planes(a.hi[s], a.lo[s]), Planes(w.hi[s], w.lo[s]), n_in, a_batch=1, a_rows_per_batch=n_out, a_ld=ks, m_per_batch=n_out,
             out_f32=rowmap(part[s], n_in, n_out, 0))
    col_sum(part, S, n_out * n_in, n_out * n_in, out, scale=scale)
    return out


def launch_count() -> int:
    return int(_lib.load().qb_launch_count())


def launch_count_reset():
    _lib.load().qb_launch_count_reset()


# ------------------------------------------------------------------ training-data simulation (csrc/simulate.cu), packed ragged rows
def sim_active_rms(x, offs, frame_off, rows, max_len, max_frames, rms, mask=None):
    """rms [rows] fp64 = std of each row over its non-silent samples (mask: the uint8 flags, packed as x, or None)"""
    power = torch.empty(max(1, rows * max(1, max_frames)), dtype=torch.float64, device=x.device)
    _lib.check(_lib.load().qb_sim_active_rms(_p(x), _p(offs), _p(frame_off), rows, max_len, max_frames, _p(power), _p(rms), _p(mask),
                                             _stream()))


def sim_place(src, src_offs, offs, shift, rows, max_len, dst):
    _lib.check(_lib.load().qb_sim_place(_p(src), _p(src_offs), _p(offs), _p(shift), rows, max_len, _p(dst), _stream()))


def sim_mix(x, other, offs, rows, max_len, snr, rms_x, rms_other, on, diff=None):
    _lib.check(_lib.load().qb_sim_mix(_p(x), _p(other), _p(offs), rows, max_len, _p(snr), _p(rms_x), _p(rms_other), _p(on), _p(diff),
                                      _stream()))


def sim_rir_prep(h, offs, rows, on, hn, win, status):
    _lib.check(_lib.load().qb_sim_rir_prep(_p(h), _p(offs), rows, _p(on), _p(hn), _p(win), _p(status), _stream()))


def sim_convolve(x, offs, rows, max_len, h, h_offs, win, on, y):
    _lib.check(_lib.load().qb_sim_convolve(_p(x), _p(offs), rows, max_len, _p(h), _p(h_offs), _p(win), _p(on), _p(y), _stream()))


def sim_bandwidth(x, offs, rows, max_len, fs_new, on, taps, tmp):
    """taps: {'down4', 'down2', 'kd4', 'wd4', 'kd2', 'wd2', 'up4', 'up2', 'ku', 'wu'} (Simulator._taps)"""
    t = taps
    _lib.check(_lib.load().qb_sim_bandwidth(_p(x), _p(offs), rows, max_len, _p(fs_new), _p(on), _p(t["down4"]), _p(t["down2"]), t["kd4"],
                                            t["wd4"], t["kd2"], t["wd2"], _p(t["up4"]), _p(t["up2"]), t["ku"], t["wu"], _p(tmp), _stream()))


def sim_clip(x, offs, rows, max_len, q, on, stats):
    _lib.check(_lib.load().qb_sim_clip(_p(x), _p(offs), rows, max_len, _p(q), _p(on), _p(stats), _stream()))


def sim_packet_loss(x, offs, lost, lost_row, packet):
    _lib.check(_lib.load().qb_sim_packet_loss(_p(x), _p(offs), _p(lost), _p(lost_row), lost.numel(), packet, _stream()))


def sim_finish(noisy, speech, interf, offs, rows, has_interf, cut_off, norm_r, cut, out_mix, out_speech, out_interf=None):
    _lib.check(_lib.load().qb_sim_finish(_p(noisy), _p(speech), _p(interf), _p(offs), rows, _p(has_interf), _p(cut_off), _p(norm_r), cut,
                                         _p(out_mix), _p(out_speech), _p(out_interf), _stream()))


def sim_enroll(e, offs, rows, cut_off, cut, out):
    _lib.check(_lib.load().qb_sim_enroll(_p(e), _p(offs), rows, _p(cut_off), cut, _p(out), _stream()))
