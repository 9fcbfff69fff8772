/*
 * libquark_b200 - C ABI of the H100-native QuarkAudio audio-token hot path.
 *
 * The reference (alibaba/unified-audio) is pure Python/PyTorch and has no FFI layer; its boundary
 * for this path is the nn.Module method surface (SURVEY.md 8b).  The entry points below are what a
 * Python binding (ctypes; see INTEGRATION.md) calls from drop-in replacements of
 *   Codec.encode / Codec.decode            QuarkAudio-HCodec/HCodec-2.0/vq/codec.py:75-99
 *   ResidualVQ.__call__ / get_output_from_indices (third-party; call sites codec.py:81-82,94-95)
 *   CustomLlamaModel.llm_forward / LLM_SFT.generate   QuarkAudio-UniSE/model/llm/llm.py:150-228,
 *                                                     llm_sft.py:93-195
 * Each op cites the reference lines whose arithmetic it replaces.
 *
 * Conventions: every pointer is a DEVICE pointer owned by the caller (row-major, contiguous,
 * 16-byte aligned) unless stated otherwise; every call is asynchronous on `stream`
 * (a cudaStream_t passed as void*); return 0 on success, negative on error
 * (qb_last_error() gives the message; no C++ exception crosses the ABI); no hidden host syncs.
 *
 * Activations are channel-last: a tensor [B, T, C] is B*T rows of C contiguous channels.  Dense
 * contractions take their operands as fp16 "planes": `hi` = rn_fp16(x) and optionally
 * `lo` = rn_fp16(x - hi).  With both planes of both operands present the GEMM issues
 * hi*hi + lo*hi + hi*lo on the tensor cores (fp32 accumulate): ~2^-21 relative operand precision.
 * With `lo` absent it is a single-pass fp16 GEMM (2^-11).  DESIGN.md "precision policy".
 */
#ifndef QUARK_B200_H_
#define QUARK_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint16_t qb_half; /* IEEE fp16 bit pattern */

/* ------------------------------------------------------------------------------------------ */
const char* qb_last_error(void);
int qb_version(void);
/* Number of kernels this library has launched since load / since the last reset (host counter). */
int64_t qb_launch_count(void);
void qb_launch_count_reset(void);

/* activation codes for the GEMM epilogue */
enum { QB_ACT_NONE = 0, QB_ACT_GELU = 1, QB_ACT_SWIGLU = 2, QB_ACT_ELU = 3, QB_ACT_TANH = 4, QB_ACT_SNAKE = 5, QB_ACT_RELU = 6 };

/* Row mapping of an output / residual tensor: GEMM row (batch b, row m) lives at
 * ptr + ((b * rows_per_batch + row_off + m) * ld + n).  Lets a GEMM write straight into the
 * interior of the next convolution's zero-padded channel-last buffer. */
typedef struct {
  void* ptr;
  int64_t ld;
  int64_t rows_per_batch;
  int64_t row_off;
} qb_rowmap;

/*
 * One dense contraction  D[b, m, n] = sum_{tap, c} A[b, m*stride + tap*dilation, c] * W[n, tap*a_ld + c]
 * i.e. nn.Linear (taps = stride = 1), a strided / dilated nn.Conv1d over a zero-padded channel-last buffer, or a
 * ConvTranspose1d (stride s, kernel k) as ceil(k/s) taps producing all s output phases as s*Cout columns
 * (bicodec/modules/encoder_decoder/wave_generator.py:42-48; weights repacked per phase at load)
 * (vq/conv.py:35-57, vq/semantic_module.py:13-52; weights repacked [Cout, k*Cin_pad] at load).
 * Epilogue:  v = acc + bias[n];  v = act(v);  v *= gamma[n];  v += residual[b,m,n];
 *            out_f32 <- v;   out planes <- split_fp16(act2(v))
 * QB_ACT_SWIGLU pairs columns (2j, 2j+1) -> silu(v[2j]) * v[2j+1] at output column j
 * (encoder_modules/transformer.py:218-226 with w1/w3 rows interleaved).
 * QB_ACT_RELU with gamma and a broadcast residual row (residual.ld = rows_per_batch = 0, row_off = 0: address ptr + n) is an
 * eval-mode conv -> ReLU -> BatchNorm1d (ecapa_tdnn.py:90-109): gamma = w / sqrt(var + eps), residual = b - mean * gamma.
 */
typedef struct {
  const qb_half* a_hi;      /* [a_batch, a_rows_per_batch, a_ld] */
  const qb_half* a_lo;      /* NULL => single-pass */
  int64_t a_batch;
  int64_t a_rows_per_batch; /* rows of the (padded) A buffer per batch; multiple of stride */
  int64_t a_ld;             /* channels per row (multiple of 64) */
  int32_t taps;
  int32_t stride;
  int64_t m_per_batch;      /* output rows per batch */
  const qb_half* w_hi;      /* [n, taps * a_ld] */
  const qb_half* w_lo;      /* NULL => single-pass */
  int64_t n;
  const float* bias;        /* [n] or NULL */
  const float* gamma;       /* [n] or NULL */
  qb_rowmap residual;       /* fp32, ptr NULL => none */
  int32_t act;              /* QB_ACT_* applied to v before gamma/residual */
  int32_t act2;             /* QB_ACT_NONE, QB_ACT_ELU or QB_ACT_SNAKE, applied only to the fp16-plane output */
  qb_rowmap out_f32;        /* ptr NULL => not written */
  qb_rowmap out_hi;         /* fp16 planes; ptr NULL => not written */
  qb_rowmap out_lo;         /* ptr NULL => hi only (same ld / mapping fields as out_hi required) */
  int32_t dilation;         /* tap spacing in input rows: A[b, m*stride + tap*dilation, c]; 0 or 1 = dense taps.
                             * (DAC residual units, bicodec/modules/blocks/layers.py:52-60: k=7, dilation 1/3/9) */
  const float* act_param;   /* [n] per-column parameter of `act`  (QB_ACT_SNAKE: alpha) or NULL */
  const float* act2_param;  /* [n] per-column parameter of `act2` (QB_ACT_SNAKE on the plane output only: the fp32 output is
                             * the residual trunk, the planes are Snake(trunk) for the next convolution) or NULL */
  int64_t a_cols;           /* channels contracted per tap (multiple of 64, <= a_ld); 0 = a_ld.  With a_hi / a_lo offset to a
                             * channel group this is a GROUPED convolution over a [.., a_ld] buffer: W is [n, taps * a_cols]
                             * (HuBERT / WavLM positional conv: k = 128, 16 groups, transformers modeling_hubert.py) */
} qb_gemm_desc;

/* wgmma / TMA persistent GEMM (the product path). */
int qb_gemm(const qb_gemm_desc* d, void* stream);
/* Name of the kernel variant qb_gemm runs for this shape (m_per_batch output rows per batch, n columns, split != 0 for the
 * 3-term mode) - static string, used by bench.py's roofline label. */
const char* qb_gemm_kernel_name(int64_t m_per_batch, int64_t n, int32_t split);
/* Plain SIMT evaluation of the same descriptor - a device-side cross-check used by tests only. */
int qb_gemm_simt(const qb_gemm_desc* d, void* stream);

/* ---------------------------------------------------------------- elementwise / normalisation */
/* x[n] fp32 -> hi/lo planes (lo may be NULL). */
int qb_split_f16(const float* x, qb_half* hi, qb_half* lo, int64_t n, void* stream);
/* Copy rows [B, rows, C] fp32 (channel-last) into planes of a padded buffer
 * [B, rows_per_batch, ld] at row offset row_off; channels C..ld-1 are zeroed; `repeat` repeats each
 * source row `repeat` times (repeat_interleave, vq/codec_decoder.py:64); act: QB_ACT_NONE / QB_ACT_ELU. */
int qb_rows_to_planes(const float* x, int64_t B, int64_t rows, int64_t C, int32_t repeat, int32_t act,
                      qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream);
/* Channel-first [B, C, T] fp32 -> channel-last planes in a padded buffer (semantic features in). */
int qb_bct_to_planes(const float* x, int64_t B, int64_t C, int64_t T, qb_half* hi, qb_half* lo, int64_t ld,
                     int64_t rows_per_batch, int64_t row_off, void* stream);
/* LayerNorm over C (eps) of fp32 rows; writes fp32 and/or planes (any may be NULL).
 * vq/codec_encoder.py:74,77; vq/codec_decoder.py:67,70 */
int qb_layernorm(const float* x, const float* w, const float* b, float eps, int64_t B, int64_t rows, int64_t C,
                 float* out_f32, qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off,
                 void* stream);
/* qb_layernorm followed by an activation (QB_ACT_NONE or QB_ACT_GELU, exact erf): wav2vec2's conv layers with
 * feat_extract_norm="layer" (conv -> LayerNorm over channels -> GELU). */
int qb_layernorm_act(const float* x, const float* w, const float* b, float eps, int64_t B, int64_t rows, int64_t C, int32_t act,
                     float* out_f32, qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream);
/* RMSNorm (encoder_modules/transformer.py:77-96; HF LlamaRMSNorm) -> fp32 and/or planes (any may be NULL). */
int qb_rmsnorm(const float* x, const float* w, float eps, int64_t rows, int64_t C, float* out_f32, qb_half* hi,
               qb_half* lo, void* stream);
/* ConvNeXt front half: depthwise conv k=7 (zero pad 3) over time + LayerNorm(1e-6) -> planes
 * (vq/conv.py:201-204).  x [B, T, C] fp32; dw_w [C,7]; dw_b [C]. */
int qb_dwconv7_ln(const float* x, const float* dw_w, const float* dw_b, const float* ln_w, const float* ln_b,
                  int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo, void* stream);
/* AdaLayerNorm variants (bicodec/modules/blocks/vocos.py:88-111): LayerNorm(1e-6) without affine, then
 * * scale[b, :] + shift[b, :] with per-clip rows `cond_stride` floats apart (scale / shift = Linear(d_vector)). */
int qb_dwconv7_adaln(const float* x, const float* dw_w, const float* dw_b, const float* scale, const float* shift,
                     int64_t cond_stride, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo, void* stream);
int qb_adalayernorm(const float* x, const float* scale, const float* shift, int64_t cond_stride, float eps, int64_t B,
                    int64_t rows, int64_t C, float* out_f32, qb_half* hi, qb_half* lo, int64_t ld,
                    int64_t rows_per_batch, int64_t row_off, void* stream);
/* Snake activation x + sin(alpha x)^2 / (alpha + 1e-9) per channel (bicodec/modules/blocks/layers.py:33-44) of fp32
 * rows [B, T, C] (clip b at x + b * x_batch_stride) -> planes in a padded buffer; channels C..ld-1 zeroed. */
int qb_snake_planes(const float* x, int64_t x_batch_stride, const float* alpha, int64_t B, int64_t T, int64_t C,
                    qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream);
/* ELU of fp32 rows [B, T, C] (clip b at x + b * x_batch_stride) -> planes in a padded buffer; channels C..ld-1 zeroed.  Reads the
 * up-sampled frames of a transposed conv's phase GEMM (the ResidualUnit's first ELU, vq/semantic_module.py:78-79). */
int qb_elu_planes(const float* x, int64_t x_batch_stride, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo, int64_t ld,
                  int64_t rows_per_batch, int64_t row_off, void* stream);
/* x[b,t,:] + vec[b,:] -> planes (prenet output + speaker d-vector, bicodec/bicodec.py:196-197). */
int qb_addvec_planes(const float* x, const float* vec, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo,
                     int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream);
/* GroupNorm(32 groups, eps) statistics then apply (+ optional swish): vq/conv.py:261,286-300.
 * x [B,T,C] fp32; stats [B,32,2] (mean, rstd).  Output fp32 and/or planes into a padded buffer. */
int qb_groupnorm_stats(const float* x, int64_t B, int64_t T, int64_t C, int32_t groups, float eps, float* stats,
                       void* stream);
int qb_groupnorm_apply(const float* x, const float* stats, const float* w, const float* b, int64_t B, int64_t T,
                       int64_t C, int32_t groups, int32_t swish, float* out_f32, qb_half* hi, qb_half* lo,
                       int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream);

/* ---------------------------------------------------------------- spectral front / back end */
/* Two-stage STFT (n_fft = P*Q; P <= 64, Q <= 64) of the padded, windowed frames (vq/codec_encoder.py:65-71): MMA chains of
 * 4 / 8 instead of the n_fft/16 of one K = n_fft DFT GEMM - the tensor core truncates on every accumulate, and at K = 1920 that
 * bias is 25x an fp32 FFT's error (csrc/elementwise.cu).
 * gather -> qb_gemm [.., 64] x W_A[2P, 64] -> twiddle -> qb_gemm [.., 128] x W_B[2*(nf/P+1), 128] -> post2.
 * qb_stft_gather: planes [(B*F*Q), 64], row (clip, f, b) col a = pad(wav)[hop f + Q a + b] * window[Q a + b].
 * qb_stft_twiddle: Y [(frames_total*Q), ldY] (cols 2 k1, 2 k1 + 1 = re, im) x twiddle[b*P + k1] = (cos, -sin)(2 pi k1 b / n_fft)
 *   -> planes [(frames_total*P), 128] (cols b = re, Q + b = im).
 * qb_stft_post2: X[k] = row (clip, f, k % P), cols 2 (k / P), 2 (k / P) + 1 of X [.., ldX] -> log(clip(|X|,1e-5)), angle/pi
 *   planes [B, rows_per_batch, ld] (channels: mag 0..nf-1, phase nf..2nf-1, zero pad); imag of DC/Nyquist forced to +0. */
int qb_stft_gather(const float* wav, int64_t B, int64_t T, int32_t hop, int32_t n_fft, int32_t P, int32_t Q, const float* window,
                   qb_half* hi, qb_half* lo, void* stream);
int qb_stft_twiddle(const float* Y, int64_t ldY, int64_t frames_total, int32_t P, int32_t Q, const float* twiddle, qb_half* hi,
                    qb_half* lo, void* stream);
int qb_stft_post2(const float* X, int64_t ldX, int64_t B, int64_t frames, int32_t nf, int32_t P, qb_half* hi, qb_half* lo, int64_t ld,
                  int64_t rows_per_batch, int64_t row_off, void* stream);
/* head output [M, ld_in] fp32 (mag | phase) -> planes [M, ld]: re = min(exp(mag),100)*cos(p),
 * im = ...*sin(p)   (vq/heads.py:55-65). */
int qb_istft_pre(const float* head, int64_t ld_in, int64_t M, int32_t nf, qb_half* hi, qb_half* lo, int64_t ld,
                 void* stream);
/* windowed frames [B, F, n_fft] fp32 -> overlap-add (n_fft a multiple of hop), trim, / window envelope
 * -> wav [B, F*hop]   (vq/spectral_ops.py:56-73). */
int qb_istft_ola(const float* frames, const float* window, int64_t B, int64_t F, int32_t n_fft, int32_t hop,
                 float* wav, void* stream);
/* Reflect padding of SConv1d (HCodec-1.0/vq/encoder_modules/conv.py:79-96,196-210): mirror-fill pad_l rows
 * before and pad_r rows after the T interior rows (starting at row_off) of a padded plane buffer. */
int qb_reflect_pad_rows(qb_half* hi, qb_half* lo, int64_t B, int64_t rows_per_batch, int64_t ld, int64_t T,
                        int64_t row_off, int32_t pad_l, int32_t pad_r, void* stream);
/* Depthwise conv over time, odd k, zero 'same' padding, channel-last fp32; w [C,k]
 * (sub-pixel up-sampler's dw conv, HCodec-1.0/vq/conv.py:84-92). */
int qb_dwconv(const float* x, const float* w, const float* bias, int64_t B, int64_t T, int64_t C, int32_t k,
              float* out, void* stream);

/* ---------------------------------------------------------------- sequence ops */
/* Non-causal multi-head attention with RoPE applied to q,k on load (encoder_modules/transformer.py:134-182), fp32 SIMT:
 * qkv [B,T,3*H*D] fp32 (q|k|v), head_dim D 64, 96 or 128.  Output planes.  The product runs head_dim 96 here (H-Codec-1.0's
 * decoder transformer: 768 / 8 heads); 64 and 128 go to qb_attention_umma. */
int qb_attention_hd(const float* qkv, int64_t B, int64_t T, int32_t heads, int32_t head_dim, const float* rope_cos,
                    const float* rope_sin, qb_half* out_hi, qb_half* out_lo, void* stream);
/* The same attention on the Hopper tensor cores (wgmma, accumulators in registers, TMA-fed operands; csrc/attention_umma.cu):
 * head_dim 64 or 128, any L; split = 0: single-pass fp16 operands, split = 1: fp16 hi + lo operands for both contractions (3 passes,
 * fp32-grade); causal = 1: query t attends keys <= t (the AR-LM's teacher-forced / prefill attention, U/model/llm/llm.py:195-216).
 * q is scaled by head_dim^-0.5; rope tables [L, head_dim] in the rotate-half layout.  workspace: 128-byte aligned,
 * qb_attention_umma_workspace_bytes(...) bytes (the fp16 operand planes a prep launch writes).  out_lo may be NULL. */
int64_t qb_attention_umma_workspace_bytes(int64_t B, int64_t L, int32_t heads, int32_t head_dim, int32_t split);
int qb_attention_umma(const float* qkv, int64_t B, int64_t L, int32_t heads, int32_t head_dim, const float* rope_cos,
                      const float* rope_sin, qb_half* out_hi, qb_half* out_lo, int32_t split, int32_t causal, void* workspace,
                      void* stream);
/* Single-layer LSTM recurrence (encoder_modules/transformer.py:115,133) on wgmma / TMA: xp [B,T,4H] fp32 already
 * holds x W_ih^T + b_ih + b_hh; output h planes [B,T,H] (out_lo may be NULL).  whh_perm: fp16 [H/U][4U][H] with
 * row (4j+g) of slice c = gate g of hidden unit c*U+j, U = qb_lstm_tc_units(H) (0: width unsupported; H % 256 == 0
 * is also required).  Any B: the rows run as independent recurrences in launches of at most 128 rows, one after
 * the other, so a row's result does not depend on B.  workspace: qb_lstm_tc_workspace_bytes(B,H). */
int32_t qb_lstm_tc_units(int64_t H);
int64_t qb_lstm_tc_workspace_bytes(int64_t B, int64_t H);
int qb_lstm_tc(const float* xp, const qb_half* whh_perm, int32_t units, int64_t B, int64_t T, int64_t H,
               qb_half* out_hi, qb_half* out_lo, void* workspace, void* stream);

/* ---------------------------------------------------------------- residual vector quantiser */
/* x [M,D] fp32, codebooks [nq,K,D] fp32 (+ their fp16 planes cb_hi/cb_lo [nq,K,D]) -> idx [M,nq] int64
 * (+ optional quantized [M,D]).  Per layer: scores |e|^2 - 2 r.e on the tensor cores (3-term split),
 * arg-min with an exact fp64 re-rank of every candidate within tolerance of the minimum, lowest index
 * wins exact ties; residual updated in fp32 (codec.py:81-82; core_vq.py:223-238,394-412).
 * neg_half_e2: [nq*K] values -|e|^2/2 followed by K values of -2.0 (epilogue constants);
 * e2max = max_j |e_j|^2 (tolerance scale).  workspace: qb_rvq_workspace_bytes(M,D,K). */
int64_t qb_rvq_workspace_bytes(int64_t M, int32_t D, int32_t K);
int qb_rvq_encode(const float* x, const float* codebooks, const qb_half* cb_hi, const qb_half* cb_lo,
                  const float* neg_half_e2, float e2max, int64_t M, int32_t D, int32_t K, int32_t nq,
                  int64_t* idx, float* quantized, void* workspace, void* stream);
/* idx [M,nq] int64 (-1 = dropped) -> out[M, out_ld] (+ col_off) = sum_q codebooks[q][idx_q]
 * summed q = 0..nq-1 in fp32 (codec.py:94-95). */
int qb_rvq_decode(const int64_t* idx, const float* codebooks, int64_t M, int32_t D, int32_t K, int32_t nq,
                  float* out, int64_t out_ld, int64_t col_off, void* stream);
/* Factorised VQ tokenize: BiCodec's semantic quantiser, FactorizedVectorQuantize.tokenize / in_project / decode_latents
 * (QuarkAudio-UniSE/model/bicodec/modules/vq/factorized_vector_quantize.py:59-61,148-152,169-187).  Per row of z [M, D_in] fp32:
 * z_e = W_in z + b_in (W_in [cdim, D_in] with the weight norm folded, fp64 sums), e = z_e / max(|z_e|, 1e-12) and
 * idx = argmax_j (2 e.c_j - |c_j|^2) over codebook_n [K, cdim] fp64 = F.normalize(codebook) - the reference's argmax of -dist
 * without the row constant |e|^2 - all in fp64, lowest index on exact ties.  idx [M] int64; z_e [M, cdim] fp32 (the in_project
 * output, before normalisation) if not NULL.  1 <= cdim <= 16. */
int qb_fvq_tokenize(const float* z, int64_t M, int32_t D_in, const float* w_in, const float* b_in, const double* codebook_n,
                    int32_t K, int32_t cdim, int64_t* idx, float* z_e, void* stream);
/* FactorizedVectorQuantize.forward's code usage in eval mode (factorized_vector_quantize.py:97-103): idx [n] int64 ->
 * perplexity = exp(-sum_k p_k log(p_k + 1e-10)), p_k = count_k / n (fp64, rounded to fp32), and active = the number of codes used at
 * least once (fp32), each a single device float.  counts: K int32 of scratch (the histogram, integer atomics).  n >= 1 and K >= 1
 * are checked; an index outside [0, K) is not counted (the indices come from qb_fvq_tokenize, which writes none). */
int qb_fvq_usage(const int64_t* idx, int64_t n, int32_t K, int32_t* counts, float* perplexity, float* active, void* stream);

/* ---------------------------------------------------------------- UniSE AR-LM (decoder-only Llama-style LM)
 * Reference: QuarkAudio-UniSE/model/llm/llm.py:150-228 (llm_forward over HF Llama decoder layers),
 * llm_sft.py:93-195 (prefill + 33 + T cached greedy steps).  The prefill / teacher-forced forward runs its
 * projections through qb_gemm; these entry points add the attention side and the KV-cache decode step. */
/* qkv [B,L,3*H*64] fp32 -> RoPE at absolute positions pos0.., q scaled by 1/8 -> q32 [B,H,L,64]; K/V appended
 * to the static fp32 cache [B,H,Lmax,64] at pos0.. */
int qb_lm_qkv_prep(const float* qkv, int64_t B, int64_t L, int32_t heads, int32_t pos0, const float* rope_cos,
                   const float* rope_sin, float* q32, float* k_cache, float* v_cache, int32_t Lmax, void* stream);
/* causal flash attention over the cache: query t (absolute position pos0+t) sees keys 0..pos0+t; operands are
 * split into fp16 hi/lo planes on the fly and multiplied as 3-term split MMAs (fp32-grade scores). */
int qb_lm_flash_attn(const float* q32, const float* k_cache, const float* v_cache, int64_t B, int64_t L,
                     int32_t heads, int32_t pos0, int32_t Lmax, qb_half* out_hi, qb_half* out_lo, void* stream);
/* ---- KV-cache decode step ----
 * Weights are pre-packed ONCE with qb_lm_pack_weight: row-major [n][k] fp32 -> [n][k/4] 16-byte groups
 * {hi[4], lo[4]} of fp16 (hi = rn16(w), lo = rn16(w - hi)): 4 bytes / parameter like fp32, and one 16-byte load is
 * directly the B fragment of two MMA k-slots.  Each kernel issues its weight loads before `griddepcontrol.wait` and is
 * launched as a programmatic dependent of its predecessor (works inside stream capture); products are 3-term
 * fp16-split mma.sync tiles with fp32 accumulation.
 * Replaces: HF Llama decoder layer on one cached token - QuarkAudio-UniSE/model/llm/llm.py:195-228 driven by
 * llm_sft.py:155-191. */
int qb_lm_pack_weight(const float* w, int64_t n, int64_t k, qb_half* out /* [n][2k] */, void* stream);
/* One decoder layer for ONE new token per sequence (B <= 32): x [B,hidden] updated in place.  `pos` points at B device ints
 * (not modified here): row b's RoPE angle and K/V append use pos[b] and its attention reads keys 0..pos[b], so rows whose
 * conditioning prefixes (llm_sft.py:108-122) differ in length decode together.  wqkv = packed [q;k;v] rows [3*hidden, hidden]; scratch q_buf/attn_buf [B,hidden],
 * mlp_buf [B,inter].  The RMSNorm weights must be FOLDED into the following projection by the caller BEFORE packing
 * (wqkv' = wqkv diag(in_norm), wgate' / wup' likewise with post_norm): the kernels apply only the per-row 1/rms. */
int qb_lm_decode_layer_tc(float* x, int64_t B, int32_t hidden, int32_t heads, int32_t inter, const qb_half* wqkv,
                          const qb_half* wo, const qb_half* wgate, const qb_half* wup, const qb_half* wdown,
                          float* k_cache, float* v_cache, int32_t Lmax, const int32_t* pos, const float* rope_cos,
                          const float* rope_sin, float* q_buf, float* attn_buf, float* mlp_buf, void* stream);
/* Keys whose K / V rows one lane of the cached-decode attention keeps in flight per trip: 8 (default; a single decode chain is
 * latency-bound) or 4 (several chains sharing the GPU are throughput-bound - LLM_SFT.generate's lanes select it).  Process-wide;
 * read at launch (and therefore fixed inside a captured graph).  Tokens do not depend on it only up to the fp32 summation order of
 * the online softmax: set it once per decode state. */
int qb_lm_set_att_unroll(int32_t keys_per_lane);
/* Final RMSNorm + packed output head restricted to columns [range[0], range[1]) (device ints; llm_sft.py:148-153)
 * + greedy arg-max (llm.py:286-287, do_sample=False) -> out_ids[b*out_stride + slot[0]]; x_next[b] =
 * embedding[token]; then slot[0]++ and pos[b]++ for every row (pos: B device ints; slot is int32[2], second word is
 * scratch).  B <= 32.
 * w_head must have final_norm folded in BEFORE packing (w_head' = w_head diag(final_norm)); max_cols and the range
 * width must be multiples of 16; part_val/part_idx: scratch [max_cols/16 * 32]. */
int qb_lm_head_argmax_tc(const float* x, int64_t B, int32_t hidden, const qb_half* w_head, const int32_t* range,
                         int32_t max_cols, const float* embedding, float* x_next, int64_t* out_ids, int32_t out_stride,
                         int32_t* pos, int32_t* slot, float* part_val, int32_t* part_idx, void* stream);

/* Teacher-forced loss + accuracy (CustomLlamaModel.loss_function, QuarkAudio-UniSE/model/llm/llm.py:87-104): label-smoothed KL
 * (reduction batchmean) of log_softmax(logits [M, ld >= V]) against the smoothed one-hot targets [M] int64, and the arg-max
 * accuracy -> out = {loss, accuracy}; workspace: 2*M floats.  One pass over the logits, deterministic reduction. */
int qb_lm_loss(const float* logits, int64_t ld, int64_t M, int32_t V, const int64_t* targets, float label_smoothing, float* workspace,
               float* out, void* stream);
/* ---- training: gradients of the teacher-forced loss (csrc/lm_train.cu) ----
 * Deterministic: no floating-point atomics, fixed-order reductions, fp64 partials where a sum runs over tokens.  The dense
 * contractions of the backward pass are qb_gemm calls in the 3-term split mode; these entry points are the rest.
 *
 * Attention dropout mask (transformers' Llama attention in train mode: dropout on the softmax output, before P V): key j of query i in
 * head h of batch row b, decoder layer `layer`, is kept iff (r >> 8) >= thr, where r is word (j & 3) of
 * Philox4x32-10(key = {seed & 0xffffffff, seed >> 32}, counter = {i, j >> 2, b * heads + h, layer}) and thr is the float dropout_p as
 * received times 2^24, rounded to the nearest integer with ties to even (so a caller's double p counts as (float)p); kept probabilities
 * are scaled by 1 / (1 - p).  The mask is a pure function of (seed, layer, b, h, i, j), so the backward pass regenerates it.
 *
 * qb_lm_attn_train_fwd: causal attention, head_dim 64, fp32 SIMT.  qkv [B*L, 3*heads*64] fp32 (rope tables as qb_attention_umma)
 * -> qs = RoPE(q) / 8, kr = RoPE(k), v, each [B*heads, L, 64] (kept for the backward pass), out [B*L, heads*64] fp32 and the row
 * log-sum-exp lse [B*heads, L] of the undropped scores.  0 <= dropout_p < 1.
 * qb_lm_attn_train_bwd: dout [B*L, heads*64] -> dqkv [B*L, 3*heads*64] (RoPE undone on dq and dk), P recomputed from lse with the same
 * mask; dK / dV summed per key tile and dQ per query tile.  workspace: B*heads*L floats. */
int qb_lm_attn_train_fwd(const float* qkv, int64_t B, int64_t L, int32_t heads, const float* rope_cos, const float* rope_sin,
                         float dropout_p, uint64_t seed, int32_t layer, float* qs, float* kr, float* v, float* out, float* lse,
                         void* stream);
int qb_lm_attn_train_bwd(const float* qs, const float* kr, const float* v, const float* out, const float* dout, const float* lse,
                         int64_t B, int64_t L, int32_t heads, const float* rope_cos, const float* rope_sin, float dropout_p,
                         uint64_t seed, int32_t layer, float* dqkv, float* workspace, void* stream);
/* Gradient of qb_lm_loss's loss times *grad_loss (a device float) w.r.t. the logits, times M * scale: *grad_loss * (softmax(logits) - t)
 * * scale with t the smoothed target -> out fp32 and hi / lo planes, all [M, ld_out] (columns V.. zero).  Most entries are ~1/V, below
 * fp16's normal range: a power-of-two scale near V (<= 2^14, so that |out| <= 2^14 |*grad_loss|) keeps the planes fp32-grade while
 * |*grad_loss| * 2^14 stays well inside fp16's range (lo overflows from |out| ~ 2^17, and at |*grad_loss| ~ 2^-16 the ~1/V entries fall
 * into fp16 subnormals).  LLM_SFT passes a unit *grad_loss and multiplies the finished parameter gradients by the real one.  The caller
 * takes the scale back out (LLM_SFT: the head GEMM's gamma; qb_col_sum / qb_embedding_bwd scale the parameter gradients). */
int qb_lm_loss_bwd(const float* logits, int64_t ld, int64_t M, int32_t V, const int64_t* targets, float label_smoothing,
                   const float* grad_loss, float scale, float* out, qb_half* out_hi, qb_half* out_lo, int64_t ld_out, void* stream);
/* RMSNorm backward (eps as qb_rmsnorm): dx = (accumulate ? dx : 0) + d/dx; gw [rows, C] = dy * x * rms^-1 (qb_col_sum gives dw). */
int qb_rmsnorm_bwd(const float* x, const float* w, const float* dy, float eps, int64_t rows, int64_t C, float* dx, int32_t accumulate,
                   float* gw, void* stream);
/* out[c] = (accumulate ? out[c] : 0) + scale * sum over r = 0..rows-1 in order of x[r * ld + c], in fp64 (chunks of 128 rows, then the
 * chunks in order).  workspace: qb_col_sum_workspace_bytes(rows, C). */
int64_t qb_col_sum_workspace_bytes(int64_t rows, int64_t C);
int qb_col_sum(const float* x, int64_t rows, int64_t C, int64_t ld, double scale, void* workspace, float* out, int32_t accumulate,
               void* stream);
/* gu [M, 2*inter] fp32, (gate, up) interleaved per column: qb_swiglu -> h = silu(gate) * up, fp32 and planes [M, inter];
 * qb_swiglu_bwd: dh [M, inter] -> d(gate, up) [M, 2*inter] fp32 and planes. */
int qb_swiglu(const float* gu, int64_t M, int64_t inter, float* h, qb_half* hi, qb_half* lo, void* stream);
int qb_swiglu_bwd(const float* gu, const float* dh, int64_t M, int64_t inter, float* dgu, qb_half* hi, qb_half* lo, void* stream);
/* x [rows, cols] fp32 (row pitch ldx) -> hi / lo planes [S][cols][ks], element (s, c, k) = x[s*ks + k, c], S = ceil(rows / ks), rows
 * past `rows` zero; ks a multiple of 64.  Slice s is the A or W operand of one split-K slice of a weight gradient dW = dY^T X. */
int qb_transpose_split(const float* x, int64_t rows, int64_t cols, int64_t ldx, int64_t ks, qb_half* hi, qb_half* lo, void* stream);
/* Embedding gradient: out[v] (+)= scale * sum over k with ids[k] == v, in increasing k and in fp64, of dx row (k / Lt) * L + P + k % Lt
 * (rows of H floats); ids [n] int64 in [0, V).  H <= 1024. */
int qb_embedding_bwd(const float* dx, const int64_t* ids, int64_t n, int64_t Lt, int64_t L, int64_t P, int32_t H, int32_t V,
                     double scale, float* out, int32_t accumulate, void* stream);

/* Sampled decoding step (CustomLlamaModel.sample_logits, QuarkAudio-UniSE/model/llm/llm.py:253-289, as called from
 * llm_sft.py:155-161,184-190 with the reference defaults temperature 0.8, top_k 50, top_p 0.95, do_sample=True):
 * as qb_lm_head_argmax_tc, but the head also writes the range logits to `logits` [B][max_cols] and the token is drawn as
 * top-k (ties at the k-th value kept) -> top-p over the survivors' softmax (sorted descending; the first token always stays)
 * -> / temperature -> softmax -> inverse-CDF draw over the kept tokens in descending-logit order at
 * u = Philox4x32-10(key = {seed[0], seed[1]}, counter = {step (= slot[0]), row, seed[2], 0}).x >> 8) * 2^-24.
 * seed: device uint32[4] {seed_lo, seed_hi, call_counter, 0}; debug: optional device float [B][4] = {u, survivors after
 * top-k, kept after top-p, sum of the kept exp((l - max)/T)} or NULL.  0 < temperature <= 1.
 * top_k <= 0 applies no top-k filter and top_k >= the range width keeps every token of the range (llm.py:262 runs torch.topk on
 * the range-masked row); top_p >= 1 applies no top-p filter.  1 <= top_k <= 1024 runs a kernel that stores the survivors above
 * the k-th value and walks them on one thread; any other top_k runs one that stores and sorts every survivor (up to the whole
 * range, max_cols <= 8192: row keys + 8 bytes per survivor slot, 96 KB of shared memory at 8192) and makes the top-p cut, the
 * normaliser and the draw fixed-order block-wide scans.  Both are deterministic (no floating-point atomics).  The scans sum in
 * another order than the reference's sequential torch.cumsum, so a token whose cumulative probability lies within ~1e-6 of
 * top_p (or of the draw's target) can fall on the other side of the boundary. */
int qb_lm_head_sample_tc(const float* x, int64_t B, int32_t hidden, const qb_half* w_head, const int32_t* range,
                         int32_t max_cols, const float* embedding, float* x_next, int64_t* out_ids, int32_t out_stride,
                         int32_t* pos, int32_t* slot, float* part_val, int32_t* part_idx, float* logits,
                         float temperature, int32_t top_k, float top_p, const uint32_t* seed, float* debug, void* stream);
/* qb_lm_head_sample_tc with one random stream per row: row_keys is device uint32[B][2] = {key_lo, key_hi} per row, and row b's
 * uniform at step s (= slot[0]) is (Philox4x32-10(key = row_keys[b], counter = {s, 0, 0, 0}).x >> 8) * 2^-24, a function of
 * its key and the step only (not of b, the batch size or the call), so a row draws the same tokens in any batch.  A row keyed
 * k draws what row 0 of call 0 draws from qb_lm_head_sample_tc with seed k. */
int qb_lm_head_sample_rows_tc(const float* x, int64_t B, int32_t hidden, const qb_half* w_head, const int32_t* range,
                              int32_t max_cols, const float* embedding, float* x_next, int64_t* out_ids, int32_t out_stride,
                              int32_t* pos, int32_t* slot, float* part_val, int32_t* part_idx, float* logits,
                              float temperature, int32_t top_k, float top_p, const uint32_t* row_keys, float* debug,
                              void* stream);

/* ---------------------------------------------------------------- SSL feature front ends + tokenizer glue (SURVEY 8f.2 / 8f.3)
 * HuBERT-base / WavLM-base-plus (transformers modeling_hubert / modeling_wavlm) as the reference drives them from
 * HCodecTokenizer.extract_ssl_features (QuarkAudio-HCodec/HCodec-2.0/audio_tokenizer.py:47-61) and
 * Model.extract_semantic_features (QuarkAudio-UniSE/model/model.py:38-51).  The dense contractions (Resample as a 2-tap
 * Toeplitz GEMM, conv layers 1-6, projections, grouped positional conv via `a_cols`, attention, FFN) run on qb_gemm /
 * qb_attention_hd / qb_layernorm; these entry points add what is not a contraction. */
/* Feature-encoder layer 0: x [B, T_in] fp32 -> Conv1d(1, C, k, stride, bias=False) -> GroupNorm(C groups: per channel over
 * time, eps) -> GELU(erf) -> planes of a channel-last buffer [B, rows_per_batch, ld].  y_scratch: [B, T0, C] fp32 with
 * T0 = (T_in - k) / stride + 1; workspace: qb_ssl_conv0_workspace_bytes(B, T0, C). */
int64_t qb_ssl_conv0_workspace_bytes(int64_t B, int64_t T0, int32_t C);
int qb_ssl_conv0_gn_gelu(const float* x, int64_t B, int64_t T_in, const float* w, int32_t C, int32_t k, int32_t stride,
                         const float* gn_w, const float* gn_b, float eps, float* y_scratch, void* workspace, qb_half* hi,
                         qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream);
/* wav2vec2-large-xlsr-53 (transformers Wav2Vec2Model, conv_bias=True) feature-encoder layer 0: x [B, T_in] fp32 ->
 * Conv1d(1, C, k, stride) + bias -> y [B, T0, C] fp32, T0 = (T_in - k) / stride + 1 (LayerNorm + GELU: qb_layernorm_act). */
int qb_ssl_conv0_bias(const float* x, int64_t B, int64_t T_in, const float* w, const float* bias, int32_t C, int32_t k,
                      int32_t stride, float* y, void* stream);
/* Wav2Vec2FeatureExtractor(do_normalize=True): per utterance out = (x - mean) / sqrt(var + eps), population variance,
 * statistics in fp64 (BiCodecTokenizer.extract_wav2vec2_features, QuarkAudio-UniSE/model/bicodec/audio_tokenizer.py:74-90). */
int qb_wav_normalize(const float* x, int64_t B, int64_t T, float eps, float* out, void* stream);
/* WavLM-base-plus attention (transformers modeling_wavlm.WavLMAttention as UniSE drives it, U/model/model.py:30,38-51):
 * gate[b, h, t] = ga (gb const_h - 1) + 2, (ga, gb) = sigmoid of the two 4-sums of Linear(head_dim -> 8)(x[b, t, head h]);
 * qb_attention_relbias: softmax(q k^T / sqrt(d) + gate[b, h, i] * rel_table[h, (j - i) + T - 1]) v, no rotary embedding;
 * qkv [B, T, 3*heads*64] fp32, rel_table [heads, 2T - 1] (bucketed relative-position embedding per distance), output planes. */
int qb_wavlm_gate(const float* x, int64_t B, int64_t T, int32_t heads, int32_t head_dim, const float* w, const float* bias,
                  const float* cst, float* gate, void* stream);
int qb_attention_relbias(const float* qkv, int64_t B, int64_t T, int32_t heads, int32_t head_dim, const float* rel_table,
                         const float* gate, qb_half* out_hi, qb_half* out_lo, void* stream);
/* out = scale * x (accumulate == 0) or out += scale * x: the running mean over the 13 hidden states (audio_tokenizer.py:55). */
int qb_axpy(const float* x, float scale, int64_t n, int32_t accumulate, float* out, void* stream);
/* x [B, T, C] fp32 -> sign(x) * |x| ** power (audio_tokenizer.py:57-60; power <= 0: copy), written channel-first [B, C, T]
 * (channel_first != 0: the layout Codec.encode takes) or channel-last. */
int qb_ssl_compress(const float* x, int64_t B, int64_t T, int32_t C, float power, int32_t channel_first, float* out, void* stream);
/* out[b, i] = x[b, i - left] (zero outside, or wrapped modulo T_in when wrap != 0): pad_wav (audio_tokenizer.py:63-66),
 * F.pad(wavs, (160, 160)) (:51), wrap padding of UniSE segments (QuarkAudio-UniSE/model/model.py:175-181). */
int qb_pad_wav(const float* x, int64_t B, int64_t T_in, int64_t left, int64_t T_out, int32_t wrap, float* out, void* stream);

/* ---------------------------------------------------------------- BiCodec global (speaker) tokens (SURVEY 8f.1, csrc/speaker.cu)
 * BiCodec.get_global_tokens (QuarkAudio-UniSE/model/bicodec/bicodec.py:174-178): MelSpectrogram -> ECAPA-TDNN latent ->
 * PerceiverResampler -> ResidualFSQ indices.  Convolutions and linears run on qb_gemm (Conv1dReluBn as QB_ACT_RELU + gamma + a
 * broadcast residual row); the DFT is the two-stage one of the STFT above (qb_stft_twiddle).
 * qb_mel_gather: torch.stft(center=True, pad_mode="reflect") framing of wav [B, L], 1 + L / hop frames, in qb_stft_gather's layout
 *   (torchaudio MelSpectrogram, bicodec.py:201-221; window [n_fft] = the win_length window zero-padded to the middle of n_fft).
 * qb_spec_magnitude: |X[k]|, k < nf, of the second DFT stage (layout of qb_stft_post2) -> planes [M, ld], zero past nf. */
int qb_mel_gather(const float* wav, int64_t B, int64_t L, int32_t hop, int32_t n_fft, int32_t P, int32_t Q, const float* window,
                  qb_half* hi, qb_half* lo, void* stream);
int qb_spec_magnitude(const float* X, int64_t ldX, int64_t M, int32_t nf, int32_t P, qb_half* hi, qb_half* lo, int64_t ld, void* stream);
/* x [B*T rows, pitch ldx] (+ y [B*T rows, pitch ldy], or NULL) over C channels -> planes of a padded buffer [B, rows_per_batch, ld]
 * at row_off, channels C..ld-1 zeroed: Res2Conv1dReluBn's sp + spx[i] (modules/speaker/ecapa_tdnn.py:68-83). */
int qb_add_planes(const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo,
                  int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream);
/* SE_Connect (ecapa_tdnn.py:116-129): s [B, C] = sigmoid(W2 relu(W1 mean_t z + b1) + b2), z [B, T, C]; W1 [R, C], W2 [C, R]; the
 * time mean is a fixed-order fp64 sum.  qb_se_apply: x + z * s (ecapa_tdnn.py:150) -> fp32 out [B*T, C] and / or planes at column
 * col_off of rows of ld channels (the block's slice of the 3 x C concat, ecapa_tdnn.py:203). */
int qb_se_gate(const float* z, int64_t B, int64_t T, int32_t C, const float* w1, const float* b1, int32_t R, const float* w2,
               const float* b2, float* s, void* stream);
int qb_se_apply(const float* z, const float* s, const float* x, int64_t B, int64_t T, int32_t C, float* out, qb_half* hi, qb_half* lo,
                int64_t ld, int64_t col_off, void* stream);
/* GEGLU (perceiver_encoder.py:232-235): h [rows, 2*inner] fp32 (value | gate, the reference's chunk order) -> planes [rows, ld] =
 * gelu_erf(gate) * value, zero past inner.  A kernel rather than a GEMM epilogue: an epilogue variant grew the GEMM kernels' code by a
 * fifth and measurably slowed the H-Codec path that never uses it. */
int qb_geglu_planes(const float* h, int64_t rows, int32_t inner, qb_half* hi, qb_half* lo, int64_t ld, void* stream);
/* fp32 cross attention, head_dim 64, scale 1/8 (perceiver_encoder.py:135-178,280-294): q [B, Nq, heads*64], kv [B, Nk, 2*heads*64]
 * (keys | values) -> planes [B*Nq, heads*64].  Nk <= 3072. */
int qb_cross_attention(const float* q, const float* kv, int64_t B, int64_t Nq, int64_t Nk, int32_t heads, qb_half* out_hi,
                       qb_half* out_lo, void* stream);
/* RMSNorm F.normalize(x) * sqrt(dim) * gamma (perceiver_encoder.py:195-214) -> project_in (W [n_levels, dim], b) -> FSQ bound,
 * round half to even, codes_to_indices (finite_scalar_quantization.py:126-157; residual_fsq.py:158-252 with one quantizer):
 * x [rows, dim] fp32 -> idx [rows] int32; z [rows, n_levels] (project_in output) and xn [rows, dim] (normed rows) if not NULL.
 * `levels` is a HOST array of n_levels <= 8 entries; num_quantizers other than 1 is refused. */
int qb_fsq_tokenize(const float* x, int64_t rows, int32_t dim, const float* gamma, const float* w_in, const float* b_in, int32_t n_levels,
                    const int32_t* levels, int32_t num_quantizers, int32_t* idx, float* z, float* xn, void* stream);
/* ASTP with global context (pooling_layers.py:119-144), the pooling of ECAPA_TDNN's x-vector (ecapa_tdnn.py:205-207), around qb_gemm:
 * x is the fp32 latent [B, T, C] channel-last.  Per (clip, channel) every time sum runs over the T frames in order in fp64.
 * qb_asp_context: [mean | sqrt(var + 1e-7)] with the unbiased variance (torch.var, divisor T - 1; T >= 2) -> out [B, 2C] fp32 and
 *   planes [B, ld] (columns 0..2C-1), the A operand of linear1's context part.
 * qb_asp_tanh_planes: tanh(h[b*T + t, :] + row[b, :]) over N columns -> planes [B*T, ld], zero past N: linear1 split into its x
 *   part h (a GEMM over the frames) and its context part plus bias (one row per clip), which a GEMM epilogue cannot add (act comes
 *   before residual, and a row map has no per-clip broadcast).
 * qb_asp_pool: alpha = softmax over T of logits [B, T, C] (maximum subtracted), mean = sum alpha x, std = sqrt(max(sum alpha x^2 -
 *   mean^2, 1e-7)) -> out [B, 2C] = [mean | std] fp32 and planes [B, ld], the input of the BatchNorm-folded final linear. */
int qb_asp_context(const float* x, int64_t B, int64_t T, int32_t C, float* out, qb_half* hi, qb_half* lo, int64_t ld, void* stream);
int qb_asp_tanh_planes(const float* h, const float* row, int64_t B, int64_t T, int32_t N, qb_half* hi, qb_half* lo, int64_t ld,
                       void* stream);
int qb_asp_pool(const float* x, const float* logits, int64_t B, int64_t T, int32_t C, float* out, qb_half* hi, qb_half* lo, int64_t ld,
                void* stream);

/* ---------------------------------------------------------------- H-Codec-1.5 adaptive frame-rate primitives (SURVEY 8f.4)
 * FlexiCodec._perform_similarity_alignment_vectorized (HCodec-1.5/adaptive/modeling_flexicodec_new.py:828-921): h [B, T, D] fp32 ->
 * sim [B, T-1] (cosine similarity of consecutive frames), seg [B, T] (frame -> token: a token ends where sim <= threshold or after
 * max_tokens_per_group frames), lengths [B, T] (frames per token, 0 past the last), n_groups [B].  qb_alignment_matrix expands seg
 * into the reference's dense [B, G, T] 0/1 matrix for the callers that want it. */
int qb_similarity_alignment(const float* h, int64_t B, int64_t T, int32_t D, float threshold, int32_t max_tokens_per_group, float* sim,
                            int32_t* seg, int32_t* lengths, int32_t* n_groups, void* stream);
int qb_alignment_matrix(const int32_t* seg, int64_t B, int64_t T, int64_t G, float* align, void* stream);
/* Codec._inject_length_to_codes_index / _extract_length_from_codes_index (HCodec-1.5/vq/codec_adaptive.py:68-80): codes [B, nq, G]
 * int64, lengths [B, G]: packed = (length - 1) * codebook_size + code; unpack returns code % K and length = code / K + 1 of row 0. */
int qb_pack_lengths(const int64_t* codes, const int32_t* lengths, int64_t B, int32_t nq, int64_t G, int32_t codebook_size, int64_t* out,
                    void* stream);
int qb_unpack_lengths(const int64_t* codes, int64_t B, int32_t nq, int64_t G, int32_t codebook_size, int64_t* plain, int32_t* lengths,
                      void* stream);
/* FlexiCodec._deaggregate_features_from_token_lengths (modeling_flexicodec_new.py:1007-1041): x [B, C, G] (4- or 8-byte elements)
 * repeated per token length -> out [B, C, T_out] zero padded; offsets / totals from qb_length_offsets (exclusive prefix sums). */
int qb_length_offsets(const int32_t* lengths, int64_t B, int64_t G, int32_t* offsets, int32_t* totals, void* stream);
int qb_deaggregate(const void* x, int32_t elem_bytes, const int32_t* lengths, const int32_t* offsets, int64_t B, int64_t C, int64_t G,
                   int64_t T_out, void* out, void* stream);
/* QueryTokenAggregator (adaptive/model_blocks/mimi/transformer.py:740-826), the data movement either side of its transformer:
 * qb_agg_interleave builds the [B, T+G, D] sequence (frames in order, the query of a group = group mean + query_embedding right behind
 * the group's last frame, padded groups = the bare embedding at the tail) from channel-last feats [B, T, D], the frame -> token map
 * seg [B, T], lengths / offsets [B, G] (contiguous) and n_groups [B]; qpos [B, G] receives the row of every query.
 * qb_agg_gather reads the transformer's output rows at qpos -> tokens [B*G, D], zero for padded groups. */
int qb_agg_interleave(const float* feats, const int32_t* seg, const int32_t* lengths, const int32_t* offsets, const int32_t* n_groups,
                      const float* query_embedding, int64_t B, int64_t T, int64_t G, int32_t D, float* out, int32_t* qpos,
                      void* stream);
int qb_agg_gather(const float* x, const int32_t* qpos, const int32_t* n_groups, int64_t B, int64_t L, int64_t G, int32_t D, float* out,
                  void* stream);

/* ==========================================================================================================
 * Handle-level contract (SURVEY.md 8b): what a non-Python caller binds for H-Codec-2.0 and its residual quantisers.  A
 * handle owns its repacked weight arena, workspace and per-device context; every tensor argument is a caller-owned DEVICE
 * pointer (row-major, contiguous, 16-byte aligned); calls are stream-ordered and asynchronous, return 0 / negative, and
 * never synchronise the device after `*_load`.  A handle is bound to the device current at creation and is not
 * thread-safe.  The op-level entry points above are what these are built from (csrc/engine.cu); `Codec`
 * (unified_audio_b200/codec.py) calls these for the product path.  The UniSE AR-LM has no handle: `LLM_SFT`
 * (unified_audio_b200/llm.py) composes the op-level LM entry points above, and its C surface is the decode step
 * (qb_lm_decode_layer_tc + qb_lm_head_argmax_tc / qb_lm_head_sample_tc).
 * ========================================================================================================== */
typedef struct qb_handle qb_handle;   /* per-device context */
typedef struct qb_codec qb_codec;     /* H-Codec-2.0 model: weights + workspace */
typedef struct qb_rvq qb_rvq;         /* one residual vector quantiser (codebooks + search constants) */

/* A named fp32 tensor of the reference's state-dict (device pointer, contiguous). */
typedef struct {
  const char* name;      /* e.g. "encoder.prior_net.0.pwconv1.linear.weight" */
  const float* data;
  int32_t ndim;
  int64_t shape[4];
} qb_tensor;

enum { QB_PRECISION_MIXED = 0, QB_PRECISION_ACCURATE = 1, QB_PRECISION_FAST = 2, QB_PRECISION_MIXED_DEC16 = 3 };

/* H-Codec-2.0 hyper-parameters (QuarkAudio-HCodec/HCodec-2.0/conf/large_12.5hz_config.yaml; vq/codec.py:18-49). */
typedef struct {
  int32_t dim, intermediate_dim, dimension;          /* encoder/decoder width 1536, ConvNeXt hidden 4608, latent 512 */
  int32_t n_fft, hop_length;                         /* 1920 / 960 (n_fft == 2*hop required) */
  int32_t enc_convnext_layers, enc_transformer_layers;
  int32_t dec_convnext_layers, dec_transformer_layers;
  int32_t dec_input_channels;                        /* 2 * dimension */
  int32_t frame_stride;                              /* 50 Hz frames per token = 50 / target_frame_rate (4) */
  int32_t num_quantizers, codebook_size;
  int32_t sem_input_channels, sem_encode_channels, sem_out_channels;
  int32_t sem_n_blocks;
  int32_t sem_strides[8];
  int32_t precision;                                 /* QB_PRECISION_* (DESIGN.md "precision policy") */
} qb_codec_cfg;

int qb_init(int device, qb_handle** out);
/* stream-ordered device-to-device copy (lets a tap callback written in a language without a CUDA binding keep a buffer) */
int qb_memcpy_d2d(void* dst, const void* src, int64_t bytes, void* stream);
void qb_handle_free(qb_handle* h);
/* last error of this thread's most recent failing call (same buffer as qb_last_error()) */
const char* qb_handle_last_error(qb_handle* h);

/* Builds the model from the reference's state-dict tensors (names as `Codec.state_dict()` gives them: `encoder.*`,
 * `decoder.*`, `semantic_encoder.*`, `quantizer.layers.{i}._codebook.embed`, `semantic_quantizer...`): repacks every weight
 * once (fp16 planes, conv taps, interleaved SwiGLU rows, LSTM unit-major slices, DFT matrices in fp64).  Synchronous.
 * Replaces Codec.__init__ + load_state_dict (vq/codec.py:18-49, audio_tokenizer.py:27-35). */
int qb_codec_load(qb_handle* h, const qb_codec_cfg* cfg, const qb_tensor* named_weights, int32_t n, qb_codec** out);
void qb_codec_free(qb_codec* c);
/* Codec.encode (vq/codec.py:75-87): wav [B,T] fp32 (T a multiple of hop*frame_stride), feat [B,768,T/hop] fp32 ->
 * acoustic / semantic codes int64 [B, nq, N], N = T / (hop*frame_stride). */
int qb_codec_encode(qb_codec* c, const float* wav, int64_t B, int64_t T, const float* feat, int64_t* ac_codes,
                    int64_t* sem_codes, void* stream);
/* Codec.decode (vq/codec.py:89-99): codes int64 [B, nq, N] x2 -> wav [B, N*hop*frame_stride] fp32. */
int qb_codec_decode(qb_codec* c, const int64_t* ac_codes, const int64_t* sem_codes, int64_t B, int64_t N, float* wav,
                    void* stream);
/* Debug taps: when set, the engine calls `cb(user, name, dev_ptr, B, rows, C)` right after enqueueing the kernels that produce
 * the named intermediate ([B, rows, C] fp32, channel-last); the callee may enqueue a copy on the same stream.  NULL disables. */
typedef void (*qb_tap_fn)(void* user, const char* name, const float* data, int64_t B, int64_t rows, int64_t C);
int qb_codec_set_tap(qb_codec* c, qb_tap_fn cb, void* user);
/* Semantic decoder of a loaded codec (HCodec-2.0/vq/semantic_module.py:252-299, built at vq/codec.py:50-52 and called by
 * Codec.forward only, vq/codec.py:71): k3 conv -> per block {k3 conv at stride 1 | ConvTranspose1d(2s, s) otherwise} +
 * 2 x ResidualUnit(ELU, k3 conv, ELU, 1x1 conv, + x) -> k3 conv.  Its own cfg, so qb_codec_cfg keeps its layout.  `named` holds
 * the reference's semantic_decoder.* tensors (block widths are read from their shapes); the transposed convs are repacked into
 * phase GEMM weights here, at the codec's semantic-encoder precision.  A codec holds one semantic decoder: a second load fails. */
typedef struct {
  int32_t code_dim, output_channels;                 /* 512 -> 768 (semantic_decoder_config) */
  int32_t n_blocks;                                  /* len(strides) <= 8 */
  int32_t strides[8];
} qb_semantic_decoder_cfg;
int qb_codec_load_semantic_decoder(qb_codec* c, const qb_semantic_decoder_cfg* cfg, const qb_tensor* named, int32_t n);
/* pred_feat [B, output_channels, N * prod(strides)] fp32 channel-first = the semantic decoder on the semantic codes' codebook-row
 * sums (vq/codec.py:65-71 with get_output_from_indices); sem_codes int64 [B, nq, N]. */
int qb_codec_semantic_decode(qb_codec* c, const int64_t* sem_codes, int64_t B, int64_t N, float* pred_feat, void* stream);
/* Row-level access to the two quantisers of a loaded codec (which = 0 acoustic, 1 semantic). */
qb_rvq* qb_codec_rvq(qb_codec* c, int32_t which);

/* ---- UniSE training-data simulation (csrc/simulate.cu): TrainDataLoadIter.process_one_sample after the file reads
 * (QuarkAudio-UniSE/dataloader/data_module.py:106-140,207-235) and simulate_data with everything it calls (dataloader/simulation/
 * simulate.py:10-192, rir_utils.py:464-517, detect_non_silence.py:1-98).  Signals are packed ragged rows: one fp32 buffer, int64
 * offsets [rows + 1] (row r = buf[offs[r] .. offs[r + 1])).  Every random parameter is drawn on the host and passed per row; `on`
 * (int32 per row) selects the rows a stage applies to.  All reductions are fixed-order with fp64 partials: bit-reproducible. */
/* mix_noise's rms (simulate.py:25-26) = x[detect_non_silence(x)].std(): frame variance (frame 1024, shift 512, zero padding to whole
 * frames, boxcar window; detect_non_silence.py:1-98), frames with power / mean > 0.01, one flag per shift, the last repeated; rows
 * shorter than 1024 or of zero mean power select every sample -> rms [rows] fp64, mask (uint8 per sample, packed as x) or NULL.
 * frame_off [rows + 1]: frames per row (0 below 1024 samples) cumulated; power: fp64 workspace of frame_off[rows] entries. */
int qb_sim_active_rms(const float* x, const int64_t* offs, const int64_t* frame_off, int64_t rows, int64_t max_len, int64_t max_frames,
                      double* power, double* rms, uint8_t* mask, void* stream);
/* mix_noise's alignment (simulate.py:13-23): dst_r[n] = src_r[(n + shift[r]) mod len(src_r)], n < len(dst_r) (dst packed by offs):
 * wrap padding from an offset (shift = -offset mod len) or a cut at an offset (shift = offset); empty source rows give zeros. */
int qb_sim_place(const float* src, const int64_t* src_offs, const int64_t* offs, const int64_t* shift, int64_t rows, int64_t max_len,
                 float* dst, void* stream);
/* mix_noise (simulate.py:28-29) in place on rows with on[r]: x = other * (10^(-snr/20) rms_x / (rms_other + 1e-10)) + x; diff (or
 * NULL) = x_after - x_before, the interferer of simulate.py:147. */
int qb_sim_mix(float* x, const float* other, const int64_t* offs, int64_t rows, int64_t max_len, const double* snr, const double* rms_x,
               const double* rms_other, const int32_t* on, float* diff, void* stream);
/* simulate.py:153 + get_rir_start_sample (rir_utils.py:483-517) on rows with on[r]: hn = h / (max|h| + 1e-5); win [rows, 2] = the
 * early part [start, end) around the first peak of |hn| with strict thresholds at 0.1 peak (end = peak + 1 when nothing after the peak
 * falls below); status[r] = 1 when the peak is the last sample (the reference fails there), else 0. */
int qb_sim_rir_prep(const float* h, const int64_t* offs, int64_t rows, const int32_t* on, float* hn, int64_t* win, int32_t* status,
                    void* stream);
/* add_reverberation (rir_utils.py:340-350): y_r[n] = sum_{k in [k0, k1)} h_r[k] x_r[n - k] for n < len(x_r), [k0, k1) = win[r] or the
 * whole h_r when win is NULL (estimate_early_rir's zeroed RIR is the window); rows off copy x.  y != x. */
int qb_sim_convolve(const float* x, const int64_t* offs, int64_t rows, int64_t max_len, const float* h, const int64_t* h_offs,
                    const int64_t* win, const int32_t* on, float* y, void* stream);
/* bandwidth_limitation (simulate.py:33-52) in place on rows with on[r] and fs_new[r] in {4000, 8000}: 16 kHz -> fs_new -> 16 kHz,
 * cut to the row's length, with torchaudio's sinc_interp_hann taps (soxr_hq in the reference): down taps [kd] with `wd` leading
 * zeros of padding, up taps [o, ku] with `wu`.  tmp: a buffer packed as x. */
int qb_sim_bandwidth(float* x, const int64_t* offs, int64_t rows, int64_t max_len, const int32_t* fs_new, const int32_t* on,
                     const float* down4, const float* down2, int32_t kd4, int32_t wd4, int32_t kd2, int32_t wd2, const float* up4,
                     const float* up2, int32_t ku, int32_t wu, float* tmp, void* stream);
/* clipping (simulate.py:55-76) in place on rows with on[r]: np.quantile(x_r, q[r, 0:2]) ('linear', evaluated in fp64 from exact order
 * statistics found by radix select -> stats [rows, 4] fp32), np.clip in fp64, rounded once to fp32. */
int qb_sim_clip(float* x, const int64_t* offs, int64_t rows, int64_t max_len, const double* q, const int32_t* on, float* stats,
                void* stream);
/* packet_loss (simulate.py:115-123): x_{lost_row[i]}[lost[i] * packet .. (lost[i] + 1) * packet) = 0 for i < n_lost. */
int qb_sim_packet_loss(float* x, const int64_t* offs, const int64_t* lost, const int32_t* lost_row, int64_t n_lost, int32_t packet,
                       void* stream);
/* simulate.py:181-190 then data_module.py:217-229: the 0.99 peak rule over noisy / speech / interf, the cut at cut_off[r] (wrap
 * padding when < 0) to `cut` samples, and normalize_src_tgt (has_interf 0) or normalize_mix_speech_inferf with the host uniform
 * norm_r[r] -> out_mix, out_speech, out_interf (NULL: not written) [rows, cut]. */
int qb_sim_finish(const float* noisy, const float* speech, const float* interf, const int64_t* offs, int64_t rows, const int32_t* has_interf,
                  const int64_t* cut_off, const double* norm_r, int64_t cut, float* out_mix, float* out_speech, float* out_interf,
                  void* stream);
/* data_module.py:231-233: enrollment cut at cut_off[r] (wrap padding when < 0) to `cut` samples, e / (max|e| + 1e-5) * 0.99. */
int qb_sim_enroll(const float* e, const int64_t* offs, int64_t rows, const int64_t* cut_off, int64_t cut, float* out, void* stream);

/* ResidualVQ (third-party vector_quantize_pytorch; call sites vq/codec.py:81-82,94-95): codebooks [nq, K, D] fp32. */
int qb_rvq_load(qb_handle* h, const float* codebooks, int32_t nq, int32_t K, int32_t D, qb_rvq** out);
void qb_rvq_free(qb_rvq* q);
/* x [M, D] fp32 -> idx [M, nq] int64 (+ quantized [M, D] or NULL) */
int qb_rvq_encode_rows(qb_rvq* q, const float* x, int64_t M, int64_t* idx, float* quantized_or_null, void* stream);
/* idx [M, nq] int64 -> out [M, D] fp32 (sum over layers, q = 0..nq-1 in order) */
int qb_rvq_decode_rows(qb_rvq* q, const int64_t* idx, int64_t M, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QUARK_B200_H_ */
