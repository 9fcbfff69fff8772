// BiCodec global (speaker) tokens: what is not a contraction on the path
//   ref_wav -> MelSpectrogram -> ECAPA-TDNN latent -> PerceiverResampler -> residual FSQ indices
// (QuarkAudio-UniSE/model/bicodec/bicodec.py:174-178, 201-221; modules/speaker/*.py; modules/fsq/*.py).
// Every convolution and linear of the path is a qb_gemm (3-term split); these kernels frame and take the magnitude of the
// spectrum around the two-stage DFT GEMMs, form the Res2Net sums, compute squeeze-excitation, run the perceiver's cross
// attention and GEGLU, and quantise; the ASTP kernels pool the ECAPA latent into the x-vector's statistics (ecapa_tdnn.py:195-210).
// fp32 arithmetic, except the fp64 time sums of the SE mean and the pooling; deterministic: no atomics, fixed reduction orders.
#include <atomic>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

#define QB_LAUNCH_END()              \
  g_launches++;                      \
  QB_CHECK_CUDA(cudaGetLastError()); \
  return 0

__device__ __forceinline__ void put_planes(__half* hi, __half* lo, long long o, float v) {
  __half h, l;
  split_f16(v, h, l);
  hi[o] = h;
  if (lo) lo[o] = l;
}

static unsigned grid_for(long long total) {
  const long long g = ceil_div(total, 256);
  return (unsigned)(g < 132 * 32 ? g : 132 * 32);
}

// torch.stft(center=True, pad_mode="reflect") framing for the two-stage DFT (layout of qb_stft_gather): row (clip, f, b), column
// a < P holds xpad[hop f + Q a + b] * window[Q a + b] with xpad[i] = x[reflect(i - n_fft / 2)]; columns P..63 are zero.
__global__ void mel_gather_kernel(const float* __restrict__ wav, long long L, int hop, int n_fft, int P, int Q, int F,
                                  const float* __restrict__ win, __half* __restrict__ hi, __half* __restrict__ lo, long long total) {
  const long long half = n_fft / 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int a = (int)(i & 63);
    const long long row = i >> 6;
    const int b = (int)(row % Q);
    const long long cf = row / Q;
    const int f = (int)(cf % F);
    const long long clip = cf / F;
    float v = 0.f;
    if (a < P) {
      const int s = Q * a + b;
      const float w = win[s];
      if (w != 0.f) {
        long long j = (long long)hop * f + s - half;
        if (j < 0) j = -j;
        if (j >= L) j = 2 * (L - 1) - j;
        v = wav[clip * L + j] * w;
      }
    }
    put_planes(hi, lo, i, v);
  }
}

// |X[k]| (k < nf; X[k] at row k % P, column pair k / P of the second DFT stage) -> planes [M, ld], zero beyond nf.  The imaginary
// parts of DC and Nyquist are exactly zero in a real FFT; the GEMM leaves rounding residue there, so they are dropped.
__global__ void spec_mag_kernel(const float* __restrict__ X, long long ldX, int nf, int P, __half* __restrict__ hi,
                                __half* __restrict__ lo, long long ld) {
  const long long m = blockIdx.x;
  const float* xr = X + m * P * ldX;
  for (int k = threadIdx.x; k < ld; k += blockDim.x) {
    float v = 0.f;
    if (k < nf) {
      const float* p = xr + (long long)(k % P) * ldX + 2 * (k / P);
      v = (k == 0 || k == nf - 1) ? fabsf(p[0]) : hypotf(p[0], p[1]);
    }
    put_planes(hi, lo, m * ld + k, v);
  }
}

__global__ void add_planes_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ y, long long ldy, int T,
                                  int C, __half* __restrict__ hi, __half* __restrict__ lo, long long ld, long long rpb,
                                  long long off) {
  const long long r = blockIdx.x;               // b * T + t
  const long long b = r / T, t = r % T;
  const long long o = (b * rpb + off + t) * ld;
  for (int c = threadIdx.x; c < ld; c += blockDim.x) {
    float v = 0.f;
    if (c < C) {
      v = x[r * ldx + c];
      if (y) v += y[r * ldy + c];
    }
    put_planes(hi, lo, o + c, v);
  }
}

// SE_Connect (ecapa_tdnn.py:116-129) up to the gate: s[b, :] = sigmoid(W2 relu(W1 mean_t z[b, t, :] + b1) + b2).  One block per
// clip; the time mean is a sequential fp64 sum per channel (fixed order), the two linears are warp dot products in fp32.
__global__ void se_gate_kernel(const float* __restrict__ z, int T, int C, const float* __restrict__ w1, const float* __restrict__ b1,
                               int R, const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ s) {
  extern __shared__ float sm[];
  float* mean = sm;
  float* h = sm + C;
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float* zb = z + (long long)b * T * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double acc = 0.0;
    for (int t = 0; t < T; ++t) acc += zb[(long long)t * C + c];
    mean[c] = (float)(acc / T);
  }
  __syncthreads();
  for (int r = warp; r < R; r += nw) {
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) acc = fmaf(w1[(long long)r * C + c], mean[c], acc);
    acc = warp_sum(acc) + b1[r];
    if (lane == 0) h[r] = acc > 0.f ? acc : 0.f;
  }
  __syncthreads();
  for (int c = warp; c < C; c += nw) {
    float acc = 0.f;
    for (int r = lane; r < R; r += 32) acc = fmaf(w2[(long long)c * R + r], h[r], acc);
    acc = warp_sum(acc) + b2[c];
    if (lane == 0) s[(long long)b * C + c] = sigmoid_acc(acc);
  }
}

// SE_Res2Block's tail (ecapa_tdnn.py:127,150): out = x + z * s[b, c], rounded as the reference rounds it (product, then sum).
__global__ void se_apply_kernel(const float* __restrict__ z, const float* __restrict__ s, const float* __restrict__ x, int T, int C,
                                float* __restrict__ out, __half* __restrict__ hi, __half* __restrict__ lo, long long ld,
                                long long col_off) {
  const long long r = blockIdx.x;
  const long long b = r / T;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = __fadd_rn(x[r * C + c], __fmul_rn(z[r * C + c], s[b * C + c]));
    if (out) out[r * C + c] = v;
    if (hi) put_planes(hi, lo, r * ld + col_off + c, v);
  }
}

// GEGLU (perceiver_encoder.py:232-235): x, gate = h.chunk(2); gelu(gate) * x with the exact erf -> planes, zero past inner
__global__ void geglu_planes_kernel(const float* __restrict__ h, int inner, __half* __restrict__ hi, __half* __restrict__ lo,
                                    long long ld) {
  const long long r = blockIdx.x;
  const float* hr = h + r * 2 * inner;
  for (int c = threadIdx.x; c < ld; c += blockDim.x) put_planes(hi, lo, r * ld + c, c < inner ? gelu_erf(hr[inner + c]) * hr[c] : 0.f);
}

// Non-causal cross attention, head_dim 64, fp32 throughout (perceiver_encoder.py:135-178, the non-flash Attend path): one warp per
// (clip, head, query); scores of all keys kept in shared memory, softmax with the maximum subtracted, then the value sum.
constexpr int XATT_WARPS = 4;
__global__ void cross_attention_kernel(const float* __restrict__ q, const float* __restrict__ kv, int Nq, int Nk, int H,
                                       __half* __restrict__ hi, __half* __restrict__ lo) {
  extern __shared__ float sc_all[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * XATT_WARPS + warp, h = blockIdx.y, b = blockIdx.z;
  if (i >= Nq) return;
  float* sc = sc_all + (long long)warp * Nk;
  const int D = H * 64;
  const float* qr = q + ((long long)b * Nq + i) * D + h * 64;
  const float q0 = qr[2 * lane], q1 = qr[2 * lane + 1];
  const float* kb = kv + (long long)b * Nk * 2 * D + h * 64;
  const float* vb = kb + D;
  float mx = -INFINITY;
  for (int j = 0; j < Nk; ++j) {
    const float2 k = *reinterpret_cast<const float2*>(kb + (long long)j * 2 * D + 2 * lane);
    const float d = warp_sum(fmaf(q0, k.x, q1 * k.y)) * 0.125f;      // dim_head ** -0.5
    mx = fmaxf(mx, d);
    if (lane == 0) sc[j] = d;
  }
  __syncwarp();
  float sum = 0.f;
  for (int j = lane; j < Nk; j += 32) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float o0 = 0.f, o1 = 0.f;
  for (int j = 0; j < Nk; ++j) {
    const float p = sc[j];
    const float2 v = *reinterpret_cast<const float2*>(vb + (long long)j * 2 * D + 2 * lane);
    o0 = fmaf(p, v.x, o0);
    o1 = fmaf(p, v.y, o1);
  }
  const long long o = ((long long)b * Nq + i) * D + h * 64 + 2 * lane;
  put_planes(hi, lo, o, o0 / sum);
  put_planes(hi, lo, o + 1, o1 / sum);
}

struct FsqLevels {
  int n;
  int L[8];
};

// PerceiverResampler's final RMSNorm (perceiver_encoder.py:195-214) + ResidualFSQ with one quantizer (residual_fsq.py:158-252,
// finite_scalar_quantization.py:126-157): one warp per latent row.
__global__ void fsq_tokenize_kernel(const float* __restrict__ x, long long rows, int dim, const float* __restrict__ gamma,
                                    const float* __restrict__ w_in, const float* __restrict__ b_in, const FsqLevels lv,
                                    int32_t* __restrict__ idx, float* __restrict__ z_out, float* __restrict__ xn_out) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * dim;
  float ss = 0.f;
  for (int c = lane; c < dim; c += 32) ss = fmaf(xr[c], xr[c], ss);
  const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);           // F.normalize
  const float scale = sqrtf((float)dim);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int c = lane; c < dim; c += 32) {
    const float v = (xr[c] / nrm) * scale * gamma[c];
    if (xn_out) xn_out[row * dim + c] = v;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < lv.n) acc[j] = fmaf(w_in[(long long)j * dim + c], v, acc[j]);
  }
  // The index is built in integers: sum_j (q_j + L_j / 2) * prod_{i<j} L_i, exact for any codebook up to 2^24 entries, and the
  // index indices_to_level_indices() inverts.  The reference's float steps (codes_to_indices(): code = q / hw, then
  // (code * hw + hw) * basis, truncated) give the same integer for every level up to 25, but only when each op is rounded on its
  // own: contracted into FMAs, fl(-2/3) * 3 + 3 is 0.99999994 and truncation loses one (levels 6 and 7).  From level 26 on even
  // the unfused terms stop being exact integers (fl(-7/13) * 13 + 13 = 5.9999995); the kernel still gives the exact index.
  int index = 0, basis = 1;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j >= lv.n) break;
    const float zj = warp_sum(acc[j]) + b_in[j];
    if (z_out && lane == 0) z_out[row * lv.n + j] = zj;
    const int L = lv.L[j];
    const float half_l = (float)(L - 1) * 1.001f / 2.f;            // bound(): (levels - 1) * (1 + eps) / 2
    const float offset = (L % 2 == 0) ? 0.5f : 0.f;
    const float shift = atanhf(offset / half_l);
    const float q = rintf(tanhf(zj + shift) * half_l - offset);     // torch.round: half to even
    index += ((int)q + L / 2) * basis;
    basis *= L;
  }
  if (lane == 0) idx[row] = index;
}

// ASTP with global context (pooling_layers.py:119-144), the x-vector branch of ECAPA_TDNN.forward (ecapa_tdnn.py:195-210).  One
// thread per (clip, channel), channels on threadIdx so that every frame's read is coalesced; each thread walks the T frames of its
// channel in order with fp64 accumulators, so the result does not depend on the launch shape and no atomics are used.
constexpr int ASP_THREADS = 128;

// context: mean_c and sqrt(var_c + 1e-7) with torch.var's unbiased divisor T - 1 (two passes: the mean, then the squared deviations)
__global__ void asp_context_kernel(const float* __restrict__ x, int T, int C, float* __restrict__ out, __half* __restrict__ hi,
                                   __half* __restrict__ lo, long long ld) {
  const int c = blockIdx.x * ASP_THREADS + threadIdx.x, b = blockIdx.y;
  if (c >= C) return;
  const float* xc = x + (long long)b * T * C + c;
  double s = 0.0;
  for (int t = 0; t < T; ++t) s += (double)xc[(long long)t * C];
  const double mean = s / T;
  double q = 0.0;
  for (int t = 0; t < T; ++t) {
    const double d = (double)xc[(long long)t * C] - mean;
    q = fma(d, d, q);
  }
  const float m = (float)mean, sd = (float)sqrt(q / (T - 1) + 1e-7);
  out[(long long)b * 2 * C + c] = m;
  out[(long long)b * 2 * C + C + c] = sd;
  put_planes(hi, lo, b * ld + c, m);
  put_planes(hi, lo, b * ld + C + c, sd);
}

// tanh(h[b*T + t, n] + row[b, n]) -> planes [B*T, ld], zero past N: linear1's x part (a GEMM over the frames) plus its context
// part and bias (one row per clip), then the tanh (pooling_layers.py:138-139)
__global__ void asp_tanh_planes_kernel(const float* __restrict__ h, const float* __restrict__ row, int T, int N, __half* __restrict__ hi,
                                       __half* __restrict__ lo, long long ld) {
  const long long r = blockIdx.x;
  const float* hr = h + r * N;
  const float* rr = row + (r / T) * N;
  for (int n = threadIdx.x; n < ld; n += blockDim.x) put_planes(hi, lo, r * ld + n, n < N ? tanhf(hr[n] + rr[n]) : 0.f);
}

// attentive statistics (pooling_layers.py:140-143): alpha = softmax over T of the logits (maximum subtracted), mean = sum alpha x,
// std = sqrt(max(sum alpha x^2 - mean^2, 1e-7)); exponentials and sums in fp64
__global__ void asp_pool_kernel(const float* __restrict__ x, const float* __restrict__ logits, int T, int C, float* __restrict__ out,
                                __half* __restrict__ hi, __half* __restrict__ lo, long long ld) {
  const int c = blockIdx.x * ASP_THREADS + threadIdx.x, b = blockIdx.y;
  if (c >= C) return;
  const long long base = (long long)b * T * C + c;
  float mx = -INFINITY;
  for (int t = 0; t < T; ++t) mx = fmaxf(mx, logits[base + (long long)t * C]);
  double se = 0.0, s1 = 0.0, s2 = 0.0;
  for (int t = 0; t < T; ++t) {
    const double e = exp((double)logits[base + (long long)t * C] - (double)mx);
    const double v = (double)x[base + (long long)t * C];
    se += e;
    s1 = fma(e, v, s1);
    s2 = fma(e * v, v, s2);
  }
  const double mean = s1 / se, var = s2 / se - mean * mean;
  const float m = (float)mean, sd = (float)sqrt(fmax(var, 1e-7));
  out[(long long)b * 2 * C + c] = m;
  out[(long long)b * 2 * C + C + c] = sd;
  put_planes(hi, lo, b * ld + c, m);
  put_planes(hi, lo, b * ld + C + c, sd);
}

}  // namespace qb
using namespace qb;

extern "C" int qb_mel_gather(const float* wav, int64_t B, int64_t L, int32_t hop, int32_t n_fft, int32_t P, int32_t Q, const float* window,
                             qb_half* hi, qb_half* lo, void* stream) {
  QB_REQUIRE(wav && window && hi && B >= 1 && hop >= 1 && P * Q == n_fft && P <= 64 && 2 * Q <= 128 && n_fft % 2 == 0,
             "mel_gather: needs n_fft == P*Q, P <= 64, Q <= 64");
  QB_REQUIRE(L > n_fft / 2, "mel_gather: reflect padding of n_fft / 2 = %d needs more than that many samples (got %lld)", n_fft / 2,
             (long long)L);
  const int64_t F = 1 + L / hop;
  const long long total = B * F * Q * 64;
  mel_gather_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(wav, L, hop, n_fft, P, Q, (int)F, window, (__half*)hi,
                                                                       (__half*)lo, total);
  QB_LAUNCH_END();
}

extern "C" int qb_spec_magnitude(const float* X, int64_t ldX, int64_t M, int32_t nf, int32_t P, qb_half* hi, qb_half* lo, int64_t ld,
                                 void* stream) {
  QB_REQUIRE(X && hi && M >= 1 && nf >= 2 && nf <= ld && P >= 1 && ldX >= 2 * ((nf - 1) / P + 1), "spec_magnitude: bad args");
  spec_mag_kernel<<<(unsigned)M, 256, 0, (cudaStream_t)stream>>>(X, ldX, nf, P, (__half*)hi, (__half*)lo, ld);
  QB_LAUNCH_END();
}

extern "C" int qb_add_planes(const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t B, int64_t T, int64_t C, qb_half* hi,
                             qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream) {
  QB_REQUIRE(x && hi && B >= 1 && T >= 1 && C >= 1 && C <= ld && ldx >= C && (!y || ldy >= C) && row_off + T <= rows_per_batch,
             "add_planes: bad args");
  add_planes_kernel<<<(unsigned)(B * T), 64, 0, (cudaStream_t)stream>>>(x, ldx, y, ldy, (int)T, (int)C, (__half*)hi, (__half*)lo, ld,
                                                                       rows_per_batch, row_off);
  QB_LAUNCH_END();
}

extern "C" int qb_se_gate(const float* z, int64_t B, int64_t T, int32_t C, const float* w1, const float* b1, int32_t R, const float* w2,
                          const float* b2, float* s, void* stream) {
  QB_REQUIRE(z && w1 && b1 && w2 && b2 && s && B >= 1 && T >= 1 && C >= 1 && R >= 1 && (size_t)(C + R) * 4 <= 48 * 1024,
             "se_gate: bad args");
  se_gate_kernel<<<(unsigned)B, 512, (C + R) * 4, (cudaStream_t)stream>>>(z, (int)T, C, w1, b1, R, w2, b2, s);
  QB_LAUNCH_END();
}

extern "C" int qb_se_apply(const float* z, const float* s, const float* x, int64_t B, int64_t T, int32_t C, float* out, qb_half* hi,
                           qb_half* lo, int64_t ld, int64_t col_off, void* stream) {
  QB_REQUIRE(z && s && x && (out || hi) && B >= 1 && T >= 1 && C >= 1 && (!hi || col_off + C <= ld), "se_apply: bad args");
  se_apply_kernel<<<(unsigned)(B * T), 256, 0, (cudaStream_t)stream>>>(z, s, x, (int)T, C, out, (__half*)hi, (__half*)lo, ld, col_off);
  QB_LAUNCH_END();
}

extern "C" int qb_geglu_planes(const float* h, int64_t rows, int32_t inner, qb_half* hi, qb_half* lo, int64_t ld, void* stream) {
  QB_REQUIRE(h && hi && rows >= 1 && inner >= 1 && inner <= ld, "geglu_planes: bad args");
  geglu_planes_kernel<<<(unsigned)rows, 128, 0, (cudaStream_t)stream>>>(h, inner, (__half*)hi, (__half*)lo, ld);
  QB_LAUNCH_END();
}

extern "C" int qb_cross_attention(const float* q, const float* kv, int64_t B, int64_t Nq, int64_t Nk, int32_t heads, qb_half* out_hi,
                                  qb_half* out_lo, void* stream) {
  QB_REQUIRE(q && kv && out_hi && B >= 1 && Nq >= 1 && Nk >= 1 && heads >= 1, "cross_attention: bad args");
  QB_REQUIRE((size_t)XATT_WARPS * Nk * 4 <= 48 * 1024, "cross_attention: at most %d keys (got %lld)", 48 * 1024 / (4 * XATT_WARPS),
             (long long)Nk);
  dim3 grid((unsigned)ceil_div(Nq, XATT_WARPS), (unsigned)heads, (unsigned)B);
  cross_attention_kernel<<<grid, 32 * XATT_WARPS, XATT_WARPS * Nk * 4, (cudaStream_t)stream>>>(q, kv, (int)Nq, (int)Nk, heads,
                                                                                                (__half*)out_hi, (__half*)out_lo);
  QB_LAUNCH_END();
}

extern "C" int qb_fsq_tokenize(const float* x, int64_t rows, int32_t dim, const float* gamma, const float* w_in, const float* b_in,
                               int32_t n_levels, const int32_t* levels, int32_t num_quantizers, int32_t* idx, float* z, float* xn,
                               void* stream) {
  QB_REQUIRE(num_quantizers == 1, "fsq_tokenize: residual FSQ with %d quantizers (one is supported, as on the detokenize side)",
             num_quantizers);
  QB_REQUIRE(x && gamma && w_in && b_in && levels && idx && rows >= 1 && dim >= 1 && n_levels >= 1 && n_levels <= 8,
             "fsq_tokenize: bad args (at most 8 levels)");
  FsqLevels lv{};
  lv.n = n_levels;
  double cb = 1.0;
  for (int j = 0; j < n_levels; ++j) {
    QB_REQUIRE(levels[j] >= 2, "fsq_tokenize: levels must be >= 2");
    lv.L[j] = levels[j];
    cb *= levels[j];
  }
  QB_REQUIRE(cb <= (double)(1 << 24), "fsq_tokenize: codebook larger than 2^24 entries");
  fsq_tokenize_kernel<<<(unsigned)ceil_div(rows, 8), 256, 0, (cudaStream_t)stream>>>(x, rows, dim, gamma, w_in, b_in, lv, idx, z, xn);
  QB_LAUNCH_END();
}

extern "C" int qb_asp_context(const float* x, int64_t B, int64_t T, int32_t C, float* out, qb_half* hi, qb_half* lo, int64_t ld,
                              void* stream) {
  QB_REQUIRE(x && out && hi && B >= 1 && C >= 1 && 2 * (int64_t)C <= ld, "asp_context: bad args (ld must hold 2 C columns)");
  QB_REQUIRE(T >= 2 && T <= INT32_MAX, "asp_context: the unbiased variance needs T >= 2 frames (got %lld)", (long long)T);
  asp_context_kernel<<<dim3((unsigned)ceil_div(C, ASP_THREADS), (unsigned)B), ASP_THREADS, 0, (cudaStream_t)stream>>>(
      x, (int)T, C, out, (__half*)hi, (__half*)lo, ld);
  QB_LAUNCH_END();
}

extern "C" int qb_asp_tanh_planes(const float* h, const float* row, int64_t B, int64_t T, int32_t N, qb_half* hi, qb_half* lo, int64_t ld,
                                  void* stream) {
  QB_REQUIRE(h && row && hi && B >= 1 && T >= 1 && T <= INT32_MAX && N >= 1 && N <= ld, "asp_tanh_planes: bad args");
  asp_tanh_planes_kernel<<<(unsigned)(B * T), 128, 0, (cudaStream_t)stream>>>(h, row, (int)T, N, (__half*)hi, (__half*)lo, ld);
  QB_LAUNCH_END();
}

extern "C" int qb_asp_pool(const float* x, const float* logits, int64_t B, int64_t T, int32_t C, float* out, qb_half* hi, qb_half* lo,
                           int64_t ld, void* stream) {
  QB_REQUIRE(x && logits && out && hi && B >= 1 && T >= 1 && T <= INT32_MAX && C >= 1 && 2 * (int64_t)C <= ld,
             "asp_pool: bad args (ld must hold 2 C columns)");
  asp_pool_kernel<<<dim3((unsigned)ceil_div(C, ASP_THREADS), (unsigned)B), ASP_THREADS, 0, (cudaStream_t)stream>>>(
      x, logits, (int)T, C, out, (__half*)hi, (__half*)lo, ld);
  QB_LAUNCH_END();
}
