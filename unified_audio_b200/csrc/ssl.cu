// SSL feature front end kernels (SURVEY.md 8f.2 / 8f.3): the pieces of HuBERT-base / WavLM-base-plus that are not dense
// contractions, and the caller-side glue of the tokenizers.
//   HCodecTokenizer.extract_ssl_features   QuarkAudio-HCodec/HCodec-2.0/audio_tokenizer.py:47-61
//   Model.extract_semantic_features        QuarkAudio-UniSE/model/model.py:38-51
//   transformers HubertFeatureEncoder layer 0 (Conv1d(1, 512, k=10, s=5, bias=False) -> GroupNorm(512 groups) -> GELU)
//   Wav2Vec2FeatureExtractor(do_normalize=True) and Wav2Vec2 (feat_extract_norm="layer") layer 0: Conv1d(1, 512, k=10, s=5) + bias;
//   its LayerNorm over channels + GELU is qb_layernorm_act (elementwise.cu)
// Everything else of the encoders runs on the wgmma GEMM / attention / LayerNorm ops of this library
// (unified_audio_b200/ssl.py).
#include <atomic>
#include <cstdio>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

// ---- conv layer 0: one input channel.  Block = SSL_TT output frames x all C channels; thread c keeps w[c][0..k) in registers;
// writes y [B, T0, C] fp32 (channel-last, coalesced over c), plus bias[c] when given, and (part != NULL) fp64 per-(block, channel)
// partial sums for the per-channel GroupNorm over time (deterministic: partials are reduced in a fixed order by ssl_gn_stats_kernel).
constexpr int SSL_TT = 64, SSL_KMAX = 16;
__global__ void __launch_bounds__(512)
ssl_conv0_kernel(const float* __restrict__ x, long long x_stride, int T_in, const float* __restrict__ w, const float* __restrict__ bias,
                 int C, int k, int s, int T0, float* __restrict__ y, double* __restrict__ part) {
  extern __shared__ float xs[];                         // (SSL_TT - 1) * s + k input samples
  const int b = blockIdx.y, t0 = blockIdx.x * SSL_TT;
  const int nt = min(SSL_TT, T0 - t0), need = (nt - 1) * s + k;
  for (int i = threadIdx.x; i < need; i += blockDim.x) {
    const int src = t0 * s + i;
    xs[i] = src < T_in ? x[(long long)b * x_stride + src] : 0.f;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float wr[SSL_KMAX];
#pragma unroll
    for (int j = 0; j < SSL_KMAX; ++j) wr[j] = j < k ? w[c * k + j] : 0.f;
    const float b0 = bias ? bias[c] : 0.f;
    double sum = 0.0, sq = 0.0;
    for (int t = 0; t < nt; ++t) {
      float acc = b0;
#pragma unroll
      for (int j = 0; j < SSL_KMAX; ++j)
        if (j < k) acc = fmaf(wr[j], xs[t * s + j], acc);
      y[((long long)b * T0 + t0 + t) * C + c] = acc;
      sum += acc;
      sq += (double)acc * acc;
    }
    if (part) {
      double* p = part + (((long long)b * gridDim.x + blockIdx.x) * C + c) * 2;
      p[0] = sum; p[1] = sq;
    }
  }
}
__global__ void ssl_gn_stats_kernel(const double* __restrict__ part, int nblk, int C, int T0, float eps, float* __restrict__ stats) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (c >= C) return;
  double S = 0.0, Q = 0.0;
  for (int i = 0; i < nblk; ++i) {
    const double* p = part + (((long long)b * nblk + i) * C + c) * 2;
    S += p[0]; Q += p[1];
  }
  const double mean = S / T0;
  double var = Q / T0 - mean * mean;
  if (var < 0) var = 0;
  stats[((long long)b * C + c) * 2] = (float)mean;
  stats[((long long)b * C + c) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
}
// per-channel GroupNorm apply + exact (erf) GELU -> planes of the next conv's channel-last buffer
__global__ void ssl_gn_gelu_kernel(const float* __restrict__ y, const float* __restrict__ stats, const float* __restrict__ gw,
                                   const float* __restrict__ gb, long long T0, int C, __half* __restrict__ hi, __half* __restrict__ lo,
                                   long long ld, long long rpb, long long off, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long t = (i / C) % T0, b = i / ((long long)C * T0);
    const float* st = stats + (b * C + c) * 2;
    const float v = gelu_erf((y[i] - st[0]) * st[1] * gw[c] + gb[c]);
    __half h, l;
    split_f16(v, h, l);
    const long long o = (b * rpb + off + t) * ld + c;
    hi[o] = h;
    if (lo) lo[o] = l;
  }
}

// ---- Wav2Vec2FeatureExtractor.zero_mean_unit_var_norm: one block per utterance, two-pass fp64 statistics (population variance)
// reduced in a fixed order, out = (x - mean) / sqrt(var + eps) rounded once to fp32.
constexpr int WN_THREADS = 1024;
__device__ double block_sum_f64(double v, double* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[wid] = v;
  __syncthreads();
  double t = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
  __syncthreads();
  return t;
}
__global__ void __launch_bounds__(WN_THREADS)
wav_normalize_kernel(const float* __restrict__ x, long long T, double eps, float* __restrict__ out) {
  __shared__ double red[WN_THREADS / 32];
  const float* xb = x + (long long)blockIdx.x * T;
  float* ob = out + (long long)blockIdx.x * T;
  double s = 0.0;
  for (long long i = threadIdx.x; i < T; i += blockDim.x) s += xb[i];
  const double mean = block_sum_f64(s, red) / (double)T;
  double q = 0.0;
  for (long long i = threadIdx.x; i < T; i += blockDim.x) { const double d = xb[i] - mean; q += d * d; }
  const double inv = 1.0 / sqrt(block_sum_f64(q, red) / (double)T + eps);
  for (long long i = threadIdx.x; i < T; i += blockDim.x) ob[i] = (float)((xb[i] - mean) * inv);
}

// out (+)= scale * x  (running mean of the encoder's hidden states, audio_tokenizer.py:55)
__global__ void axpy_kernel(const float* __restrict__ x, float scale, long long n, int accumulate, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = accumulate ? fmaf(scale, x[i], out[i]) : scale * x[i];
}
// mean [B, T, C] -> sign(x) * |x| ** p (audio_tokenizer.py:57-60; p <= 0: identity) written channel-first [B, C, T] (the layout
// Codec.encode takes) or channel-last
__global__ void ssl_compress_kernel(const float* __restrict__ x, long long T, int C, float p, int channel_first, long long total,
                                    float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long t = (i / C) % T, b = i / ((long long)C * T);
    float v = x[i];
    if (p > 0.f) {
      // reference: symbol = (x > 0) * 2 - 1 (so x == 0 -> -1 * 0 ** 0.3 = -0.0); magnitude = |x| ** 0.3
      const float m = powf(fabsf(v), p);
      v = v > 0.f ? m : -m;
    }
    out[channel_first ? (b * C + c) * T + t : i] = v;
  }
}
// pad_wav (audio_tokenizer.py:63-66) / F.pad(wavs, (160, 160)) (:51) / wrap padding of UniSE segments (U/model/model.py:175-181):
// out[b, i] = in[b, (i - left) (mod T_in if wrap)] or 0 outside
__global__ void pad_wav_kernel(const float* __restrict__ x, long long T_in, long long left, long long T_out, int wrap,
                               float* __restrict__ out, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / T_out, j = i % T_out - left;
    float v = 0.f;
    if (j >= 0 && j < T_in) v = x[b * T_in + j];
    else if (wrap && T_in > 0) { long long m = j % T_in; if (m < 0) m += T_in; v = x[b * T_in + m]; }
    out[i] = v;
  }
}
static inline unsigned ssl_grid(long long total) {
  long long g = (total + 255) / 256;
  return (unsigned)(g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g));
}
}  // namespace qb
using namespace qb;

extern "C" int64_t qb_ssl_conv0_workspace_bytes(int64_t B, int64_t T0, int32_t C) {
  return (B * ceil_div(T0, SSL_TT) * C * 2) * 8 + B * C * 2 * 4;
}

extern "C" int qb_ssl_conv0_gn_gelu(const float* x, int64_t B, int64_t T_in, const float* w, int32_t C, int32_t k, int32_t stride,
                                    const float* gn_w, const float* gn_b, float eps, float* y_scratch, void* workspace, qb_half* hi,
                                    qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(x && w && gn_w && gn_b && y_scratch && workspace && hi, "ssl_conv0: bad args");
  QB_REQUIRE(k >= 1 && k <= SSL_KMAX && stride >= 1 && T_in >= k, "ssl_conv0: kernel size %d unsupported (<= %d)", k, SSL_KMAX);
  const int64_t T0 = (T_in - k) / stride + 1;
  QB_REQUIRE(C <= ld && row_off + T0 <= rows_per_batch, "ssl_conv0: plane buffer too small");
  const int nblk = (int)ceil_div(T0, SSL_TT);
  double* part = (double*)workspace;
  float* stats = (float*)((uint8_t*)workspace + (size_t)B * nblk * C * 2 * 8);
  dim3 grid((unsigned)nblk, (unsigned)B);
  const size_t smem = ((size_t)(SSL_TT - 1) * stride + k) * 4;
  ssl_conv0_kernel<<<grid, 512, smem, st>>>(x, T_in, (int)T_in, w, nullptr, C, k, stride, (int)T0, y_scratch, part);
  ssl_gn_stats_kernel<<<dim3((unsigned)ceil_div(C, 128), (unsigned)B), 128, 0, st>>>(part, nblk, C, (int)T0, eps, stats);
  const long long total = B * T0 * C;
  ssl_gn_gelu_kernel<<<ssl_grid(total), 256, 0, st>>>(y_scratch, stats, gn_w, gn_b, T0, C, (__half*)hi, (__half*)lo, ld, rows_per_batch,
                                                     row_off, total);
  g_launches += 3;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_ssl_conv0_bias(const float* x, int64_t B, int64_t T_in, const float* w, const float* bias, int32_t C, int32_t k,
                                 int32_t stride, float* y, void* stream) {
  QB_REQUIRE(x && w && bias && y && B >= 1 && C >= 1, "ssl_conv0_bias: bad args");
  QB_REQUIRE(k >= 1 && k <= SSL_KMAX && stride >= 1 && T_in >= k, "ssl_conv0_bias: kernel size %d unsupported (<= %d)", k, SSL_KMAX);
  const int64_t T0 = (T_in - k) / stride + 1;
  dim3 grid((unsigned)ceil_div(T0, SSL_TT), (unsigned)B);
  const size_t smem = ((size_t)(SSL_TT - 1) * stride + k) * 4;
  ssl_conv0_kernel<<<grid, 512, smem, (cudaStream_t)stream>>>(x, T_in, (int)T_in, w, bias, C, k, stride, (int)T0, y, nullptr);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_wav_normalize(const float* x, int64_t B, int64_t T, float eps, float* out, void* stream) {
  QB_REQUIRE(x && out && B >= 0 && T >= 1, "wav_normalize: bad args");
  if (B == 0) return 0;
  wav_normalize_kernel<<<(unsigned)B, WN_THREADS, 0, (cudaStream_t)stream>>>(x, T, (double)eps, out);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_axpy(const float* x, float scale, int64_t n, int32_t accumulate, float* out, void* stream) {
  QB_REQUIRE(x && out && n >= 0, "axpy: bad args");
  if (n == 0) return 0;
  axpy_kernel<<<ssl_grid(n), 256, 0, (cudaStream_t)stream>>>(x, scale, n, accumulate, out);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_ssl_compress(const float* x, int64_t B, int64_t T, int32_t C, float power, int32_t channel_first, float* out,
                               void* stream) {
  QB_REQUIRE(x && out, "ssl_compress: bad args");
  const long long total = B * T * C;
  if (total == 0) return 0;
  ssl_compress_kernel<<<ssl_grid(total), 256, 0, (cudaStream_t)stream>>>(x, T, C, power, channel_first, total, out);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_pad_wav(const float* x, int64_t B, int64_t T_in, int64_t left, int64_t T_out, int32_t wrap, float* out,
                          void* stream) {
  QB_REQUIRE(x && out && T_out >= 0 && T_in >= 0, "pad_wav: bad args");
  const long long total = B * T_out;
  if (total == 0) return 0;
  pad_wav_kernel<<<ssl_grid(total), 256, 0, (cudaStream_t)stream>>>(x, T_in, left, T_out, wrap, out, total);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
