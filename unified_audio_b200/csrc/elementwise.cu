// Memory-bound kernels of the H-Codec path: plane conversion, normalisations, ConvNeXt depthwise
// front half, spectral pre/post-processing.  All are HBM/L2-bound; design rules: channel-last rows,
// 128-bit vector accesses along C, one warp (or block) per row, fp32 statistics (two-pass).
#include <atomic>

#include <cstdlib>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

#define QB_LAUNCH_END()            \
  g_launches++;                    \
  QB_CHECK_CUDA(cudaGetLastError()); \
  return 0

__device__ __forceinline__ void store_planes(__half* hi, __half* lo, long long o, float v) {
  __half h, l;
  split_f16(v, h, l);
  hi[o] = h;
  if (lo) lo[o] = l;
}

// ------------------------------------------------------------------ split
__global__ void split_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) store_planes(hi, lo, i, x[i]);
}

// ------------------------------------------------------------------ rows -> planes (padded buffer)
__global__ void rows_to_planes_kernel(const float* __restrict__ x, int rows, int C, int repeat, int act,
                                      __half* __restrict__ hi, __half* __restrict__ lo, long long ld, long long rpb,
                                      long long off) {
  const int r_out = blockIdx.x, b = blockIdx.y;
  const float* src = x + ((long long)b * rows + r_out / repeat) * C;
  const long long o = ((long long)b * rpb + off + r_out) * ld;
  for (int c = threadIdx.x; c < ld; c += blockDim.x) {
    float v = c < C ? src[c] : 0.f;
    if (act == QB_ACT_ELU) v = elu_f(v);
    store_planes(hi, lo, o + c, v);
  }
}

__global__ void bct_to_planes_kernel(const float* __restrict__ x, int C, int T, __half* __restrict__ hi,
                                     __half* __restrict__ lo, long long ld, long long rpb, long long off) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t < T) ? x[((long long)b * C + c) * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < ld) store_planes(hi, lo, ((long long)b * rpb + off + t) * ld + c, c < C ? tile[threadIdx.x][i] : 0.f);
  }
}

// ------------------------------------------------------------------ LayerNorm / RMSNorm (warp per row)
// ACT = QB_ACT_GELU applies the exact GELU after the affine (wav2vec2's conv layers: conv -> LayerNorm over channels -> GELU)
template <int ACT>
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bz,
                                 float eps, long long rows_total, int rows, int C, float* __restrict__ out,
                                 __half* __restrict__ hi, __half* __restrict__ lo, long long ld, long long rpb,
                                 long long off, long long wb_bstride) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows_total) return;
  const float* xr = x + row * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
  const float mean = warp_sum(s) / C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) { float d = xr[c] - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  const long long b = row / rows, r = row % rows;
  const long long o = (b * rpb + off + r) * ld;
  w += b * wb_bstride;            // AdaLayerNorm: per-clip scale / shift rows (stride 0 = ordinary affine LayerNorm)
  bz += b * wb_bstride;
  for (int c = lane; c < C; c += 32) {
    float v = (xr[c] - mean) * rstd * w[c] + bz[c];
    if (ACT == QB_ACT_GELU) v = gelu_erf(v);
    if (out) out[row * C + c] = v;
    if (hi) store_planes(hi, lo, o + c, v);
  }
}

__global__ void rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, float eps, long long rows, int C,
                               float* __restrict__ out, __half* __restrict__ hi, __half* __restrict__ lo) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) q += xr[c] * xr[c];
  const float r = rsqrtf(warp_sum(q) / C + eps);
  for (int c = lane; c < C; c += 32) {
    const float v = xr[c] * r * w[c];
    if (out) out[row * C + c] = v;
    if (hi) store_planes(hi, lo, row * C + c, v);
  }
}

// ------------------------------------------------------------------ ConvNeXt: dwconv k7 + LayerNorm
// One warp per (b,t) row; the 7 input rows come from L1/L2 (neighbouring warps of the block share
// them).  dw_w is [C,7] as the reference stores it (conv.weight[C,1,7]).
__global__ void dwconv7_ln_kernel(const float* __restrict__ x, const float* __restrict__ dw_w,
                                  const float* __restrict__ dw_b, const float* __restrict__ ln_w,
                                  const float* __restrict__ ln_b, int T, int C, long long rows_total,
                                  __half* __restrict__ hi, __half* __restrict__ lo, long long ln_bstride) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + wi;
  if (row >= rows_total) return;
  float* y = sm + (size_t)wi * C;
  const int t = (int)(row % T);
  const float* xb = x + (row - t) * C;  // start of this clip
  float s = 0.f;
  for (int c = lane; c < C; c += 32) {
    float acc = dw_b[c];
    const float* wc = dw_w + (long long)c * 7;
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      int tt = t + j - 3;
      if (tt >= 0 && tt < T) acc = fmaf(wc[j], xb[(long long)tt * C + c], acc);
    }
    y[c] = acc;
    s += acc;
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) { float d = y[c] - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum(q) / C + 1e-6f);
  ln_w += (row / T) * ln_bstride;      // per-clip scale / shift (AdaLayerNorm) when the stride is non-zero
  ln_b += (row / T) * ln_bstride;
  for (int c = lane; c < C; c += 32) store_planes(hi, lo, row * C + c, (y[c] - mean) * rstd * ln_w[c] + ln_b[c]);
}

// v2: block = (TT consecutive frames of one clip) x (all channels); one thread owns 4 channels
// (float4 along C => fully coalesced 16 B accesses) and slides a 7-row register window over time, so
// each input row is read once per block (halo re-reads hit L2).  LayerNorm statistics for the TT rows
// are block-reduced together in one round (equal-count (mean, M2) merges, see below).  <= 85 registers at 384 threads keeps
// two CTAs per SM: a 768-thread one-CTA-per-SM variant with all loads hoisted measured 1.7x SLOWER (barrier stalls idle the SM).
template <int TT, int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB)
dwconv7_ln_v2_kernel(const float4* __restrict__ x, const float* __restrict__ dw_w, const float4* __restrict__ dw_b,
                     const float4* __restrict__ ln_w, const float4* __restrict__ ln_b, int T, int C4,
                     __half* __restrict__ hi, __half* __restrict__ lo, long long ln_bstride4) {
  __shared__ float red[16][TT], red2[16][TT];
  __shared__ float tot[TT], tot2[TT];
  const int b = blockIdx.y, t0 = blockIdx.x * TT, c4 = threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  float w[28];
  {
    const float4* wp = reinterpret_cast<const float4*>(dw_w + (size_t)c4 * 28);
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      float4 v = wp[i];
      w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
    }
  }
  const float4 bias = dw_b[c4];
  const float4* xb = x + (size_t)b * T * C4 + c4;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 win[7];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const int tt = t0 - 3 + j;
    win[j] = (tt >= 0 && tt < T) ? xb[(size_t)tt * C4] : zero;
  }
  float4 y[TT];
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    const int tt = t0 + i + 3;
    win[6] = (tt < T) ? xb[(size_t)tt * C4] : zero;
    float4 a = bias;
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      a.x = fmaf(w[j], win[j].x, a.x);
      a.y = fmaf(w[7 + j], win[j].y, a.y);
      a.z = fmaf(w[14 + j], win[j].z, a.z);
      a.w = fmaf(w[21 + j], win[j].w, a.w);
    }
    y[i] = a;
#pragma unroll
    for (int j = 0; j < 6; ++j) win[j] = win[j + 1];
  }
  // LayerNorm statistics in ONE block round: every thread starts from the exact (mean, M2) of its 4 channels and
  // equal-count partials are merged pairwise (Chan et al.): m = (ma + mb)/2, M2 = M2a + M2b + (mb - ma)^2 * n/2 -
  // a centred variance (no E[x^2] - mean^2 cancellation) without a second pass over the block.
  float mean[TT], rstd[TT];
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    float m = 0.25f * ((y[i].x + y[i].y) + (y[i].z + y[i].w));
    const float dx = y[i].x - m, dy = y[i].y - m, dz = y[i].z - m, dw = y[i].w - m;
    float q = (dx * dx + dy * dy) + (dz * dz + dw * dw);
    float n_half = 2.f;                       // n/2 for partials of n = 4 values
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float mo = __shfl_xor_sync(0xffffffffu, m, o), qo = __shfl_xor_sync(0xffffffffu, q, o);
      const float d = mo - m;
      q = q + qo + d * d * n_half;
      m = 0.5f * (m + mo);
      n_half *= 2.f;
    }
    if (lane == 0) { red[warp][i] = m; red2[warp][i] = q; }
  }
  __syncthreads();
  if (threadIdx.x < TT) {                     // merge the warps' partials (128 values each) sequentially
    float m = red[0][threadIdx.x], q = red2[0][threadIdx.x], n = 128.f;
    for (int wv = 1; wv < nwarps; ++wv) {
      const float mo = red[wv][threadIdx.x], qo = red2[wv][threadIdx.x];
      const float d = mo - m, nt = n + 128.f;
      q = q + qo + d * d * (n * 128.f / nt);
      m = m + d * (128.f / nt);
      n = nt;
    }
    tot[threadIdx.x] = m;
    tot2[threadIdx.x] = rsqrtf(q / n + 1e-6f);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < TT; ++i) { mean[i] = tot[i]; rstd[i] = tot2[i]; }
  const float4 lw = ln_w[b * ln_bstride4 + c4], lb = ln_b[b * ln_bstride4 + c4];     // stride 0: static affine
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    const int t = t0 + i;
    if (t < T) {
      const float v0 = (y[i].x - mean[i]) * rstd[i] * lw.x + lb.x, v1 = (y[i].y - mean[i]) * rstd[i] * lw.y + lb.y;
      const float v2 = (y[i].z - mean[i]) * rstd[i] * lw.z + lb.z, v3 = (y[i].w - mean[i]) * rstd[i] * lw.w + lb.w;
      __half h0, h1, h2, h3, l0, l1, l2, l3;
      split_f16(v0, h0, l0); split_f16(v1, h1, l1); split_f16(v2, h2, l2); split_f16(v3, h3, l3);
      const size_t o = ((size_t)b * T + t) * C4 + c4;
      __half2 hh[2] = {__halves2half2(h0, h1), __halves2half2(h2, h3)};
      reinterpret_cast<uint2*>(hi)[o] = *reinterpret_cast<uint2*>(hh);
      if (lo) {
        __half2 ll[2] = {__halves2half2(l0, l1), __halves2half2(l2, l3)};
        reinterpret_cast<uint2*>(lo)[o] = *reinterpret_cast<uint2*>(ll);
      }
    }
  }
}

// ------------------------------------------------------------------ GroupNorm
__global__ void groupnorm_stats_kernel(const float* __restrict__ x, int T, int C, int G, float eps,
                                       float* __restrict__ stats) {
  const int g = blockIdx.x, b = blockIdx.y, cpg = C / G;
  const float* xb = x + (long long)b * T * C + g * cpg;
  const int n = T * cpg;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float v = xb[(long long)(i / cpg) * C + (i % cpg)];
    s += v;
    q += (double)v * v;
  }
  __shared__ double ss[32], sq[32];
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
  if ((threadIdx.x & 31) == 0) { ss[threadIdx.x >> 5] = s; sq[threadIdx.x >> 5] = q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0, Q = 0;
    for (int i = 0; i < (blockDim.x >> 5); ++i) { S += ss[i]; Q += sq[i]; }
    double mean = S / n, var = Q / n - mean * mean;
    if (var < 0) var = 0;
    stats[((long long)b * G + g) * 2] = (float)mean;
    stats[((long long)b * G + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

// float4 variants (C and C/G multiples of 4): 16-byte loads, fp64 accumulation kept (the variance is E[x^2] - mean^2)
__global__ void groupnorm_stats_v4_kernel(const float4* __restrict__ x, int T, int C4, int G, float eps,
                                          float* __restrict__ stats) {
  const int g = blockIdx.x, b = blockIdx.y, cpg4 = C4 / G;
  const float4* xb = x + (long long)b * T * C4 + g * cpg4;
  const int n4 = T * cpg4;
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const int r = i / cpg4, c = i - r * cpg4;
    const float4 v = xb[(long long)r * C4 + c];
    s += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
    q += ((double)v.x * v.x + (double)v.y * v.y) + ((double)v.z * v.z + (double)v.w * v.w);
  }
  __shared__ double ss[32], sq[32];
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
  if ((threadIdx.x & 31) == 0) { ss[threadIdx.x >> 5] = s; sq[threadIdx.x >> 5] = q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0, Q = 0;
    for (int i = 0; i < (blockDim.x >> 5); ++i) { S += ss[i]; Q += sq[i]; }
    const double n = 4.0 * n4, mean = S / n;
    double var = Q / n - mean * mean;
    if (var < 0) var = 0;
    stats[((long long)b * G + g) * 2] = (float)mean;
    stats[((long long)b * G + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

__global__ void groupnorm_apply_v4_kernel(const float4* __restrict__ x, const float* __restrict__ stats,
                                          const float4* __restrict__ w, const float4* __restrict__ bz, int T, int C4, int cpg4,
                                          int G, int swish, float4* __restrict__ out, __half* __restrict__ hi,
                                          __half* __restrict__ lo, long long ld, long long rpb, long long off, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c4 = (int)(i % C4);
  const long long r = i / C4;
  const int t = (int)(r % T);
  const long long b = r / T;
  const float2 st = *reinterpret_cast<const float2*>(stats + (b * G + c4 / cpg4) * 2);
  const float4 xv = x[i], wv = __ldg(w + c4), bv = __ldg(bz + c4);
  float v[4] = {(xv.x - st.x) * st.y * wv.x + bv.x, (xv.y - st.x) * st.y * wv.y + bv.y,
                (xv.z - st.x) * st.y * wv.z + bv.z, (xv.w - st.x) * st.y * wv.w + bv.w};
  if (swish) {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = v[e] * sigmoid_acc(v[e]);
  }
  if (out) out[i] = make_float4(v[0], v[1], v[2], v[3]);
  if (hi) {
    __half h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) split_f16(v[e], h[e], l[e]);
    const long long o = ((b * rpb + off + t) * ld) / 4 + c4;          // ld is a multiple of 4 on this path
    __half2 hh[2] = {__halves2half2(h[0], h[1]), __halves2half2(h[2], h[3])};
    reinterpret_cast<uint2*>(hi)[o] = *reinterpret_cast<uint2*>(hh);
    if (lo) {
      __half2 ll[2] = {__halves2half2(l[0], l[1]), __halves2half2(l[2], l[3])};
      reinterpret_cast<uint2*>(lo)[o] = *reinterpret_cast<uint2*>(ll);
    }
  }
}

__global__ void groupnorm_apply_kernel(const float* __restrict__ x, const float* __restrict__ stats,
                                       const float* __restrict__ w, const float* __restrict__ bz, int T, int C, int G,
                                       int swish, float* __restrict__ out, __half* __restrict__ hi,
                                       __half* __restrict__ lo, long long ld, long long rpb, long long off) {
  const int t = blockIdx.x, b = blockIdx.y, cpg = C / G;
  const long long ri = ((long long)b * T + t) * C, ro = ((long long)b * rpb + off + t) * ld;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float* st = stats + ((long long)b * G + c / cpg) * 2;
    float v = (x[ri + c] - st[0]) * st[1] * w[c] + bz[c];
    if (swish) v = v * sigmoid_acc(v);
    if (out) out[ri + c] = v;
    if (hi) store_planes(hi, lo, ro + c, v);
  }
}

// ------------------------------------------------------------------ spectral
__global__ void istft_pre_kernel(const float* __restrict__ head, long long ld_in, int nf, __half* __restrict__ hi,
                                 __half* __restrict__ lo, long long ld) {
  const long long m = blockIdx.x;
  const float* hp = head + m * ld_in;
  const long long o = m * ld;
  for (int k = threadIdx.x; k < ld; k += blockDim.x) {
    if (k < nf) {
      float mag = fminf(expf(hp[k]), 100.f), ph = hp[nf + k];
      float sn, cs;
      sincosf(ph, &sn, &cs);
      store_planes(hi, lo, o + k, mag * cs);
      store_planes(hi, lo, o + nf + k, mag * sn);
    } else if (k >= 2 * nf) {
      store_planes(hi, lo, o + k, 0.f);
    }
  }
}

__global__ void istft_ola_kernel(const float* __restrict__ frames, const float* __restrict__ window, int F, int n_fft,
                                 int hop, float* __restrict__ wav) {
  const int pad = (n_fft - hop) / 2, R = n_fft / hop;
  const int b = blockIdx.y;
  const long long len = (long long)F * hop;
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= len) return;
  const long long u = t + pad;
  const int f_hi = (int)(u / hop);
  float acc = 0.f, env = 0.f;
  for (int r = R - 1; r >= 0; --r) {       // frames in increasing order f_hi-R+1 .. f_hi (fold's accumulation order)
    const int f = f_hi - r;
    if (f >= 0 && f < F) {
      const int i = (int)(u - (long long)f * hop);
      acc += frames[((long long)b * F + f) * n_fft + i];
      env += window[i] * window[i];
    }
  }
  wav[(long long)b * len + t] = acc / env;
}

// mirror-fill the pad rows of a channel-last padded plane buffer (reflect padding of SConv1d,
// HCodec-1.0/vq/encoder_modules/conv.py:79-96,196-210): row off-i <- row off+i, row off+T-1+i <- row off+T-1-i
__global__ void reflect_pad_rows_kernel(__half* __restrict__ hi, __half* __restrict__ lo, long long rpb, long long ld,
                                        int T, int off, int pad_l, int pad_r) {
  const int b = blockIdx.y, pr = blockIdx.x;          // pr < pad_l: left rows, else right rows
  long long dst, src;
  if (pr < pad_l) { dst = off - 1 - pr; src = off + 1 + pr; }
  else { const int i = pr - pad_l; dst = off + T + i; src = off + T - 2 - i; }
  const long long d = ((long long)b * rpb + dst) * ld, s2 = ((long long)b * rpb + src) * ld;
  for (int c = threadIdx.x; c < ld / 8; c += blockDim.x) {
    reinterpret_cast<uint4*>(hi + d)[c] = reinterpret_cast<const uint4*>(hi + s2)[c];
    if (lo) reinterpret_cast<uint4*>(lo + d)[c] = reinterpret_cast<const uint4*>(lo + s2)[c];
  }
}

// depthwise conv over time, odd kernel k, zero 'same' padding, channel-last fp32 (sub-pixel up-sampler's dw conv,
// vq/conv.py:84-92).  w [C,k].
__global__ void dwconv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                              int T, int C, int k, float* __restrict__ out) {
  const int t = blockIdx.x, b = blockIdx.y, h = k / 2;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = bias ? bias[c] : 0.f;
    for (int j = 0; j < k; ++j) {
      const int tt = t + j - h;
      if (tt >= 0 && tt < T) acc = fmaf(w[(long long)c * k + j], x[((long long)b * T + tt) * C + c], acc);
    }
    out[((long long)b * T + t) * C + c] = acc;
  }
}


// ------------------------------------------------------------------ two-stage (Cooley-Tukey) STFT front end
// The windowed real DFT of a frame as ONE K = n_fft contraction chains n_fft/16 tensor-core MMAs (x3 split terms) into one
// accumulator; the tensor core truncates at every accumulate, so the bias grows with the chain: measured 7e-6 of the largest
// magnitude at K = 1920 - 25x the error of an fp32 FFT, enough to move log|S| of a tiny bin by 1e-2 and to flip the sign of
// a vanishing imaginary part (phase +-1) ten times per 64 clips.  With n_fft = P*Q, s = Q a + b, k = k1 + P k2:
//   X[k1 + P k2] = sum_b e^{-2 pi i k2 b / Q} * ( e^{-2 pi i k1 b / n_fft} * sum_a xw[Q a + b] e^{-2 pi i k1 a / P} )
// i.e. a P-point DFT per residue b (GEMM A, K = P <= 64), a twiddle, a Q-point DFT per k1 (GEMM B, K = 2Q <= 128): chains of
// 4 and 8 MMAs - fp32-FFT-grade accuracy on the same tensor-core GEMM.
//   gather:  planes A[(clip, f, b), a] = pad(wav)[hop f + Q a + b] * window[Q a + b]          (a < P; cols P..63 zero)
//   twiddle: planes Z[(clip, f, k1), c*Q + b] = (Y[(clip, f, b), (k1, c)] * e^{-2 pi i k1 b / n_fft})_c,  c = re / im
//   post:    log(clip(|X|, 1e-5)), angle(X) / pi with X[k] read at row k % P, column pair k / P
__global__ void stft_gather_kernel(const float* __restrict__ wav, long long T, int hop, int n_fft, int P, int Q, int F,
                                   const float* __restrict__ win, __half* __restrict__ hi, __half* __restrict__ lo, long long total) {
  const int pad = (n_fft - hop) / 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int a = (int)(i & 63);
    const long long row = i >> 6;
    const int b = (int)(row % Q);
    const long long cf = row / Q;                   // clip * F + f
    const int f = (int)(cf % F);
    const long long clip = cf / F;
    float v = 0.f;
    if (a < P) {
      const int sidx = Q * a + b;
      const long long src = (long long)hop * f + sidx - pad;
      if (src >= 0 && src < T) v = wav[clip * T + src] * win[sidx];
    }
    store_planes(hi, lo, i, v);
  }
}
__global__ void stft_twiddle_kernel(const float* __restrict__ Y, long long ldY, int P, int Q, const float2* __restrict__ tw,
                                    __half* __restrict__ hi, __half* __restrict__ lo, long long total) {
  // one thread per (clip-frame, k1, b): reads the complex Y, writes re at column b and im at column Q + b of row (cf, k1)
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i % Q);
    const int k1 = (int)((i / Q) % P);
    const long long cf = i / ((long long)Q * P);
    const float* y = Y + (cf * Q + b) * ldY + 2 * k1;
    const float yr = y[0], yi = y[1];
    const float2 w = tw[b * P + k1];                // (cos, -sin)(2 pi k1 b / n_fft)
    const float zr = fmaf(yr, w.x, -yi * w.y), zi = fmaf(yr, w.y, yi * w.x);
    const long long o = (cf * P + k1) * 128;
    store_planes(hi, lo, o + b, zr);
    store_planes(hi, lo, o + Q + b, zi);
  }
}
__global__ void stft_post2_kernel(const float* __restrict__ X, long long ldX, int frames, int nf, int P, __half* __restrict__ hi,
                                  __half* __restrict__ lo, long long ld, long long rpb, long long off) {
  const int f = blockIdx.x, b = blockIdx.y;
  const float* xr = X + ((long long)b * frames + f) * P * ldX;
  const long long o = ((long long)b * rpb + off + f) * ld;
  for (int k = threadIdx.x; k < ld; k += blockDim.x) {
    if (k < nf) {
      const float* p = xr + (long long)(k % P) * ldX + 2 * (k / P);
      const float re = p[0], im = (k == 0 || k == nf - 1) ? 0.f : p[1];
      store_planes(hi, lo, o + k, logf(fmaxf(hypotf(re, im), 1e-5f)));
      store_planes(hi, lo, o + nf + k, atan2f(im, re) * 0.31830988618379067154f);
    } else if (k >= 2 * nf) {
      store_planes(hi, lo, o + k, 0.f);
    }
  }
}

}  // namespace qb
using namespace qb;

extern "C" int qb_split_f16(const float* x, qb_half* hi, qb_half* lo, int64_t n, void* stream) {
  QB_REQUIRE(x && hi && n >= 0, "split: bad args");
  if (n == 0) return 0;
  int blocks = (int)(ceil_div(n, 256) < 132 * 16 ? ceil_div(n, 256) : 132 * 16);
  split_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, (__half*)hi, (__half*)lo, n);
  QB_LAUNCH_END();
}

extern "C" int qb_rows_to_planes(const float* x, int64_t B, int64_t rows, int64_t C, int32_t repeat, int32_t act,
                                 qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off,
                                 void* stream) {
  QB_REQUIRE(x && hi && repeat >= 1 && C <= ld, "rows_to_planes: bad args");
  QB_REQUIRE(row_off + rows * repeat <= rows_per_batch, "rows_to_planes: rows overflow the padded buffer");
  dim3 grid((unsigned)(rows * repeat), (unsigned)B);
  rows_to_planes_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, (int)rows, (int)C, repeat, act, (__half*)hi,
                                                               (__half*)lo, ld, rows_per_batch, row_off);
  QB_LAUNCH_END();
}

extern "C" int qb_bct_to_planes(const float* x, int64_t B, int64_t C, int64_t T, qb_half* hi, qb_half* lo, int64_t ld,
                                int64_t rows_per_batch, int64_t row_off, void* stream) {
  QB_REQUIRE(x && hi && C <= ld && row_off + T <= rows_per_batch, "bct_to_planes: bad args");
  dim3 grid((unsigned)ceil_div(T, 32), (unsigned)ceil_div(ld, 32), (unsigned)B), block(32, 8);
  bct_to_planes_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, (int)C, (int)T, (__half*)hi, (__half*)lo, ld,
                                                                rows_per_batch, row_off);
  QB_LAUNCH_END();
}

extern "C" int qb_layernorm(const float* x, const float* w, const float* b, float eps, int64_t B, int64_t rows,
                            int64_t C, float* out_f32, qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch,
                            int64_t row_off, void* stream) {
  QB_REQUIRE(x && w && b && (out_f32 || hi), "layernorm: bad args");
  QB_REQUIRE(!hi || (C <= ld && row_off + rows <= rows_per_batch), "layernorm: plane buffer too small");
  const long long total = B * rows;
  layernorm_kernel<QB_ACT_NONE><<<(unsigned)ceil_div(total, 8), 256, 0, (cudaStream_t)stream>>>(
      x, w, b, eps, total, (int)rows, (int)C, out_f32, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off, 0);
  QB_LAUNCH_END();
}

extern "C" int qb_layernorm_act(const float* x, const float* w, const float* b, float eps, int64_t B, int64_t rows, int64_t C,
                                int32_t act, float* out_f32, qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch,
                                int64_t row_off, void* stream) {
  QB_REQUIRE(x && w && b && (out_f32 || hi), "layernorm_act: bad args");
  QB_REQUIRE(act == QB_ACT_NONE || act == QB_ACT_GELU, "layernorm_act: activation %d unsupported (none / gelu)", act);
  QB_REQUIRE(!hi || (C <= ld && row_off + rows <= rows_per_batch), "layernorm_act: plane buffer too small");
  const long long total = B * rows;
  if (act == QB_ACT_GELU)
    layernorm_kernel<QB_ACT_GELU><<<(unsigned)ceil_div(total, 8), 256, 0, (cudaStream_t)stream>>>(
        x, w, b, eps, total, (int)rows, (int)C, out_f32, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off, 0);
  else
    layernorm_kernel<QB_ACT_NONE><<<(unsigned)ceil_div(total, 8), 256, 0, (cudaStream_t)stream>>>(
        x, w, b, eps, total, (int)rows, (int)C, out_f32, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off, 0);
  QB_LAUNCH_END();
}

extern "C" int qb_adalayernorm(const float* x, const float* scale, const float* shift, int64_t cond_stride, float eps,
                               int64_t B, int64_t rows, int64_t C, float* out_f32, qb_half* hi, qb_half* lo, int64_t ld,
                               int64_t rows_per_batch, int64_t row_off, void* stream) {
  QB_REQUIRE(x && scale && shift && (out_f32 || hi), "adalayernorm: bad args");
  QB_REQUIRE(!hi || (C <= ld && row_off + rows <= rows_per_batch), "adalayernorm: plane buffer too small");
  const long long total = B * rows;
  layernorm_kernel<QB_ACT_NONE><<<(unsigned)ceil_div(total, 8), 256, 0, (cudaStream_t)stream>>>(
      x, scale, shift, eps, total, (int)rows, (int)C, out_f32, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off,
      cond_stride);
  QB_LAUNCH_END();
}

extern "C" int qb_rmsnorm(const float* x, const float* w, float eps, int64_t rows, int64_t C, float* out_f32, qb_half* hi,
                          qb_half* lo, void* stream) {
  QB_REQUIRE(x && w && (hi || out_f32), "rmsnorm: bad args");
  rmsnorm_kernel<<<(unsigned)ceil_div(rows, 8), 256, 0, (cudaStream_t)stream>>>(x, w, eps, rows, (int)C, out_f32,
                                                                                 (__half*)hi, (__half*)lo);
  QB_LAUNCH_END();
}

static int dwconv7_ln_launch(const float* x, const float* dw_w, const float* dw_b, const float* ln_w, const float* ln_b,
                             int64_t ln_bstride, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo, void* stream) {
  QB_REQUIRE(x && dw_w && dw_b && ln_w && ln_b && hi, "dwconv7_ln: bad args");
  if (C % 128 == 0 && C / 4 <= 512 && ln_bstride % 4 == 0) {
    constexpr int TT = 8;
    dim3 grid((unsigned)ceil_div(T, TT), (unsigned)B);
    if (C / 4 <= 384)      // <= 85 registers: two CTAs per SM, one's loads overlap the other's reduction / stores
      dwconv7_ln_v2_kernel<TT, 384, 2><<<grid, (unsigned)(C / 4), 0, (cudaStream_t)stream>>>(
          (const float4*)x, dw_w, (const float4*)dw_b, (const float4*)ln_w, (const float4*)ln_b, (int)T, (int)(C / 4),
          (__half*)hi, (__half*)lo, (long long)(ln_bstride / 4));
    else
      dwconv7_ln_v2_kernel<TT, 512, 1><<<grid, (unsigned)(C / 4), 0, (cudaStream_t)stream>>>(
          (const float4*)x, dw_w, (const float4*)dw_b, (const float4*)ln_w, (const float4*)ln_b, (int)T, (int)(C / 4),
          (__half*)hi, (__half*)lo, (long long)(ln_bstride / 4));
    QB_LAUNCH_END();
  }
  const int warps = 8;
  const size_t smem = (size_t)warps * C * sizeof(float);
  QB_REQUIRE(smem <= 200 * 1024, "dwconv7_ln: C too large");
  QB_CHECK_CUDA(cudaFuncSetAttribute(dwconv7_ln_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const long long total = B * T;
  dwconv7_ln_kernel<<<(unsigned)ceil_div(total, warps), warps * 32, smem, (cudaStream_t)stream>>>(
      x, dw_w, dw_b, ln_w, ln_b, (int)T, (int)C, total, (__half*)hi, (__half*)lo, (long long)ln_bstride);
  QB_LAUNCH_END();
}

extern "C" int qb_dwconv7_ln(const float* x, const float* dw_w, const float* dw_b, const float* ln_w,
                             const float* ln_b, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo,
                             void* stream) {
  return dwconv7_ln_launch(x, dw_w, dw_b, ln_w, ln_b, 0, B, T, C, hi, lo, stream);
}

extern "C" int qb_dwconv7_adaln(const float* x, const float* dw_w, const float* dw_b, const float* scale,
                                const float* shift, int64_t cond_stride, int64_t B, int64_t T, int64_t C, qb_half* hi,
                                qb_half* lo, void* stream) {
  return dwconv7_ln_launch(x, dw_w, dw_b, scale, shift, cond_stride, B, T, C, hi, lo, stream);
}

// ------------------------------------------------------------------ BiCodec WaveGenerator glue
// Snake (bicodec/modules/blocks/layers.py:33-38): x + sin(alpha x)^2 / (alpha + 1e-9), per channel, written as fp16 planes
// into the interior of the next convolution's zero-padded channel-last buffer.  x rows of clip b start at
// x + b * x_bstride (the transposed-conv GEMM leaves its output as a strided view).
// 8 channels per thread: two 16-byte loads, one 16-byte store per plane
__global__ void snake_planes_v8_kernel(const float* __restrict__ x, long long x_bstride, const float* __restrict__ alpha,
                                       int T, int C8, int ld8, __half* __restrict__ hi, __half* __restrict__ lo,
                                       long long rpb, long long off, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % ld8);
  const long long r = i / ld8;
  const int t = (int)(r % T);
  const long long b = r / T;
  float v[8];
  if (c8 < C8) {
    const float4* xp = reinterpret_cast<const float4*>(x + b * x_bstride + ((long long)t * C8 + c8) * 8);
    const float4* ap = reinterpret_cast<const float4*>(alpha + c8 * 8);
    const float4 x0 = xp[0], x1 = xp[1], a0 = __ldg(ap), a1 = __ldg(ap + 1);
    const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
    const float as[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float sn = sinf(as[e] * xs[e]);
      v[e] = fmaf(1.0f / (as[e] + 1e-9f), sn * sn, xs[e]);
    }
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
  }
  __half2 h2[4], l2[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    __half a, bq, la, lb;
    split_f16(v[2 * e], a, la);
    split_f16(v[2 * e + 1], bq, lb);
    h2[e] = __halves2half2(a, bq);
    l2[e] = __halves2half2(la, lb);
  }
  const long long o = ((b * rpb + off + t) * ld8 + c8);
  reinterpret_cast<uint4*>(hi)[o] = *reinterpret_cast<uint4*>(h2);
  if (lo) reinterpret_cast<uint4*>(lo)[o] = *reinterpret_cast<uint4*>(l2);
}

__global__ void snake_planes_kernel(const float* __restrict__ x, long long x_bstride, const float* __restrict__ alpha,
                                    int T, int C, __half* __restrict__ hi, __half* __restrict__ lo, long long ld,
                                    long long rpb, long long off, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % ld);
  const long long r = i / ld;
  const int t = (int)(r % T);
  const long long b = r / T;
  float v = 0.f;
  if (c < C) {
    const float xv = x[b * x_bstride + (long long)t * C + c], a = alpha[c];
    const float sn = sinf(a * xv);
    v = xv + sn * sn / (a + 1e-9f);
  }
  store_planes(hi, lo, (b * rpb + off + t) * ld + c, v);
}

// ELU of rows with a batch pitch -> planes: the up-sampled frames of a transposed conv sit inside its phase GEMM's output rows,
// offset by the padding, so clip b starts at x + b * x_bstride rather than at b * T * C
__global__ void elu_planes_kernel(const float* __restrict__ x, long long x_bstride, int T, int C, __half* __restrict__ hi,
                                  __half* __restrict__ lo, long long ld, long long rpb, long long off, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % ld);
  const long long r = i / ld;
  const int t = (int)(r % T);
  const long long b = r / T;
  const float v = c < C ? elu_f(x[b * x_bstride + (long long)t * C + c]) : 0.f;
  store_planes(hi, lo, (b * rpb + off + t) * ld + c, v);
}

// x[b, t, c] + vec[b, c] -> planes (the speaker d-vector added to every frame, bicodec/bicodec.py:197)
__global__ void addvec_planes_kernel(const float* __restrict__ x, const float* __restrict__ vec, int T, int C,
                                     __half* __restrict__ hi, __half* __restrict__ lo, long long ld, long long rpb,
                                     long long off, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % ld);
  const long long r = i / ld;
  const int t = (int)(r % T);
  const long long b = r / T;
  const float v = c < C ? x[(b * T + t) * C + c] + vec[b * C + c] : 0.f;
  store_planes(hi, lo, (b * rpb + off + t) * ld + c, v);
}

extern "C" int qb_snake_planes(const float* x, int64_t x_batch_stride, const float* alpha, int64_t B, int64_t T, int64_t C,
                               qb_half* hi, qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off,
                               void* stream) {
  QB_REQUIRE(x && alpha && hi && C <= ld && row_off + T <= rows_per_batch, "snake_planes: bad args");
  const long long total = B * T * ld;
  if (C % 8 == 0 && ld % 8 == 0 && x_batch_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(alpha) & 15) == 0) {
    snake_planes_v8_kernel<<<(unsigned)ceil_div(total / 8, 256), 256, 0, (cudaStream_t)stream>>>(
        x, x_batch_stride, alpha, (int)T, (int)(C / 8), (int)(ld / 8), (__half*)hi, (__half*)lo, rows_per_batch, row_off,
        total / 8);
    QB_LAUNCH_END();
  }
  snake_planes_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
      x, x_batch_stride, alpha, (int)T, (int)C, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off, total);
  QB_LAUNCH_END();
}

extern "C" int qb_elu_planes(const float* x, int64_t x_batch_stride, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo,
                             int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream) {
  QB_REQUIRE(x && hi && T >= 1 && C <= ld && row_off + T <= rows_per_batch && x_batch_stride >= T * C, "elu_planes: bad args");
  const long long total = B * T * ld;
  elu_planes_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
      x, x_batch_stride, (int)T, (int)C, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off, total);
  QB_LAUNCH_END();
}

extern "C" int qb_addvec_planes(const float* x, const float* vec, int64_t B, int64_t T, int64_t C, qb_half* hi, qb_half* lo,
                                int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream) {
  QB_REQUIRE(x && vec && hi && C <= ld && row_off + T <= rows_per_batch, "addvec_planes: bad args");
  const long long total = B * T * ld;
  addvec_planes_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
      x, vec, (int)T, (int)C, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off, total);
  QB_LAUNCH_END();
}

extern "C" int qb_groupnorm_stats(const float* x, int64_t B, int64_t T, int64_t C, int32_t groups, float eps,
                                  float* stats, void* stream) {
  QB_REQUIRE(x && stats && C % groups == 0, "groupnorm_stats: bad args");
  dim3 grid((unsigned)groups, (unsigned)B);
  if (C % 4 == 0 && (C / groups) % 4 == 0) {
    groupnorm_stats_v4_kernel<<<grid, 512, 0, (cudaStream_t)stream>>>((const float4*)x, (int)T, (int)(C / 4), groups, eps, stats);
    QB_LAUNCH_END();
  }
  groupnorm_stats_kernel<<<grid, 512, 0, (cudaStream_t)stream>>>(x, (int)T, (int)C, groups, eps, stats);
  QB_LAUNCH_END();
}

extern "C" int qb_groupnorm_apply(const float* x, const float* stats, const float* w, const float* b, int64_t B,
                                  int64_t T, int64_t C, int32_t groups, int32_t swish, float* out_f32, qb_half* hi,
                                  qb_half* lo, int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream) {
  QB_REQUIRE(x && stats && w && b && (out_f32 || hi), "groupnorm_apply: bad args");
  QB_REQUIRE(!hi || (C <= ld && row_off + T <= rows_per_batch), "groupnorm_apply: plane buffer too small");
  if (C % 4 == 0 && (C / groups) % 4 == 0 && (!hi || ld % 4 == 0)) {
    const long long total = B * T * (C / 4);
    groupnorm_apply_v4_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const float4*)x, stats, (const float4*)w, (const float4*)b, (int)T, (int)(C / 4), (int)(C / groups / 4), groups, swish,
        (float4*)out_f32, (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off, total);
    QB_LAUNCH_END();
  }
  dim3 grid((unsigned)T, (unsigned)B);
  groupnorm_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, stats, w, b, (int)T, (int)C, groups, swish, out_f32,
                                                                (__half*)hi, (__half*)lo, ld, rows_per_batch, row_off);
  QB_LAUNCH_END();
}

extern "C" int qb_istft_pre(const float* head, int64_t ld_in, int64_t M, int32_t nf, qb_half* hi, qb_half* lo,
                            int64_t ld, void* stream) {
  QB_REQUIRE(head && hi && 2 * nf <= ld && 2 * nf <= ld_in, "istft_pre: bad args");
  istft_pre_kernel<<<(unsigned)M, 256, 0, (cudaStream_t)stream>>>(head, ld_in, nf, (__half*)hi, (__half*)lo, ld);
  QB_LAUNCH_END();
}

extern "C" int qb_istft_ola(const float* frames, const float* window, int64_t B, int64_t F, int32_t n_fft, int32_t hop,
                            float* wav, void* stream) {
  QB_REQUIRE(frames && window && wav && hop > 0 && n_fft % hop == 0 && (n_fft - hop) % 2 == 0, "istft_ola: bad args");
  dim3 grid((unsigned)ceil_div(F * hop, 256), (unsigned)B);
  istft_ola_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(frames, window, (int)F, n_fft, hop, wav);
  QB_LAUNCH_END();
}

extern "C" int qb_reflect_pad_rows(qb_half* hi, qb_half* lo, int64_t B, int64_t rows_per_batch, int64_t ld, int64_t T,
                                   int64_t row_off, int32_t pad_l, int32_t pad_r, void* stream) {
  QB_REQUIRE(hi && ld % 8 == 0 && pad_l >= 0 && pad_r >= 0 && row_off >= pad_l && row_off + T + pad_r <= rows_per_batch,
             "reflect_pad_rows: bad args");
  QB_REQUIRE(T > pad_l && T > pad_r, "reflect_pad_rows: input shorter than the reflection");
  if (pad_l + pad_r == 0) return 0;
  dim3 grid((unsigned)(pad_l + pad_r), (unsigned)B);
  reflect_pad_rows_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((__half*)hi, (__half*)lo, rows_per_batch, ld, (int)T,
                                                                 (int)row_off, pad_l, pad_r);
  QB_LAUNCH_END();
}

extern "C" int qb_dwconv(const float* x, const float* w, const float* bias, int64_t B, int64_t T, int64_t C, int32_t k,
                         float* out, void* stream) {
  QB_REQUIRE(x && w && out && k % 2 == 1, "dwconv: bad args");
  dim3 grid((unsigned)T, (unsigned)B);
  dwconv_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, w, bias, (int)T, (int)C, k, out);
  QB_LAUNCH_END();
}

extern "C" int qb_stft_gather(const float* wav, int64_t B, int64_t T, int32_t hop, int32_t n_fft, int32_t P, int32_t Q,
                              const float* window, qb_half* hi, qb_half* lo, void* stream) {
  QB_REQUIRE(wav && window && hi && P * Q == n_fft && P <= 64 && 2 * Q <= 128 && T % hop == 0 && (n_fft - hop) % 2 == 0,
             "stft_gather: needs n_fft == P*Q, P <= 64, Q <= 64, T a multiple of hop");
  const int64_t F = T / hop;
  const long long total = B * F * Q * 64;
  stft_gather_kernel<<<(unsigned)(ceil_div(total, 256) < 132 * 32 ? ceil_div(total, 256) : 132 * 32), 256, 0, (cudaStream_t)stream>>>(
      wav, T, hop, n_fft, P, Q, (int)F, window, (__half*)hi, (__half*)lo, total);
  QB_LAUNCH_END();
}

extern "C" int qb_stft_twiddle(const float* Y, int64_t ldY, int64_t frames_total, int32_t P, int32_t Q, const float* twiddle,
                               qb_half* hi, qb_half* lo, void* stream) {
  QB_REQUIRE(Y && twiddle && hi && ldY >= 2 * P && 2 * Q <= 128, "stft_twiddle: bad args");
  const long long total = frames_total * P * Q;
  stft_twiddle_kernel<<<(unsigned)(ceil_div(total, 256) < 132 * 32 ? ceil_div(total, 256) : 132 * 32), 256, 0, (cudaStream_t)stream>>>(
      Y, ldY, P, Q, (const float2*)twiddle, (__half*)hi, (__half*)lo, total);
  QB_LAUNCH_END();
}

extern "C" int qb_stft_post2(const float* X, int64_t ldX, int64_t B, int64_t frames, int32_t nf, int32_t P, qb_half* hi, qb_half* lo,
                             int64_t ld, int64_t rows_per_batch, int64_t row_off, void* stream) {
  QB_REQUIRE(X && hi && 2 * nf <= ld && row_off + frames <= rows_per_batch && ldX >= 2 * ((nf - 1) / P + 1), "stft_post2: bad args");
  dim3 grid((unsigned)frames, (unsigned)B);
  stft_post2_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(X, ldX, (int)frames, nf, P, (__half*)hi, (__half*)lo, ld, rows_per_batch,
                                                           row_off);
  QB_LAUNCH_END();
}
