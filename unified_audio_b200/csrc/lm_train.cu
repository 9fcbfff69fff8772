// Backward pass of the UniSE AR-LM's teacher-forced loss (QuarkAudio-UniSE/model/llm/llm_sft.py:37-89, llm.py:87-104,150-228) and the
// training forward's attention with dropout.  Every kernel here is deterministic: no floating-point atomics, every reduction runs
// in a fixed order, and reductions over tokens carry fp64 partials.  The dense contractions of the backward pass (data gradients
// dX = dY W and weight gradients dW = dY^T X) run on qb_gemm in the 3-term split mode; this file adds what is not a contraction and
// the transposing split that turns token-major rows into the feature-major planes a weight gradient contracts over.
#include <atomic>
#include <cmath>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

#define QB_TRAIN_LAUNCHED(n)         \
  g_launches += (n);                 \
  QB_CHECK_CUDA(cudaGetLastError()); \
  return 0

// ------------------------------------------------------------------------------------------ dropout mask
// keep(seed, layer, b, h, i, j) = (Philox4x32-10(key = {seed_lo, seed_hi}, counter = {i, j >> 2, b * heads + h, layer}).word[j & 3]
// >> 8) >= thr, thr = (float)p * 2^24 rounded half-to-even (llrint of an exact double): one Philox call gives the mask of four
// consecutive keys (include/quark_b200.h).
__device__ __forceinline__ uint4 philox4(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

struct DropCfg {
  uint32_t k0, k1, thr, layer;
  float keep_scale;   // 1 / (1 - p)
};

// mask bits of keys 4*j4 .. 4*j4+3 for query i (bit r = key 4*j4 + r kept)
__device__ __forceinline__ uint32_t keep_bits(const DropCfg& dc, int i, int j4, int bh) {
  if (dc.thr == 0u) return 0xFu;
  const uint4 r = philox4(dc.k0, dc.k1, (uint32_t)i, (uint32_t)j4, (uint32_t)bh, dc.layer);
  return (uint32_t)((r.x >> 8) >= dc.thr) | ((uint32_t)((r.y >> 8) >= dc.thr) << 1) | ((uint32_t)((r.z >> 8) >= dc.thr) << 2) |
         ((uint32_t)((r.w >> 8) >= dc.thr) << 3);
}

// ------------------------------------------------------------------------------------------ causal attention, training forward
// Tiles of 32 queries x 32 keys, 256 threads: thread t owns query row t / 8 (eight threads per row, one warp holds four rows), the
// four consecutive keys 4 * (t % 8) .. +3 of each key tile for the scores, and the eight head dimensions 8 * (t % 8) .. +7 of the
// output.  fp32 SIMT arithmetic throughout (fp32-grade like the split-operand eval kernel).
constexpr int AT = 32;
constexpr int APAD = 65;

// qkv [B*L, 3*H] fp32 -> qs = RoPE(q) / 8, kr = RoPE(k), vv = v, each [B*heads, L, 64]
__global__ void lm_train_qkv_kernel(const float* __restrict__ qkv, int L, int heads, const float* __restrict__ rcos,
                                    const float* __restrict__ rsin, float* __restrict__ qs, float* __restrict__ kr, float* __restrict__ vv) {
  const long long row = blockIdx.x;                  // b * L + t
  const int b = (int)(row / L), t = (int)(row % L);
  const int H = heads * 64;
  const float* src = qkv + row * 3 * H;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    const int h = c >> 6, d = c & 63;
    const long long o = (((long long)b * heads + h) * L + t) * 64 + d;
    const float cs = rcos[(long long)t * 64 + d], sn = rsin[(long long)t * 64 + d];
    const int pd = d < 32 ? d + 32 : d - 32;
    const float sg = d < 32 ? -1.f : 1.f;
    const float q = src[c], qp = src[h * 64 + pd];
    const float k = src[H + c], kp = src[H + h * 64 + pd];
    qs[o] = (q * cs + sg * qp * sn) * 0.125f;
    kr[o] = k * cs + sg * kp * sn;
    vv[o] = src[2 * H + c];
  }
}

__global__ void __launch_bounds__(256)
lm_attn_train_fwd_kernel(const float* __restrict__ qs, const float* __restrict__ kr, const float* __restrict__ vv, int L, int heads,
                         DropCfg dc, float* __restrict__ out, float* __restrict__ lse) {
  __shared__ float sQ[AT][APAD], sK[AT][APAD], sV[AT][64], sP[AT][AT + 1];
  const int tid = threadIdx.x, ri = tid >> 3, g = tid & 7;
  const int bh = blockIdx.y, b = bh / heads, h = bh % heads;
  const int q0 = blockIdx.x * AT;
  const float* Q = qs + (long long)bh * L * 64;
  const float* K = kr + (long long)bh * L * 64;
  const float* V = vv + (long long)bh * L * 64;
  for (int e = tid; e < AT * 64; e += 256) {
    const int r = e >> 6, d = e & 63;
    sQ[r][d] = q0 + r < L ? Q[(long long)(q0 + r) * 64 + d] : 0.f;
  }
  const int qi = q0 + ri;
  float m = -1e30f, l = 0.f, acc[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) acc[u] = 0.f;
  const int q_last = min(q0 + AT, L) - 1;
  for (int k0 = 0; k0 <= q_last; k0 += AT) {
    __syncthreads();
    for (int e = tid; e < AT * 64; e += 256) {
      const int r = e >> 6, d = e & 63;
      const bool ok = k0 + r < L;
      sK[r][d] = ok ? K[(long long)(k0 + r) * 64 + d] : 0.f;
      sV[r][d] = ok ? V[(long long)(k0 + r) * 64 + d] : 0.f;
    }
    __syncthreads();
    float s[4];
    float tmax = -1e30f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int j = 4 * g + r, kj = k0 + j;
      float a = 0.f;
#pragma unroll 16
      for (int d = 0; d < 64; ++d) a = fmaf(sQ[ri][d], sK[j][d], a);
      s[r] = (kj <= qi && qi < L) ? a : -INFINITY;
      tmax = fmaxf(tmax, s[r]);
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
    const float mn = fmaxf(m, tmax);
    const float alpha = expf(m - mn);
    const uint32_t kb = qi < L ? keep_bits(dc, qi, (k0 >> 2) + g, bh) : 0u;
    float ps = 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float p = expf(s[r] - mn);
      ps += p;
      sP[ri][4 * g + r] = ((kb >> r) & 1u) ? p * dc.keep_scale : 0.f;
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
    l = l * alpha + ps;
    m = mn;
    __syncwarp();
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] *= alpha;
    for (int j = 0; j < AT; ++j) {
      const float p = sP[ri][j];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] = fmaf(p, sV[j][8 * g + u], acc[u]);
    }
  }
  if (qi < L) {
    const float inv = 1.f / l;
    float* o = out + ((long long)b * L + qi) * heads * 64 + h * 64 + 8 * g;
#pragma unroll
    for (int u = 0; u < 8; ++u) o[u] = acc[u] * inv;
    if (g == 0) lse[(long long)bh * L + qi] = m + logf(l);
  }
}

// D[bh, i] = sum_d dO[i, d] * O[i, d] (token-major rows of [B*L, heads*64]); fp64 sum
__global__ void lm_attn_bwd_dot_kernel(const float* __restrict__ o, const float* __restrict__ dout, int L, int heads, long long rows,
                                       float* __restrict__ D) {
  const long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= rows * heads) return;
  const long long row = w / heads;
  const int h = (int)(w % heads);
  const long long base = row * heads * 64 + h * 64;
  double a = (double)o[base + lane] * dout[base + lane] + (double)o[base + lane + 32] * dout[base + lane + 32];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) a += __shfl_xor_sync(0xffffffffu, a, s);
  if (lane == 0) {
    const int b = (int)(row / L), t = (int)(row % L);
    D[((long long)b * heads + h) * L + t] = (float)a;
  }
}

// P[i][j] (dropped and scaled) and dS[i][j] of one 32 x 32 tile: thread (ri, g) computes query ri, keys 4g .. 4g+3
__device__ __forceinline__ void attn_bwd_tile(const float (*sQ)[APAD], const float (*sK)[APAD], const float (*sV)[APAD],
                                              const float (*sdO)[APAD], const float* sL, const float* sD, int q0, int k0, int L, int bh,
                                              const DropCfg& dc, float (*sP)[AT + 1], float (*sS)[AT + 1]) {
  const int tid = threadIdx.x, ri = tid >> 3, g = tid & 7;
  const int qi = q0 + ri;
  const uint32_t kb = qi < L ? keep_bits(dc, qi, (k0 >> 2) + g, bh) : 0u;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int j = 4 * g + r, kj = k0 + j;
    float s = 0.f, dp = 0.f;
#pragma unroll 16
    for (int d = 0; d < 64; ++d) {
      s = fmaf(sQ[ri][d], sK[j][d], s);
      dp = fmaf(sdO[ri][d], sV[j][d], dp);
    }
    const bool ok = kj <= qi && qi < L && kj < L;
    const float p = ok ? expf(s - sL[ri]) : 0.f;
    const float keep = ((kb >> r) & 1u) ? dc.keep_scale : 0.f;
    sP[ri][j] = p * keep;
    sS[ri][j] = p * (dp * keep - sD[ri]);
  }
}

__device__ __forceinline__ void load_rows64(float (*dst)[APAD], const float* src, long long stride, int r0, int L) {
  for (int e = threadIdx.x; e < AT * 64; e += 256) {
    const int r = e >> 6, d = e & 63;
    dst[r][d] = r0 + r < L ? src[(long long)(r0 + r) * stride + d] : 0.f;
  }
}

// RoPE undone on a gradient row held in shared memory: x_rot = x cos + rot(x) sin, rot(x) = [-x2, x1]  =>
// dx[d] = g[d] cos[d] + g[d+32] sin[d+32] (d < 32),  dx[d] = g[d] cos[d] - g[d-32] sin[d-32] (d >= 32)
__device__ __forceinline__ float unrope(const float* gr, const float* cs, const float* sn, int d) {
  return d < 32 ? gr[d] * cs[d] + gr[d + 32] * sn[d + 32] : gr[d] * cs[d] - gr[d - 32] * sn[d - 32];
}

// dK, dV of one key tile: loop over the query tiles at and after it
__global__ void __launch_bounds__(256)
lm_attn_train_dkv_kernel(const float* __restrict__ qs, const float* __restrict__ kr, const float* __restrict__ vv,
                         const float* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ D, int L, int heads,
                         const float* __restrict__ rcos, const float* __restrict__ rsin, DropCfg dc, float* __restrict__ dqkv) {
  __shared__ float sQ[AT][APAD], sK[AT][APAD], sV[AT][APAD], sdO[AT][APAD], sP[AT][AT + 1], sS[AT][AT + 1], sL[AT], sD[AT];
  const int tid = threadIdx.x, rj = tid >> 3, g = tid & 7;
  const int bh = blockIdx.y, b = bh / heads, h = bh % heads, H = heads * 64;
  const int k0 = blockIdx.x * AT;
  const long long hb = (long long)bh * L * 64;
  load_rows64(sK, kr + hb, 64, k0, L);
  load_rows64(sV, vv + hb, 64, k0, L);
  float dk[8], dv[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) dk[u] = dv[u] = 0.f;
  for (int q0 = k0; q0 < L; q0 += AT) {
    __syncthreads();
    load_rows64(sQ, qs + hb, 64, q0, L);
    load_rows64(sdO, dout + ((long long)b * L) * H + h * 64, H, q0, L);
    if (tid < AT) {
      sL[tid] = q0 + tid < L ? lse[(long long)bh * L + q0 + tid] : 0.f;
      sD[tid] = q0 + tid < L ? D[(long long)bh * L + q0 + tid] : 0.f;
    }
    __syncthreads();
    attn_bwd_tile(sQ, sK, sV, sdO, sL, sD, q0, k0, L, bh, dc, sP, sS);
    __syncthreads();
    for (int i = 0; i < AT; ++i) {
      const float p = sP[i][rj], ds = sS[i][rj];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        dv[u] = fmaf(p, sdO[i][8 * g + u], dv[u]);
        dk[u] = fmaf(ds, sQ[i][8 * g + u], dk[u]);
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < 8; ++u) sK[rj][8 * g + u] = dk[u];
  __syncthreads();
  const int kj = k0 + rj;
  if (kj < L) {
    float* o = dqkv + ((long long)b * L + kj) * 3 * H + h * 64;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int d = 8 * g + u;
      o[H + d] = unrope(sK[rj], rcos + (long long)kj * 64, rsin + (long long)kj * 64, d);
      o[2 * H + d] = dv[u];
    }
  }
}

// dQ of one query tile: loop over the key tiles up to it
__global__ void __launch_bounds__(256)
lm_attn_train_dq_kernel(const float* __restrict__ qs, const float* __restrict__ kr, const float* __restrict__ vv,
                        const float* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ D, int L, int heads,
                        const float* __restrict__ rcos, const float* __restrict__ rsin, DropCfg dc, float* __restrict__ dqkv) {
  __shared__ float sQ[AT][APAD], sK[AT][APAD], sV[AT][APAD], sdO[AT][APAD], sP[AT][AT + 1], sS[AT][AT + 1], sL[AT], sD[AT];
  const int tid = threadIdx.x, ri = tid >> 3, g = tid & 7;
  const int bh = blockIdx.y, b = bh / heads, h = bh % heads, H = heads * 64;
  const int q0 = blockIdx.x * AT;
  const long long hb = (long long)bh * L * 64;
  load_rows64(sQ, qs + hb, 64, q0, L);
  load_rows64(sdO, dout + ((long long)b * L) * H + h * 64, H, q0, L);
  if (tid < AT) {
    sL[tid] = q0 + tid < L ? lse[(long long)bh * L + q0 + tid] : 0.f;
    sD[tid] = q0 + tid < L ? D[(long long)bh * L + q0 + tid] : 0.f;
  }
  float dq[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) dq[u] = 0.f;
  const int q_last = min(q0 + AT, L) - 1;
  for (int k0 = 0; k0 <= q_last; k0 += AT) {
    __syncthreads();
    load_rows64(sK, kr + hb, 64, k0, L);
    load_rows64(sV, vv + hb, 64, k0, L);
    __syncthreads();
    attn_bwd_tile(sQ, sK, sV, sdO, sL, sD, q0, k0, L, bh, dc, sP, sS);
    __syncwarp();                                   // row ri's dS was written by the eight threads of this warp that own it
    for (int j = 0; j < AT; ++j) {
      const float ds = sS[ri][j];
#pragma unroll
      for (int u = 0; u < 8; ++u) dq[u] = fmaf(ds, sK[j][8 * g + u], dq[u]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < 8; ++u) sQ[ri][8 * g + u] = dq[u] * 0.125f;
  __syncthreads();
  const int qi = q0 + ri;
  if (qi < L) {
    float* o = dqkv + ((long long)b * L + qi) * 3 * H + h * 64;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int d = 8 * g + u;
      o[d] = unrope(sQ[ri], rcos + (long long)qi * 64, rsin + (long long)qi * 64, d);
    }
  }
}

// ------------------------------------------------------------------------------------------ loss backward
// out = g * (softmax(logits) - t) * scale, t = 1 - ls on the target and ls / (V - 1) elsewhere; the loss's gradient is this times
// 1 / (M * scale) (KL batchmean over M rows).  Most entries are ~1/V: a power-of-two scale near V keeps them out of fp16's subnormal
// range in the planes.  Columns V .. ld_out - 1 are written as zero.  fp32 rows and fp16 hi/lo planes, both [M, ld_out].
__global__ void __launch_bounds__(256)
lm_loss_bwd_kernel(const float* __restrict__ logits, long long ld, int V, const int64_t* __restrict__ targets, float ls,
                   const float* __restrict__ gout, float scale, long long ld_out, float* __restrict__ out, __half* __restrict__ hi,
                   __half* __restrict__ lo) {
  const long long row = blockIdx.x;
  const float* x = logits + row * ld;
  __shared__ float sm[256];
  float m = -INFINITY;
  for (int c = threadIdx.x; c < V; c += 256) m = fmaxf(m, x[c]);
  sm[threadIdx.x] = m;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sm[threadIdx.x] = fmaxf(sm[threadIdx.x], sm[threadIdx.x + o]);
    __syncthreads();
  }
  const float M = sm[0];
  __syncthreads();
  float e = 0.f;
  for (int c = threadIdx.x; c < V; c += 256) e += expf(x[c] - M);
  sm[threadIdx.x] = e;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o];
    __syncthreads();
  }
  const float lse = M + logf(sm[0]);
  const int tg = (int)targets[row];
  const float t = 1.f - ls, u = ls / (float)(V - 1), sc = gout[0] * scale;
  for (long long c = threadIdx.x; c < ld_out; c += 256) {
    const float v = c < V ? (expf(x[c] - lse) - (c == tg ? t : u)) * sc : 0.f;
    out[row * ld_out + c] = v;
    split_f16(v, hi[row * ld_out + c], lo[row * ld_out + c]);
  }
}

// ------------------------------------------------------------------------------------------ RMSNorm backward
// y = x r w, r = (mean x^2 + eps)^-1/2:  dx = r (w dy) - x r^3 / C * sum_c (w dy x);  gw[row, c] = dy x r (summed over rows by
// qb_col_sum for dw).  One warp per row; dx is written or added to (accumulate).
__global__ void rmsnorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ dy, float eps,
                                   long long rows, int C, float* __restrict__ dx, int accumulate, float* __restrict__ gw) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * C;
  const float* gr = dy + row * C;
  float q = 0.f, s = 0.f;
  for (int c = lane; c < C; c += 32) {
    q += xr[c] * xr[c];
    s += w[c] * gr[c] * xr[c];
  }
  q = warp_sum(q);
  s = warp_sum(s);
  const float r = rsqrtf(q / C + eps);
  const float k = r * r * r * s / C;
  for (int c = lane; c < C; c += 32) {
    const float v = r * w[c] * gr[c] - xr[c] * k;
    dx[row * C + c] = accumulate ? dx[row * C + c] + v : v;
    gw[row * C + c] = gr[c] * xr[c] * r;
  }
}

// ------------------------------------------------------------------------------------------ column sums (fixed order, fp64)
constexpr int CS_ROWS = 128;
__global__ void col_sum_part_kernel(const float* __restrict__ x, long long rows, long long C, long long ld, double* __restrict__ part) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long r0 = (long long)blockIdx.y * CS_ROWS, r1 = min(rows, r0 + CS_ROWS);
  double a = 0.0;
  for (long long r = r0; r < r1; ++r) a += x[r * ld + c];
  part[blockIdx.y * C + c] = a;
}
__global__ void col_sum_final_kernel(const double* __restrict__ part, int chunks, long long C, double scale, float* __restrict__ out,
                                     int accumulate) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double a = 0.0;
  for (int k = 0; k < chunks; ++k) a += part[k * C + c];
  out[c] = accumulate ? out[c] + (float)(a * scale) : (float)(a * scale);
}

// ------------------------------------------------------------------------------------------ SwiGLU
// gu [M, 2I] fp32 with (gate, up) interleaved per output column (the packed gate / up weight rows); h = silu(gate) * up
__global__ void swiglu_kernel(const float2* __restrict__ gu, long long n, float* __restrict__ h, __half* __restrict__ hi,
                              __half* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float2 v = gu[i];
    const float y = silu_f(v.x) * v.y;
    h[i] = y;
    split_f16(y, hi[i], lo[i]);
  }
}
// d gate = dh * up * silu'(gate), silu'(g) = s (1 + g (1 - s)), s = sigmoid(g);  d up = dh * silu(gate)
__global__ void swiglu_bwd_kernel(const float2* __restrict__ gu, const float* __restrict__ dh, long long n, float2* __restrict__ dgu,
                                  __half2* __restrict__ hi, __half2* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float2 v = gu[i];
    const float s = 1.f / (1.f + expf(-v.x));
    const float d = dh[i];
    const float2 r = make_float2(d * v.y * s * (1.f + v.x * (1.f - s)), d * v.x * s);
    dgu[i] = r;
    __half h0, h1, l0, l1;
    split_f16(r.x, h0, l0);
    split_f16(r.y, h1, l1);
    hi[i] = __halves2half2(h0, h1);
    lo[i] = __halves2half2(l0, l1);
  }
}

// ------------------------------------------------------------------------------------------ transposing split
// x [rows, cols] fp32 (row pitch ldx) -> planes out[s][c][k] = x[s * ks + k][c], rows past `rows` zero: feature-major operands of
// a weight gradient, cut along the token axis into slices of ks (a multiple of 64) for split-K.
__global__ void transpose_split_kernel(const float* __restrict__ x, long long rows, int cols, long long ldx, long long ks, long long rows_pad,
                                       __half* __restrict__ hi, __half* __restrict__ lo) {
  __shared__ float t[32][33];
  const int c0 = blockIdx.x * 32;
  const long long r0 = (long long)blockIdx.y * 32;
  for (int yy = threadIdx.y; yy < 32; yy += 8) {
    const long long r = r0 + yy;
    const int c = c0 + threadIdx.x;
    t[yy][threadIdx.x] = (r < rows && c < cols) ? x[r * ldx + c] : 0.f;
  }
  __syncthreads();
  for (int yy = threadIdx.y; yy < 32; yy += 8) {
    const int c = c0 + yy;
    const long long r = r0 + threadIdx.x;
    if (c < cols && r < rows_pad) {
      const long long s = r / ks, k = r % ks;
      const long long o = (s * cols + c) * ks + k;
      __half h, l;
      split_f16(t[threadIdx.x][yy], h, l);
      hi[o] = h;
      lo[o] = l;
    }
  }
}

// ------------------------------------------------------------------------------------------ embedding backward
// out[v, :] (+)= scale * sum over the positions k with ids[k] == v, in increasing k, of dx[row(k), :] with row(k) = (k / Lt) * L + P + k % Lt.
// One block per id: it walks the ids in chunks of 256 and compacts the matches in order (warp ballots), then sums their rows in fp64.
__global__ void __launch_bounds__(256)
embedding_bwd_kernel(const float* __restrict__ dx, const int64_t* __restrict__ ids, long long n, long long Lt, long long L, long long P,
                     int H, double scale, float* __restrict__ out, int accumulate) {
  __shared__ long long srow[256];
  __shared__ int wcount[8];
  const int v = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long base = 0; base < n; base += 256) {
    const long long k = base + tid;
    const bool hit = k < n && ids[k] == v;
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wcount[w] = __popc(bal);
    __syncthreads();
    int off = 0, total = 0;
    for (int q = 0; q < 8; ++q) {
      if (q < w) off += wcount[q];
      total += wcount[q];
    }
    if (hit) srow[off + __popc(bal & ((1u << lane) - 1u))] = (k / Lt) * L + P + k % Lt;
    __syncthreads();
    for (int e = 0; e < total; ++e) {
      const float* r = dx + srow[e] * H;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = tid + 256 * u;
        if (c < H) acc[u] += r[c];
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int c = tid + 256 * u;
    if (c < H) {
      float* o = out + (long long)v * H + c;
      *o = accumulate ? *o + (float)(acc[u] * scale) : (float)(acc[u] * scale);
    }
  }
}

static DropCfg drop_cfg(float p, uint64_t seed, int32_t layer) {
  DropCfg dc;
  dc.k0 = (uint32_t)(seed & 0xFFFFFFFFu);
  dc.k1 = (uint32_t)(seed >> 32);
  dc.thr = (uint32_t)llrint((double)p * 16777216.0);
  dc.layer = (uint32_t)layer;
  dc.keep_scale = 1.f / (1.f - p);
  return dc;
}

}  // namespace qb

using namespace qb;

extern "C" int qb_lm_attn_train_fwd(const float* qkv, int64_t B, int64_t L, int32_t heads, const float* rope_cos, const float* rope_sin,
                                    float dropout_p, uint64_t seed, int32_t layer, float* qs, float* kr, float* v, float* out, float* lse,
                                    void* stream) {
  QB_REQUIRE(qkv && rope_cos && rope_sin && qs && kr && v && out && lse, "lm_attn_train_fwd: null pointer");
  QB_REQUIRE(B >= 1 && L >= 1 && heads >= 1 && B * heads <= 65535, "lm_attn_train_fwd: bad shape");
  QB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "lm_attn_train_fwd: dropout_p must lie in [0, 1)");
  cudaStream_t st = (cudaStream_t)stream;
  lm_train_qkv_kernel<<<(unsigned)(B * L), 256, 0, st>>>(qkv, (int)L, heads, rope_cos, rope_sin, qs, kr, v);
  lm_attn_train_fwd_kernel<<<dim3((unsigned)ceil_div(L, AT), (unsigned)(B * heads)), 256, 0, st>>>(
      qs, kr, v, (int)L, heads, drop_cfg(dropout_p, seed, layer), out, lse);
  QB_TRAIN_LAUNCHED(2);
}

extern "C" int qb_lm_attn_train_bwd(const float* qs, const float* kr, const float* v, const float* out, const float* dout, const float* lse,
                                    int64_t B, int64_t L, int32_t heads, const float* rope_cos, const float* rope_sin, float dropout_p,
                                    uint64_t seed, int32_t layer, float* dqkv, float* workspace, void* stream) {
  QB_REQUIRE(qs && kr && v && out && dout && lse && rope_cos && rope_sin && dqkv && workspace, "lm_attn_train_bwd: null pointer");
  QB_REQUIRE(B >= 1 && L >= 1 && heads >= 1 && B * heads <= 65535, "lm_attn_train_bwd: bad shape");
  QB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "lm_attn_train_bwd: dropout_p must lie in [0, 1)");
  cudaStream_t st = (cudaStream_t)stream;
  const DropCfg dc = drop_cfg(dropout_p, seed, layer);
  lm_attn_bwd_dot_kernel<<<(unsigned)ceil_div(B * L * heads, 8), 256, 0, st>>>(out, dout, (int)L, heads, B * L, workspace);
  const dim3 grid((unsigned)ceil_div(L, AT), (unsigned)(B * heads));
  lm_attn_train_dkv_kernel<<<grid, 256, 0, st>>>(qs, kr, v, dout, lse, workspace, (int)L, heads, rope_cos, rope_sin, dc, dqkv);
  lm_attn_train_dq_kernel<<<grid, 256, 0, st>>>(qs, kr, v, dout, lse, workspace, (int)L, heads, rope_cos, rope_sin, dc, dqkv);
  QB_TRAIN_LAUNCHED(3);
}

extern "C" int qb_lm_loss_bwd(const float* logits, int64_t ld, int64_t M, int32_t V, const int64_t* targets, float label_smoothing,
                              const float* grad_loss, float scale, float* out, qb_half* out_hi, qb_half* out_lo, int64_t ld_out,
                              void* stream) {
  QB_REQUIRE(logits && targets && grad_loss && out && out_hi && out_lo && M >= 1 && V >= 2 && ld >= V && ld_out >= V,
             "lm_loss_bwd: bad args");
  lm_loss_bwd_kernel<<<(unsigned)M, 256, 0, (cudaStream_t)stream>>>(logits, ld, V, targets, label_smoothing, grad_loss, scale,
                                                                     ld_out, out, (__half*)out_hi, (__half*)out_lo);
  QB_TRAIN_LAUNCHED(1);
}

extern "C" int qb_rmsnorm_bwd(const float* x, const float* w, const float* dy, float eps, int64_t rows, int64_t C, float* dx,
                              int32_t accumulate, float* gw, void* stream) {
  QB_REQUIRE(x && w && dy && dx && gw && rows >= 1 && C >= 1, "rmsnorm_bwd: bad args");
  rmsnorm_bwd_kernel<<<(unsigned)ceil_div(rows, 8), 256, 0, (cudaStream_t)stream>>>(x, w, dy, eps, rows, (int)C, dx, accumulate, gw);
  QB_TRAIN_LAUNCHED(1);
}

extern "C" int64_t qb_col_sum_workspace_bytes(int64_t rows, int64_t C) { return ceil_div(rows, CS_ROWS) * C * (int64_t)sizeof(double); }

extern "C" int qb_col_sum(const float* x, int64_t rows, int64_t C, int64_t ld, double scale, void* workspace, float* out,
                          int32_t accumulate, void* stream) {
  QB_REQUIRE(x && workspace && out && rows >= 1 && C >= 1 && ld >= C, "col_sum: bad args");
  QB_REQUIRE(ceil_div(rows, CS_ROWS) <= 65535, "col_sum: too many rows (%lld)", (long long)rows);
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = (int)ceil_div(rows, CS_ROWS);
  col_sum_part_kernel<<<dim3((unsigned)ceil_div(C, 256), (unsigned)chunks), 256, 0, st>>>(x, rows, C, ld, (double*)workspace);
  col_sum_final_kernel<<<(unsigned)ceil_div(C, 256), 256, 0, st>>>((const double*)workspace, chunks, C, scale, out, accumulate);
  QB_TRAIN_LAUNCHED(2);
}

extern "C" int qb_swiglu(const float* gu, int64_t M, int64_t inter, float* h, qb_half* hi, qb_half* lo, void* stream) {
  QB_REQUIRE(gu && h && hi && lo && M >= 1 && inter >= 1, "swiglu: bad args");
  const long long n = M * inter;
  swiglu_kernel<<<(unsigned)std::min<long long>(ceil_div(n, 256), 4096), 256, 0, (cudaStream_t)stream>>>(
      (const float2*)gu, n, h, (__half*)hi, (__half*)lo);
  QB_TRAIN_LAUNCHED(1);
}

extern "C" int qb_swiglu_bwd(const float* gu, const float* dh, int64_t M, int64_t inter, float* dgu, qb_half* hi, qb_half* lo,
                             void* stream) {
  QB_REQUIRE(gu && dh && dgu && hi && lo && M >= 1 && inter >= 1, "swiglu_bwd: bad args");
  const long long n = M * inter;
  swiglu_bwd_kernel<<<(unsigned)std::min<long long>(ceil_div(n, 256), 4096), 256, 0, (cudaStream_t)stream>>>(
      (const float2*)gu, dh, n, (float2*)dgu, (__half2*)hi, (__half2*)lo);
  QB_TRAIN_LAUNCHED(1);
}

extern "C" int qb_transpose_split(const float* x, int64_t rows, int64_t cols, int64_t ldx, int64_t ks, qb_half* hi, qb_half* lo,
                                  void* stream) {
  QB_REQUIRE(x && hi && lo && rows >= 1 && cols >= 1 && ldx >= cols && ks >= 64 && ks % 64 == 0, "transpose_split: bad args");
  const long long rows_pad = ceil_div(rows, ks) * ks;
  QB_REQUIRE(ceil_div(rows_pad, 32) <= 65535, "transpose_split: too many rows (%lld)", (long long)rows);
  transpose_split_kernel<<<dim3((unsigned)ceil_div(cols, 32), (unsigned)ceil_div(rows_pad, 32)), dim3(32, 8), 0, (cudaStream_t)stream>>>(
      x, rows, (int)cols, ldx, ks, rows_pad, (__half*)hi, (__half*)lo);
  QB_TRAIN_LAUNCHED(1);
}

extern "C" int qb_embedding_bwd(const float* dx, const int64_t* ids, int64_t n, int64_t Lt, int64_t L, int64_t P, int32_t H, int32_t V,
                                double scale, float* out, int32_t accumulate, void* stream) {
  QB_REQUIRE(dx && ids && out && n >= 1 && Lt >= 1 && L >= P + Lt && H >= 1 && H <= 1024 && V >= 1, "embedding_bwd: bad args");
  embedding_bwd_kernel<<<(unsigned)V, 256, 0, (cudaStream_t)stream>>>(dx, ids, n, Lt, L, P, H, scale, out, accumulate);
  QB_TRAIN_LAUNCHED(1);
}
