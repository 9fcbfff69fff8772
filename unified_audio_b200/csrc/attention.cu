// fp32 SIMT non-causal multi-head self-attention with fused RoPE (reference: HCodec-2.0/vq/encoder_modules/transformer.py:134-215)
// and WavLM's gated relative-position bias.  attention_kernel<D, KT, PARTS> is flash-style: PARTS threads per query row (q, o in
// registers), K/V tiles of KT keys staged in shared memory and read as warp-wide broadcasts.  Self-attention at head_dim 64 / 128
// runs on the wgmma kernel (attention_umma.cu); this one serves what that kernel does not: head_dim 96 (H-Codec-1.0's decoder) and
// the WavLM bias (head_dim 64, qb_attention_relbias).  At head_dim 64 and 128 it is the fp32 reference the wgmma kernel is tested
// against.
#include <atomic>
#include <vector>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

constexpr int ATT_THREADS = 128;

// PARTS threads share one query row, each owning D / PARTS of the head dims (q, o in registers: D = 128 would not fit one thread);
// the partial dot products are summed across the PARTS adjacent lanes.
template <int D, int KT, int PARTS = 1>
__global__ void __launch_bounds__(ATT_THREADS)
attention_kernel(const float* __restrict__ qkv, int T, int H, const float* __restrict__ rcos,
                 const float* __restrict__ rsin, float scale, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                 const float* __restrict__ rel_table = nullptr, const float* __restrict__ gate = nullptr) {
  constexpr int HD = D / 2, DP = D / PARTS, ROWS = ATT_THREADS / PARTS;
  static_assert(PARTS == 1 || PARTS == 2 || PARTS == 4, "PARTS lanes must sit in one warp");
  __shared__ __align__(16) float ks[KT][D];
  __shared__ __align__(16) float vs[KT][D];
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int part = threadIdx.x % PARTS, d0 = part * DP;
  const int tq = qt * ROWS + threadIdx.x / PARTS;
  const long long pitch = 3LL * H * D;
  const float* base = qkv + (long long)b * T * pitch;
  const bool active = tq < T;

  float q[DP], o[DP];
  if (active) {
    const float* qp = base + (long long)tq * pitch + h * D;
    const float* c = rcos + (long long)tq * D;
    const float* s = rsin + (long long)tq * D;
#pragma unroll
    for (int j = 0; j < DP; ++j) {                          // q*cos + rotate_half(q)*sin, then * head_dim^-0.5
      const int d = d0 + j;
      const float x = qp[d], y = d < HD ? -qp[d + HD] : qp[d - HD];
      q[j] = (x * c[d] + y * s[d]) * scale;
    }
  } else {
#pragma unroll
    for (int j = 0; j < DP; ++j) q[j] = 0.f;
  }
#pragma unroll
  for (int j = 0; j < DP; ++j) o[j] = 0.f;
  float m = -INFINITY, l = 0.f;
  // WavLM gated relative position bias (transformers modeling_wavlm.WavLMAttention): score[i, j] += gate[b, h, i] * table[h, j - i]
  const float gq = (rel_table && active) ? gate[((long long)b * H + h) * T + tq] : 0.f;
  const float* relrow = rel_table ? rel_table + (long long)h * (2 * T - 1) + (T - 1) - (active ? tq : 0) : nullptr;

  for (int k0 = 0; k0 < T; k0 += KT) {
    __syncthreads();
    for (int e = threadIdx.x; e < KT * HD; e += ATT_THREADS) {
      const int j = e / HD, d = e - j * HD, tk = k0 + j;
      float k1 = 0.f, k2 = 0.f, v1 = 0.f, v2 = 0.f;
      if (tk < T) {
        const float* kp = base + (long long)tk * pitch + (H + h) * D;
        const float* vp = base + (long long)tk * pitch + (2 * H + h) * D;
        const float x1 = kp[d], x2 = kp[d + HD];
        const float* c = rcos + (long long)tk * D;
        const float* s = rsin + (long long)tk * D;
        k1 = x1 * c[d] - x2 * s[d];
        k2 = x2 * c[d + HD] + x1 * s[d + HD];
        v1 = vp[d];
        v2 = vp[d + HD];
      }
      ks[j][d] = k1; ks[j][d + HD] = k2;
      vs[j][d] = v1; vs[j][d + HD] = v2;
    }
    __syncthreads();
    float sc[KT];
    float tmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < KT; ++j) {
      float acc = 0.f;
      const float4* kr = reinterpret_cast<const float4*>(ks[j] + d0);
#pragma unroll
      for (int d4 = 0; d4 < DP / 4; ++d4) {
        float4 kk = kr[d4];
        acc = fmaf(q[4 * d4], kk.x, acc);
        acc = fmaf(q[4 * d4 + 1], kk.y, acc);
        acc = fmaf(q[4 * d4 + 2], kk.z, acc);
        acc = fmaf(q[4 * d4 + 3], kk.w, acc);
      }
      if (PARTS > 1) acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      if (PARTS > 2) acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      if (relrow && k0 + j < T) acc = fmaf(gq, relrow[k0 + j], acc);
      sc[j] = (k0 + j < T) ? acc : -INFINITY;
      tmax = fmaxf(tmax, sc[j]);
    }
    const float m_new = fmaxf(m, tmax);
    const float corr = expf(m - m_new);   // m = -inf on the first tile -> 0
    l *= corr;
#pragma unroll
    for (int j = 0; j < DP; ++j) o[j] *= corr;
#pragma unroll
    for (int j = 0; j < KT; ++j) {
      const float pj = expf(sc[j] - m_new);
      l += pj;
      const float4* vr = reinterpret_cast<const float4*>(vs[j] + d0);
#pragma unroll
      for (int d4 = 0; d4 < DP / 4; ++d4) {
        float4 vv = vr[d4];
        o[4 * d4] = fmaf(pj, vv.x, o[4 * d4]);
        o[4 * d4 + 1] = fmaf(pj, vv.y, o[4 * d4 + 1]);
        o[4 * d4 + 2] = fmaf(pj, vv.z, o[4 * d4 + 2]);
        o[4 * d4 + 3] = fmaf(pj, vv.w, o[4 * d4 + 3]);
      }
    }
    m = m_new;
  }
  if (active) {
    const float inv = 1.f / l;
    const long long ob = ((long long)b * T + tq) * (long long)(H * D) + h * D + d0;
#pragma unroll
    for (int j = 0; j < DP; ++j) {
      __half hh, ll;
      split_f16(o[j] * inv, hh, ll);
      out_hi[ob + j] = hh;
      if (out_lo) out_lo[ob + j] = ll;
    }
  }
}

// gate[b, h, t] = ga * (gb * const_h - 1) + 2 with (ga, gb) = sigmoid(sum over groups of 4 of Linear(d -> 8)(x[b, t, head h]))
// (WavLMAttention.forward: gru_rel_pos_linear / gru_rel_pos_const on the layer INPUT)
__global__ void wavlm_gate_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                  const float* __restrict__ cst, int T, int H, int D, float* __restrict__ gate, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int h = (int)(i % H);
  const long long bt = i / H;
  const int t = (int)(bt % T);
  const long long b = bt / T;
  const float* xp = x + bt * (long long)(H * D) + h * D;
  float p[8];
#pragma unroll
  for (int o = 0; o < 8; ++o) {
    float acc = bias[o];
    for (int d = 0; d < D; ++d) acc = fmaf(xp[d], w[o * D + d], acc);
    p[o] = acc;
  }
  const float ga = 1.f / (1.f + expf(-(p[0] + p[1] + p[2] + p[3])));
  const float gb = 1.f / (1.f + expf(-(p[4] + p[5] + p[6] + p[7])));
  gate[(b * H + h) * T + t] = ga * (gb * cst[h] - 1.f) + 2.f;
}

}  // namespace qb
using namespace qb;

extern "C" int qb_wavlm_gate(const float* x, int64_t B, int64_t T, int32_t heads, int32_t head_dim, const float* w, const float* bias,
                             const float* cst, float* gate, void* stream) {
  QB_REQUIRE(x && w && bias && cst && gate, "wavlm_gate: bad args");
  const long long total = B * T * heads;
  wavlm_gate_kernel<<<(unsigned)ceil_div(total, 128), 128, 0, (cudaStream_t)stream>>>(x, w, bias, cst, (int)T, heads, head_dim, gate, total);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_attention_relbias(const float* qkv, int64_t B, int64_t T, int32_t heads, int32_t head_dim, const float* rel_table,
                                    const float* gate, qb_half* out_hi, qb_half* out_lo, void* stream) {
  QB_REQUIRE(qkv && rel_table && gate && out_hi && T > 0 && heads > 0, "attention_relbias: bad args");
  QB_REQUIRE(head_dim == 64, "attention_relbias: head_dim must be 64 (got %d)", head_dim);
  // no rotary embedding in WavLM: identity tables (cos = 1, sin = 0) kept in a per-process device buffer of T*64 floats
  static float* ident[2] = {nullptr, nullptr};
  static int64_t ident_rows = 0;
  if (ident_rows < T) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing((cudaStream_t)stream, &cs);
    QB_REQUIRE(cs == cudaStreamCaptureStatusNone, "attention_relbias: first call for this length must happen outside stream capture");
    const int64_t rows = (T + 1023) / 1024 * 1024;
    if (ident[0]) { cudaFree(ident[0]); cudaFree(ident[1]); }
    QB_CHECK_CUDA(cudaMalloc(&ident[0], (size_t)rows * 64 * 4));
    QB_CHECK_CUDA(cudaMalloc(&ident[1], (size_t)rows * 64 * 4));
    std::vector<float> ones((size_t)rows * 64, 1.0f);
    QB_CHECK_CUDA(cudaMemcpy(ident[0], ones.data(), ones.size() * 4, cudaMemcpyHostToDevice));
    QB_CHECK_CUDA(cudaMemset(ident[1], 0, (size_t)rows * 64 * 4));
    ident_rows = rows;
  }
  dim3 grid((unsigned)ceil_div(T, ATT_THREADS), (unsigned)heads, (unsigned)B);
  attention_kernel<64, 32><<<grid, ATT_THREADS, 0, (cudaStream_t)stream>>>(qkv, (int)T, heads, ident[0], ident[1], 0.125f, (__half*)out_hi,
                                                                         (__half*)out_lo, rel_table, gate);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_attention_hd(const float* qkv, int64_t B, int64_t T, int32_t heads, int32_t head_dim, const float* rope_cos,
                               const float* rope_sin, qb_half* out_hi, qb_half* out_lo, void* stream) {
  QB_REQUIRE(qkv && rope_cos && rope_sin && out_hi && T > 0 && heads > 0, "attention: bad args");
  QB_REQUIRE(head_dim == 64 || head_dim == 96 || head_dim == 128, "attention: head_dim must be 64, 96 or 128 (got %d)", head_dim);
  dim3 grid((unsigned)ceil_div(T, ATT_THREADS), (unsigned)heads, (unsigned)B);
  const float scale = 1.0f / sqrtf((float)head_dim);
  if (head_dim == 128) {
    grid.x = (unsigned)ceil_div(T, ATT_THREADS / 2);
    attention_kernel<128, 16, 2><<<grid, ATT_THREADS, 0, (cudaStream_t)stream>>>(qkv, (int)T, heads, rope_cos, rope_sin, scale,
                                                                               (__half*)out_hi, (__half*)out_lo);
  } else if (head_dim == 64)
    attention_kernel<64, 32><<<grid, ATT_THREADS, 0, (cudaStream_t)stream>>>(qkv, (int)T, heads, rope_cos, rope_sin, scale,
                                                                           (__half*)out_hi, (__half*)out_lo);
  else
    attention_kernel<96, 16><<<grid, ATT_THREADS, 0, (cudaStream_t)stream>>>(qkv, (int)T, heads, rope_cos, rope_sin, scale,
                                                                           (__half*)out_hi, (__half*)out_lo);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
