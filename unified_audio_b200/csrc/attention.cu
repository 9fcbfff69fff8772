// Non-causal multi-head self-attention with fused RoPE, head_dim 64
// (reference: HCodec-2.0/vq/encoder_modules/transformer.py:134-215).
// v1: fp32 SIMT flash-style kernel - one thread per query row (q, o in registers), K/V tiles of 32
// keys staged in shared memory and read as warp-wide broadcasts.  Attention is ~0.5 % of the path's
// FLOPs; the tensor-core version is attention_umma.cu.
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

extern "C" int qb_attention(const float* qkv, int64_t B, int64_t T, int32_t heads, const float* rope_cos,
                            const float* rope_sin, qb_half* out_hi, qb_half* out_lo, void* stream) {
  return qb_attention_hd(qkv, B, T, heads, 64, rope_cos, rope_sin, out_hi, out_lo, stream);
}

// =====================================================================================================
// Tensor-core path (single-pass fp16 policy): qkv_prep (RoPE + 1/sqrt(d) + fp16, head-major layout)
// followed by a flash-attention forward on mma.sync m16n8k16 (fp16 in, fp32 softmax/accumulate).
// Block = 4 warps x 16 query rows; K/V tiles of 64 keys staged in shared memory (144 B row pitch keeps
// ldmatrix conflict-free); P stays in registers (S-accumulator layout == A-fragment layout).
// =====================================================================================================
namespace qb {

__global__ void qkv_prep_kernel(const float* __restrict__ qkv, int T, int H, const float* __restrict__ rcos,
                                const float* __restrict__ rsin, __half* __restrict__ q16, __half* __restrict__ k16,
                                __half* __restrict__ v16, long long total) {
  // one thread per (b, t, h, d < 32)
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int d = (int)(i & 31);
  long long r = i >> 5;
  const int h = (int)(r % H);
  r /= H;
  const int t = (int)(r % T);
  const long long b = r / T;
  const float* base = qkv + (b * T + t) * 3LL * H * 64 + h * 64;
  const float c1 = rcos[t * 64 + d], s1 = rsin[t * 64 + d], c2 = rcos[t * 64 + d + 32], s2 = rsin[t * 64 + d + 32];
  const long long o = ((b * H + h) * T + t) * 64 + d;
  {
    const float x1 = base[d], x2 = base[d + 32];
    q16[o] = __float2half_rn((x1 * c1 - x2 * s1) * 0.125f);
    q16[o + 32] = __float2half_rn((x2 * c2 + x1 * s2) * 0.125f);
  }
  {
    const float x1 = base[H * 64 + d], x2 = base[H * 64 + d + 32];
    k16[o] = __float2half_rn(x1 * c1 - x2 * s1);
    k16[o + 32] = __float2half_rn(x2 * c2 + x1 * s2);
  }
  v16[o] = __float2half_rn(base[2 * H * 64 + d]);
  v16[o + 32] = __float2half_rn(base[2 * H * 64 + d + 32]);
}

constexpr int FA_BQ = 64, FA_BK = 64, FA_D = 64, FA_P = 72;  // pitch in halves

__device__ __forceinline__ void ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(128)
flash_attn_kernel(const __half* __restrict__ q16, const __half* __restrict__ k16, const __half* __restrict__ v16, int T,
                  int H, __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  __shared__ __align__(16) __half sq[FA_BQ * FA_P];
  __shared__ __align__(16) __half sk[FA_BK * FA_P];
  __shared__ __align__(16) __half sv[FA_BK * FA_P];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.x * FA_BQ, h = blockIdx.y, b = blockIdx.z;
  const long long head = ((long long)b * H + h) * T * FA_D;
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
  // Q tile -> smem (64 rows x 8 chunks of 16 B)
  for (int c = tid; c < FA_BQ * 8; c += 128) {
    const int r = c >> 3, ch = c & 7;
    uint4 v = (q0 + r < T) ? *reinterpret_cast<const uint4*>(q16 + head + (long long)(q0 + r) * FA_D + ch * 8) : z4;
    *reinterpret_cast<uint4*>(sq + r * FA_P + ch * 8) = v;
  }
  __syncthreads();
  uint32_t qf[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
    ldsm_x4(qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3],
            sq + (warp * 16 + (lane & 15)) * FA_P + ks * 16 + (lane >> 4) * 8);
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[j][e] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const float LOG2E = 1.4426950408889634f;

  for (int k0 = 0; k0 < T; k0 += FA_BK) {
    __syncthreads();
    for (int c = tid; c < FA_BK * 8; c += 128) {
      const int r = c >> 3, ch = c & 7;
      const bool ok = k0 + r < T;
      const long long g = head + (long long)(k0 + r) * FA_D + ch * 8;
      *reinterpret_cast<uint4*>(sk + r * FA_P + ch * 8) = ok ? *reinterpret_cast<const uint4*>(k16 + g) : z4;
      *reinterpret_cast<uint4*>(sv + r * FA_P + ch * 8) = ok ? *reinterpret_cast<const uint4*>(v16 + g) : z4;
    }
    __syncthreads();
    // S = Q K^T  (16 queries x 64 keys per warp)
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[j][e] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {   // two k-steps (32 dims) per ldmatrix.x4
        uint32_t b0, b1, b2, b3;
        // matrices: (keys 8j.., dims 32kp..+7), (.., +8..15), (.., +16..23), (.., +24..31)
        ldsm_x4(b0, b1, b2, b3, sk + (j * 8 + (lane & 7)) * FA_P + kp * 32 + (lane >> 3) * 8);
        mma16816(s[j], qf[2 * kp][0], qf[2 * kp][1], qf[2 * kp][2], qf[2 * kp][3], b0, b1);
        mma16816(s[j], qf[2 * kp + 1][0], qf[2 * kp + 1][1], qf[2 * kp + 1][2], qf[2 * kp + 1][3], b2, b3);
      }
    }
    // mask + online softmax (rows g = lane/4 and g + 8)
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int key = k0 + j * 8 + (lane & 3) * 2;
      if (key >= T) { s[j][0] = -INFINITY; s[j][2] = -INFINITY; }
      if (key + 1 >= T) { s[j][1] = -INFINITY; s[j][3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float c0 = exp2f((m0 - mn0) * LOG2E), c1 = exp2f((m1 - mn1) * LOG2E);
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = exp2f((s[j][0] - mn0) * LOG2E);
      s[j][1] = exp2f((s[j][1] - mn0) * LOG2E);
      s[j][2] = exp2f((s[j][2] - mn1) * LOG2E);
      s[j][3] = exp2f((s[j][3] - mn1) * LOG2E);
      rs0 += s[j][0] + s[j][1];
      rs1 += s[j][2] + s[j][3];
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
    m0 = mn0;
    m1 = mn1;
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] *= c0; o[j][1] *= c0; o[j][2] *= c1; o[j][3] *= c1; }
    // O += P V   (P from registers: S layout == A-fragment layout)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint32_t a0 = pack_h2(s[2 * ks][0], s[2 * ks][1]), a1 = pack_h2(s[2 * ks][2], s[2 * ks][3]);
      const uint32_t a2 = pack_h2(s[2 * ks + 1][0], s[2 * ks + 1][1]), a3 = pack_h2(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {   // two dim-tiles (16 dims) per ldmatrix.x4.trans
        uint32_t b0, b1, b2, b3;
        // matrices: (keys 16ks..+7, dims 16jp..+7), (keys +8..15, same dims), (keys ..+7, dims +8..15), (keys +8.., dims +8..)
        ldsm_x4_t(b0, b1, b2, b3, sv + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * FA_P + jp * 16 + (lane >> 4) * 8);
        mma16816(o[2 * jp], a0, a1, a2, a3, b0, b1);
        mma16816(o[2 * jp + 1], a0, a1, a2, a3, b2, b3);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = j * 8 + (lane & 3) * 2;
    if (r0 < T) {
      const long long off = ((long long)b * T + r0) * (long long)(H * FA_D) + h * FA_D + d;
      __half ha, hb, la, lb;
      split_f16(o[j][0] * i0, ha, la);
      split_f16(o[j][1] * i0, hb, lb);
      *reinterpret_cast<__half2*>(out_hi + off) = __halves2half2(ha, hb);
      if (out_lo) *reinterpret_cast<__half2*>(out_lo + off) = __halves2half2(la, lb);
    }
    if (r1 < T) {
      const long long off = ((long long)b * T + r1) * (long long)(H * FA_D) + h * FA_D + d;
      __half ha, hb, la, lb;
      split_f16(o[j][2] * i1, ha, la);
      split_f16(o[j][3] * i1, hb, lb);
      *reinterpret_cast<__half2*>(out_hi + off) = __halves2half2(ha, hb);
      if (out_lo) *reinterpret_cast<__half2*>(out_lo + off) = __halves2half2(la, lb);
    }
  }
}

}  // namespace qb

extern "C" int64_t qb_attention_tc_workspace_bytes(int64_t B, int64_t T, int32_t heads) {
  return 3 * B * heads * T * 64 * 2 + 256;
}

extern "C" int qb_attention_tc(const float* qkv, int64_t B, int64_t T, int32_t heads, const float* rope_cos,
                               const float* rope_sin, qb_half* out_hi, qb_half* out_lo, void* workspace, void* stream) {
  QB_REQUIRE(qkv && rope_cos && rope_sin && out_hi && workspace && T > 0 && heads > 0, "attention_tc: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const long long per = B * heads * T * 64;
  __half* q16 = (__half*)workspace;
  __half* k16 = q16 + per;
  __half* v16 = k16 + per;
  const long long total = B * T * heads * 32;
  qkv_prep_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(qkv, (int)T, heads, rope_cos, rope_sin, q16, k16, v16,
                                                                 total);
  g_launches++;
  dim3 grid((unsigned)ceil_div(T, FA_BQ), (unsigned)heads, (unsigned)B);
  flash_attn_kernel<<<grid, 128, 0, st>>>(q16, k16, v16, (int)T, heads, (__half*)out_hi, (__half*)out_lo);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
