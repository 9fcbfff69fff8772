// Non-causal multi-head self-attention on the Hopper tensor cores (wgmma + TMA + mbarrier), head_dim 64 / 128, with the library's
// two precision policies: single-pass fp16 operands, or the fp16 hi + lo split (3 tensor-core passes, fp32-grade) for both
// contractions.  Callers: the LSTM-transformers of the codecs (HCodec-2.0/vq/encoder_modules/transformer.py:134-215), the SSL front
// ends, and the 96 mimi transformer layers of H-Codec-1.5 (HCodec-1.5/adaptive/model_blocks/mimi/transformer.py:377-424).
//
// Two launches:
//  1. fa5_prep_kernel: qkv fp32 [B*L, 3*H*D] (the in_proj GEMM's output) -> RoPE (rotate-half tables) + 1/sqrt(D) on q -> fp16 hi (+ lo)
//     planes in the operand layouts the MMAs want, all K-major:  Q [plane*B*H + bh][L][D],  K likewise,  V TRANSPOSED [..][D][Lp]
//     (P.V contracts over keys, so V is the B operand [N = D rows] x [K = keys]).
//  2. fa5_kernel: one CTA = 128 queries of one (batch, head).  Warpgroup 0 (one thread) = TMA producer: Q once, K and V tiles of 64
//     keys double-buffered.  Warpgroups 1 and 2 each own 64 query rows.  Per key tile j:
//        S_j   = Q K_j^T            wgmma m64n64k16 from shared memory into registers (split: hi.hi + lo.hi + hi.lo per K step)
//        P_j   = exp2(S_j - m)      in registers, fp16 hi (+ lo) packed directly into the A-operand fragments of the next MMA
//        O    += P_j V_j            wgmma m64nDk16 with A from registers, accumulated in registers over ALL key tiles.
//     The reference maximum m of a row only moves when a tile exceeds it by 2^8 (P stays < 2^8: exact in fp16 hi + lo); only then are
//     that row's O accumulators and running sum rescaled.  causal = 1 skips the key tiles right of the diagonal and masks inside the
//     diagonal ones (AR-LM prefill).  Shared memory: head_dim 128 split = 192 KB, one CTA per SM.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cuda.h>

#include "common.cuh"
#include "quark_b200.h"
#include "wgmma.cuh"

namespace qb {
extern std::atomic<long long> g_launches;

constexpr int F5_BQ = 128, F5_BK = 64, F5_THREADS = 3 * 128;
constexpr float F5_RESCALE_LOG2 = 8.0f;      // the running reference max moves only when a tile exceeds it by 2^8 (P stays < 2^8: exact in fp16 hi + lo)

__device__ __forceinline__ float f5_ex2(float x) {        // ex2.approx: 2^-22 relative, one MUFU instruction (exp2f adds a denormal-range fix-up)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ---------------------------------------------------------------------------------------------- prep
// grid (ceil(L / 32), H, B), 256 threads.  q16 / k16: [(plane * BH + bh) * L + t] * D + d;  vT: [(plane * BH + bh) * D + d] * Lp + t.
template <int D>
__global__ void __launch_bounds__(256)
fa5_prep_kernel(const float* __restrict__ qkv, int L, int Lp, int H, const float* __restrict__ rcos, const float* __restrict__ rsin,
                float scale, __half* __restrict__ q16, __half* __restrict__ k16, __half* __restrict__ vT, int planes) {
  constexpr int HD = D / 2;
  __shared__ float vs[32][D + 1];
  const int t0 = blockIdx.x * 32, h = blockIdx.y, b = blockIdx.z;
  const long long BH = (long long)gridDim.z * H, bh = (long long)b * H + h;
  const long long pitch = 3LL * H * D;
  const float* base = qkv + (long long)b * L * pitch;
  for (int e = threadIdx.x; e < 32 * HD; e += 256) {
    const int tt = e / HD, d = e - tt * HD, t = t0 + tt;
    if (t >= L) continue;
    const float* row = base + (long long)t * pitch;
    const float c1 = rcos[(long long)t * D + d], s1 = rsin[(long long)t * D + d];
    const float c2 = rcos[(long long)t * D + d + HD], s2 = rsin[(long long)t * D + d + HD];
    const float q1 = row[h * D + d], q2 = row[h * D + d + HD];
    const float k1 = row[(H + h) * D + d], k2 = row[(H + h) * D + d + HD];
    const float qa = (q1 * c1 - q2 * s1) * scale, qb_ = (q2 * c2 + q1 * s2) * scale;
    const float ka = k1 * c1 - k2 * s1, kb = k2 * c2 + k1 * s2;
    const long long o = (bh * L + t) * D + d, po = BH * L * D;
    __half hh, ll;
    split_f16(qa, hh, ll); q16[o] = hh; if (planes == 2) q16[po + o] = ll;
    split_f16(qb_, hh, ll); q16[o + HD] = hh; if (planes == 2) q16[po + o + HD] = ll;
    split_f16(ka, hh, ll); k16[o] = hh; if (planes == 2) k16[po + o] = ll;
    split_f16(kb, hh, ll); k16[o + HD] = hh; if (planes == 2) k16[po + o + HD] = ll;
  }
  for (int e = threadIdx.x; e < 32 * D; e += 256) {
    const int tt = e / D, d = e - tt * D, t = t0 + tt;
    vs[tt][d] = t < L ? base[(long long)t * pitch + (2 * H + h) * D + d] : 0.f;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 32 * D; e += 256) {
    const int d = e >> 5, tt = e & 31, t = t0 + tt;
    if (t >= L) continue;
    __half hh, ll;
    split_f16(vs[tt][d], hh, ll);
    const long long o = (bh * D + d) * Lp + t;
    vT[o] = hh;
    if (planes == 2) vT[BH * D * Lp + o] = ll;
  }
}

// ---------------------------------------------------------------------------------------------- attention
template <int D, bool SPLIT>
struct F5Cfg {
  static constexpr int NPL = SPLIT ? 2 : 1, KBQ = D / 64;
  static constexpr uint32_t Q_KB = F5_BQ * 128, K_KB = F5_BK * 128;          // bytes of one 64-wide K-block of Q / of K
  static constexpr uint32_t Q_PLANE = KBQ * Q_KB, K_PLANE = KBQ * K_KB, V_PLANE = D * 128;
  static constexpr uint32_t K_SLOT = NPL * K_PLANE, V_SLOT = NPL * V_PLANE;   // K and V double-buffered
  static constexpr uint32_t OFF_Q = 0, OFF_K = OFF_Q + NPL * Q_PLANE, OFF_V = OFF_K + 2 * K_SLOT;
  static constexpr uint32_t OFF_BAR = OFF_V + 2 * V_SLOT;
  static constexpr uint32_t SMEM = OFF_BAR + 128 + 1024;                      // + barriers + slack for a 1024-byte-aligned base
  static_assert(SMEM <= 227 * 1024, "attention tile exceeds the 227 KB of shared memory a block may use");
};

template <int D, bool SPLIT>
__global__ void __launch_bounds__(F5_THREADS, 1)
fa5_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
           int L, int H, int BH, int causal, __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  using C = F5Cfg<D, SPLIT>;
  constexpr int NPL = C::NPL, KBQ = C::KBQ;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = (uint64_t*)(smem + C::OFF_BAR);
  uint64_t *q_full = bars, *k_full = bars + 1 /* [2] */, *k_empty = bars + 3 /* [2] */, *v_full = bars + 5 /* [2] */,
           *v_empty = bars + 7 /* [2] */;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int q0 = blockIdx.x * F5_BQ, h = blockIdx.y, b = blockIdx.z;
  const int bh = b * H + h;
  // causal: query t sees keys <= t, so a query tile stops at the key tile that holds its last row
  const int n_tiles = causal ? min((L + F5_BK - 1) / F5_BK, (min(q0 + F5_BQ, L) + F5_BK - 1) / F5_BK) : (L + F5_BK - 1) / F5_BK;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(k_full + s, 1); mbar_init(k_empty + s, 8); mbar_init(v_full + s, 1); mbar_init(v_empty + s, 8);
    }
    fence_mbar_init();
    prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmV);
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, NPL * C::Q_PLANE);
      for (int pl = 0; pl < NPL; ++pl)
        for (int kb = 0; kb < KBQ; ++kb)
          tma_load_3d(smem + C::OFF_Q + pl * C::Q_PLANE + kb * C::Q_KB, &tmQ, q_full, kb * 64, q0, pl * BH + bh);
      for (int j = 0; j < n_tiles; ++j) {
        const int sl = j & 1;                     // slot sl is free once both consumer warpgroups are done with tile j - 2
        if (j >= 2) mbar_wait(k_empty + sl, ((j >> 1) - 1) & 1);
        mbar_arrive_expect_tx(k_full + sl, C::K_SLOT);
        for (int pl = 0; pl < NPL; ++pl)
          for (int kb = 0; kb < KBQ; ++kb)
            tma_load_3d(smem + C::OFF_K + sl * C::K_SLOT + pl * C::K_PLANE + kb * C::K_KB, &tmK, k_full + sl, kb * 64, j * F5_BK, pl * BH + bh);
        if (j >= 2) mbar_wait(v_empty + sl, ((j >> 1) - 1) & 1);
        mbar_arrive_expect_tx(v_full + sl, C::V_SLOT);
        for (int pl = 0; pl < NPL; ++pl)
          tma_load_3d(smem + C::OFF_V + sl * C::V_SLOT + pl * C::V_PLANE, &tmV, v_full + sl, j * F5_BK, 0, pl * BH + bh);
      }
    }
  } else {
    // ===================== consumers: warpgroup cw owns query rows [cw * 64, +64) of the tile =====================
    // Thread layout of the wgmma accumulators: rows ra = 16 * (warp % 4) + lane / 4 and rb = ra + 8, columns 8j + 2 (lane % 4) + {0, 1};
    // a row's 64 keys are spread over 4 lanes.  P is taken relative to a reference maximum m that only moves when a tile exceeds it
    // by more than 2^8; then that row's O accumulators and running sum are rescaled in registers.
    const int cw = wg - 1, wq = warp & 3, quad = lane & 3;
    const int ra = cw * 64 + wq * 16 + (lane >> 2), tqa = q0 + ra, tqb = tqa + 8;
    const int kmax_a = causal ? min(L, tqa + 1) : L, kmax_b = causal ? min(L, tqb + 1) : L;
    constexpr float LOG2E = 1.4426950408889634f;
    const uint32_t sQ = smem_u32(smem + C::OFF_Q) + cw * 64 * 128;
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;   // m in log2 units (score * log2 e); l: this lane's partial sums
    mbar_wait(q_full, 0);
    for (int j = 0; j < n_tiles; ++j) {
      const int sl = j & 1, k0 = j * F5_BK;
      const uint32_t par = (j >> 1) & 1;
      const uint32_t sK = smem_u32(smem + C::OFF_K + sl * C::K_SLOT), sV = smem_u32(smem + C::OFF_V + sl * C::V_SLOT);
      // S_j = Q K_j^T; split mode issues the three terms of one K step back to back (hi.hi, lo.hi, hi.lo)
      float s[F5_BK / 2];
      mbar_wait(k_full + sl, par);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < KBQ; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t qo = kb * C::Q_KB + k * 32, ko = kb * C::K_KB + k * 32;
          Wgmma<F5_BK>::ss(s, make_wgmma_desc_sw128(sQ + qo), make_wgmma_desc_sw128(sK + ko), (kb | k) != 0 ? 1u : 0u);
          if (SPLIT) {
            Wgmma<F5_BK>::ss(s, make_wgmma_desc_sw128(sQ + C::Q_PLANE + qo), make_wgmma_desc_sw128(sK + ko), 1u);
            Wgmma<F5_BK>::ss(s, make_wgmma_desc_sw128(sQ + qo), make_wgmma_desc_sw128(sK + C::K_PLANE + ko), 1u);
          }
        }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      if (lane == 0) mbar_arrive(k_empty + sl);
      // row maxima over the visible keys
      float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
      for (int c = 0; c < F5_BK / 8; ++c)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = k0 + 8 * c + 2 * quad + e;
          if (key < kmax_a) mx_a = fmaxf(mx_a, s[4 * c + e]);
          if (key < kmax_b) mx_b = fmaxf(mx_b, s[4 * c + 2 + e]);
        }
#pragma unroll
      for (int x = 1; x <= 2; x <<= 1) {
        mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, x));
        mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, x));
      }
      mx_a *= LOG2E; mx_b *= LOG2E;
      if (j == 0) {
        m_a = mx_a; m_b = mx_b;                  // key 0 is visible to every row: finite
      } else {
        const bool need_a = mx_a > m_a + F5_RESCALE_LOG2, need_b = mx_b > m_b + F5_RESCALE_LOG2;
        if (need_a || need_b) {
          const float fa = need_a ? f5_ex2(m_a - mx_a) : 1.f, fb = need_b ? f5_ex2(m_b - mx_b) : 1.f;
          if (need_a) { l_a *= fa; m_a = mx_a; }
          if (need_b) { l_b *= fb; m_b = mx_b; }
#pragma unroll
          for (int c = 0; c < D / 8; ++c) { o[4 * c] *= fa; o[4 * c + 1] *= fa; o[4 * c + 2] *= fb; o[4 * c + 3] *= fb; }
        }
      }
      // P = exp2(S * log2e - m) as fp16 hi (+ lo), packed as the register A operand of P.V (m16n8k16 A-fragment layout)
      const bool full = k0 + F5_BK <= min(kmax_a, kmax_b);      // no masked key in this tile for either row
      uint32_t ph[F5_BK / 16][4], plo[SPLIT ? F5_BK / 16 : 1][4];
#pragma unroll
      for (int c = 0; c < F5_BK / 8; ++c)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int key = k0 + 8 * c + 2 * quad;
          const float mr = rr ? m_b : m_a;
          const int km = rr ? kmax_b : kmax_a;
          float p0 = f5_ex2(fmaf(s[4 * c + 2 * rr], LOG2E, -mr)), p1 = f5_ex2(fmaf(s[4 * c + 2 * rr + 1], LOG2E, -mr));
          if (!full) {
            p0 = key < km ? p0 : 0.f;
            p1 = key + 1 < km ? p1 : 0.f;
          }
          if (rr) l_b += p0 + p1; else l_a += p0 + p1;
          const __half2 hh = __floats2half2_rn(p0, p1);
          ph[c >> 1][(c & 1) * 2 + rr] = *reinterpret_cast<const uint32_t*>(&hh);
          if (SPLIT) {
            const float2 back = __half22float2(hh);
            const __half2 ll = __floats2half2_rn(p0 - back.x, p1 - back.y);
            plo[c >> 1][(c & 1) * 2 + rr] = *reinterpret_cast<const uint32_t*>(&ll);
          }
        }
      // O += P_j V_j (V^T tile: D rows x 64 keys, K-major)
      mbar_wait(v_full + sl, par);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < F5_BK / 16; ++k) {
        Wgmma<D>::rs(o, ph[k], make_wgmma_desc_sw128(sV + k * 32));
        if (SPLIT) {
          Wgmma<D>::rs(o, plo[k], make_wgmma_desc_sw128(sV + k * 32));
          Wgmma<D>::rs(o, ph[k], make_wgmma_desc_sw128(sV + C::V_PLANE + k * 32));
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (lane == 0) mbar_arrive(v_empty + sl);
    }
#pragma unroll
    for (int x = 1; x <= 2; x <<= 1) {
      l_a += __shfl_xor_sync(0xffffffffu, l_a, x);
      l_b += __shfl_xor_sync(0xffffffffu, l_b, x);
    }
    const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int tq = rr ? tqb : tqa;
      if (tq >= L) continue;
      const float inv = rr ? inv_b : inv_a;
      const long long ob = ((long long)b * L + tq) * (long long)(H * D) + h * D + 2 * quad;
#pragma unroll
      for (int c = 0; c < D / 8; ++c) {
        const float a = o[4 * c + 2 * rr] * inv, e = o[4 * c + 2 * rr + 1] * inv;
        const __half2 hh = __floats2half2_rn(a, e);
        *reinterpret_cast<__half2*>(out_hi + ob + 8 * c) = hh;
        if (out_lo) {
          const float2 back = __half22float2(hh);
          *reinterpret_cast<__half2*>(out_lo + ob + 8 * c) = __floats2half2_rn(a - back.x, e - back.y);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- host
typedef CUresult (*F5EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static F5EncodeFn f5_encode() {
  static F5EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (F5EncodeFn)p;
  }
  return fn;
}
// 3-D fp16 map {inner, rows, z}, 128-byte swizzle, out-of-range rows / columns read as zero
static int f5_map(CUtensorMap* m, const void* base, uint64_t inner, uint64_t rows, uint64_t z, uint64_t row_stride_elems, uint32_t box_inner,
                  uint32_t box_rows) {
  F5EncodeFn enc = f5_encode();
  QB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  const cuuint64_t dims[3] = {inner, rows, z};
  const cuuint64_t strides[2] = {row_stride_elems * 2, row_stride_elems * rows * 2};
  const cuuint32_t box[3] = {box_inner, box_rows, 1}, es[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  QB_REQUIRE(r == CUDA_SUCCESS, "attention_umma: cuTensorMapEncodeTiled failed: %d (dims %llu %llu %llu)", (int)r, (unsigned long long)inner,
             (unsigned long long)rows, (unsigned long long)z);
  return 0;
}

template <int D, bool SPLIT>
static int f5_launch(const float* qkv, int64_t B, int64_t L, int32_t H, const float* rc, const float* rs, __half* out_hi, __half* out_lo,
                     int causal, void* workspace, cudaStream_t st) {
  using C = F5Cfg<D, SPLIT>;
  constexpr int NPL = C::NPL;
  const int64_t BH = B * H, Lp = (L + 7) / 8 * 8;
  __half* q16 = (__half*)workspace;
  __half* k16 = q16 + NPL * BH * L * D;
  __half* vT = k16 + NPL * BH * L * D;
  fa5_prep_kernel<D><<<dim3((unsigned)ceil_div(L, 32), (unsigned)H, (unsigned)B), 256, 0, st>>>(qkv, (int)L, (int)Lp, H, rc, rs,
                                                                                                1.0f / sqrtf((float)D), q16, k16, vT, NPL);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  CUtensorMap tmQ, tmK, tmV;
  if (int e = f5_map(&tmQ, q16, D, L, NPL * BH, D, 64, F5_BQ)) return e;
  if (int e = f5_map(&tmK, k16, D, L, NPL * BH, D, 64, F5_BK)) return e;
  if (int e = f5_map(&tmV, vT, L, D, NPL * BH, Lp, F5_BK, D)) return e;
  QB_CHECK_CUDA(cudaFuncSetAttribute(fa5_kernel<D, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
  fa5_kernel<D, SPLIT><<<dim3((unsigned)ceil_div(L, F5_BQ), (unsigned)H, (unsigned)B), F5_THREADS, C::SMEM, st>>>(tmQ, tmK, tmV, (int)L, H,
                                                                                                                (int)BH, causal, out_hi, out_lo);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace qb
using namespace qb;

extern "C" int64_t qb_attention_umma_workspace_bytes(int64_t B, int64_t L, int32_t heads, int32_t head_dim, int32_t split) {
  const int64_t planes = split ? 2 : 1, Lp = (L + 7) / 8 * 8;
  return planes * B * heads * head_dim * (2 * L + Lp) * 2 + 1024;
}

extern "C" int qb_attention_umma(const float* qkv, int64_t B, int64_t L, int32_t heads, int32_t head_dim, const float* rope_cos,
                                 const float* rope_sin, qb_half* out_hi, qb_half* out_lo, int32_t split, int32_t causal, void* workspace, void* stream) {
  QB_REQUIRE(qkv && rope_cos && rope_sin && out_hi && workspace && B > 0 && L > 0 && heads > 0, "attention_umma: bad args");
  QB_REQUIRE(head_dim == 64 || head_dim == 128, "attention_umma: head_dim must be 64 or 128 (got %d)", head_dim);
  QB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 127) == 0, "attention_umma: workspace must be 128-byte aligned");
  QB_REQUIRE(B <= 65535 && heads <= 65535, "attention_umma: grid limits (B, heads <= 65535)");
  cudaStream_t st = (cudaStream_t)stream;
  __half *oh = (__half*)out_hi, *ol = (__half*)out_lo;
  if (head_dim == 64)
    return split ? f5_launch<64, true>(qkv, B, L, heads, rope_cos, rope_sin, oh, ol, causal ? 1 : 0, workspace, st)
                 : f5_launch<64, false>(qkv, B, L, heads, rope_cos, rope_sin, oh, ol, causal ? 1 : 0, workspace, st);
  return split ? f5_launch<128, true>(qkv, B, L, heads, rope_cos, rope_sin, oh, ol, causal ? 1 : 0, workspace, st)
               : f5_launch<128, false>(qkv, B, L, heads, rope_cos, rope_sin, oh, ol, causal ? 1 : 0, workspace, st);
}
