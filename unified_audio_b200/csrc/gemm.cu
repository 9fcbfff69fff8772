// Dense contraction kernels: wgmma/TMA persistent GEMM (product path) and a SIMT
// cross-check.  Both evaluate the same qb_gemm_desc (include/quark_b200.h).
//
// Tile: 128 (rows) x BN (cols, 256 or 128) x 64 (K) per pipeline stage, fp16 planes K-major in shared
// memory with the 128-byte TMA/wgmma swizzle; accumulators live in registers.  Warp roles (384 threads):
//   warpgroup 0     TMA producer (one thread), shrunk to 40 registers by setmaxnreg
//   warpgroups 1-2  wgmma m64nBNk16 on rows [0, 64) / [64, 128) of the tile, then the epilogue
//                   (bias/act/gamma/residual) from the accumulator registers; the producer already fills the
//                   stages of the next tile meanwhile.  232 registers each.
// The two fast epilogue kinds never wait on global memory: the tile's bias / gamma are fetched while its main loop
// runs and read from shared memory, the residual arrives by TMA into two 8 KB subtile buffers per warpgroup, and each
// 64 x 128-byte output subtile leaves by TMA store, which drains while the next tile's main loop runs.  Shared memory:
// 192 KB of stages + 32 KB of subtile buffers + the tile's bias / gamma.  On an H100 80GB HBM3 at 700 W this took the
// ConvNeXt pwconv1 / pwconv2 GEMMs from 417 / 442 to 537 / 546 TFLOP/s (scripts/gemm_table.py).
// Convolutions are expressed as `taps` shifted K-panels over a zero-padded channel-last buffer:
// the A tensor map views the buffer as [batch][rows/stride][stride*C], so tap t of output row m is
// the box at (x = (t % stride)*C + c, y = m + t / stride) - TMA-staged im2col without an im2col
// buffer.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>

#include "common.cuh"
#include "quark_b200.h"
#include "wgmma.cuh"

namespace qb {

// ------------------------------------------------------------------ error + launch accounting
static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

constexpr int QB_MAX_DEVICES = 64;
static int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev >= 0 && dev < QB_MAX_DEVICES ? dev : 0;
}

// 1: epilogue / producer warps park on their barriers (try_wait with a suspend hint) instead of spinning
#ifndef QB_PARK
#define QB_PARK 1
#endif

// What the epilogue of a launch does, decided on the host so that the consumer branches once per tile:
//   EPI_HI      (bias) (GELU | ELU | SwiGLU) -> fp16 hi plane (+ lo plane)   (ConvNeXt pwconv1, transformer w13, semantic k3 convs)
//   EPI_F32     (bias) (* gamma) (+ residual) -> fp32, and optionally (ELU) -> hi (+ lo) planes through their own row map
//               (pwconv2, o-proj, w2, residual convs, the semantic encoder's fp32 + planes convs)
//   EPI_GENERIC every other combination (Snake, tanh, ReLU, gamma or residual into planes, unaligned buffers), element by element
//               through epilogue_pair
// The two fast kinds stage each output subtile in shared memory and write it by TMA store, EPI_F32 reads its residual by TMA
// load; they need 16-byte aligned bases and row pitches (classify_epilogue).
enum EpiKind : int { EPI_GENERIC = 0, EPI_HI = 1, EPI_F32 = 2 };

struct RowMapD {
  void* ptr;
  long long ld, rpb, off;
};
struct GemmParams {
  int tiles_per_batch, num_n_tiles, num_tiles, num_kb;
  int taps, stride, cblocks, C, dil;   // C = channels contracted per tap
  int Cld;                             // channels per row of the A buffer (row stride); == C unless a_cols is given
  int m_per_batch, N;
  const float* bias;
  const float* gamma;
  const float* act_p;    // per-column parameter of `act` (Snake alpha)
  const float* act2_p;   // per-column parameter of `act2`
  RowMapD res, o32, ohi, olo;
  int act, act2;
  int epi;               // EpiKind, classified once per launch by fill_params
  // SIMT path only
  const __half *a_hi, *a_lo, *w_hi, *w_lo;
  long long a_rpb;
  int a_batch;
};

// Snake (bicodec/modules/blocks/layers.py:33-38): x + (alpha + 1e-9)^-1 * sin(alpha x)^2
// Epilogue form: sin.approx after an explicit 2*pi range reduction (|error| < 3e-7 for |alpha x| < 64, exact sinf beyond) and
// rcp.approx (1 ulp) - the accurate sinf + IEEE division cost 35 instructions per element and made the N < 256 conv GEMMs
// epilogue-bound.
__device__ __forceinline__ float snake_f(float v, float a) {
  const float t = a * v;
  float sn;
  if (fabsf(t) < 64.f) {
    const float k = rintf(t * 0.15915494309189535f);
    const float r = fmaf(k, -6.2831854820251465f, t);            // t - k * fl(2 pi)
    sn = __sinf(fmaf(k, 1.7484555e-7f, r));                      // + k * (fl(2 pi) - 2 pi)
  } else {
    sn = sinf(t);
  }
  float rc;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(a + 1e-9f));
  return fmaf(rc, sn * sn, v);
}
__device__ __forceinline__ float apply_act(int act, float v) {
  if (act == QB_ACT_GELU) return gelu_fast(v);
  if (act == QB_ACT_ELU) return elu_f(v);
  if (act == QB_ACT_TANH) return tanhf(v);
  if (act == QB_ACT_RELU) return v < 0.f ? 0.f : v;      // NaN passes, as torch.relu
  return v;
}

// Final part of the epilogue for one output element (after bias/act): gamma, residual, stores.
__device__ __forceinline__ void epi_finish_scalar(const GemmParams& p, int b, int m, int n, float v) {
  if (p.gamma) v *= __ldg(p.gamma + n);
  if (p.res.ptr) v += ((const float*)p.res.ptr)[((long long)b * p.res.rpb + p.res.off + m) * p.res.ld + n];
  if (p.o32.ptr) ((float*)p.o32.ptr)[((long long)b * p.o32.rpb + p.o32.off + m) * p.o32.ld + n] = v;
  if (p.ohi.ptr) {
    float u = p.act2 == QB_ACT_ELU ? elu_f(v) : (p.act2 == QB_ACT_SNAKE ? snake_f(v, __ldg(p.act2_p + n)) : v);
    __half h, l;
    split_f16(u, h, l);
    long long o = ((long long)b * p.ohi.rpb + p.ohi.off + m) * p.ohi.ld + n;
    ((__half*)p.ohi.ptr)[o] = h;
    if (p.olo.ptr) ((__half*)p.olo.ptr)[o] = l;
  }
}

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return (uint8_t*)(((uintptr_t)p + 1023) & ~(uintptr_t)1023);
}

// Epilogue for the accumulator pair (row m, columns n, n + 1) a thread holds after the warpgroup MMA.
__device__ __forceinline__ void epilogue_pair(const GemmParams& p, int b, int m, int n, float v0, float v1) {
  if (m >= p.m_per_batch || n >= p.N) return;
  const bool has1 = n + 1 < p.N;
  if (p.bias) {
    v0 += __ldg(p.bias + n);
    if (has1) v1 += __ldg(p.bias + n + 1);
  }
  if (p.act == QB_ACT_SWIGLU) {                // interleaved gate / up columns -> one output column n / 2 (n is even, N even)
    epi_finish_scalar(p, b, m, n >> 1, silu_f(v0) * v1);
    return;
  }
  // vectorised paths for the two epilogues that carry most of the single-pass GEMM work: ConvNeXt pwconv1 (bias + GELU -> fp16
  // hi plane) and pwconv2 (bias, gamma, + residual -> fp32); n is even, so a pair is one aligned half2 / float2 when the row
  // pitches are even and the bases 8-byte aligned
  if (has1 && p.act2 == QB_ACT_NONE && (p.act == QB_ACT_NONE || p.act == QB_ACT_GELU)) {
    if (p.ohi.ptr && !p.olo.ptr && !p.o32.ptr && !p.res.ptr && !p.gamma && (p.ohi.ld & 1) == 0 &&
        (reinterpret_cast<uintptr_t>(p.ohi.ptr) & 3) == 0) {
      if (p.act == QB_ACT_GELU) { v0 = gelu_fast(v0); v1 = gelu_fast(v1); }
      const __half2 hmax = __float2half2_rn(65504.f), hmin = __float2half2_rn(-65504.f);
      *reinterpret_cast<__half2*>((__half*)p.ohi.ptr + ((long long)b * p.ohi.rpb + p.ohi.off + m) * p.ohi.ld + n) =
          __hmax2_nan(__hmin2_nan(__floats2half2_rn(v0, v1), hmax), hmin);     // saturated, NaN kept (as f2h_sat)
      return;
    }
    if (p.o32.ptr && !p.ohi.ptr && p.act == QB_ACT_NONE && (p.o32.ld & 1) == 0 && (reinterpret_cast<uintptr_t>(p.o32.ptr) & 7) == 0 &&
        (!p.res.ptr || ((p.res.ld & 1) == 0 && (reinterpret_cast<uintptr_t>(p.res.ptr) & 7) == 0)) &&
        (!p.gamma || (reinterpret_cast<uintptr_t>(p.gamma) & 7) == 0)) {
      if (p.gamma) {
        const float2 g = __ldg(reinterpret_cast<const float2*>(p.gamma + n));
        v0 *= g.x; v1 *= g.y;
      }
      if (p.res.ptr) {
        const float2 r = *reinterpret_cast<const float2*>((const float*)p.res.ptr + ((long long)b * p.res.rpb + p.res.off + m) * p.res.ld + n);
        v0 += r.x; v1 += r.y;
      }
      *reinterpret_cast<float2*>((float*)p.o32.ptr + ((long long)b * p.o32.rpb + p.o32.off + m) * p.o32.ld + n) = make_float2(v0, v1);
      return;
    }
  }
  if (p.act == QB_ACT_SNAKE) {
    v0 = snake_f(v0, __ldg(p.act_p + n));
    if (has1) v1 = snake_f(v1, __ldg(p.act_p + n + 1));
  } else if (p.act != QB_ACT_NONE) {
    v0 = apply_act(p.act, v0);
    v1 = apply_act(p.act, v1);
  }
  epi_finish_scalar(p, b, m, n, v0);
  if (has1) epi_finish_scalar(p, b, m, n + 1, v1);
}

constexpr int GEMM_BM = 128, GEMM_BK = 64;
constexpr int GEMM_THREADS = 3 * 128;           // warpgroup 0: TMA producer; warpgroups 1-2: MMA + epilogue, 64 rows each
// register split after setmaxnreg: 128 * 40 + 256 * 232 = 64512 of the SM's 65536 (the launch reserves 384 * 168)
constexpr int GEMM_PRODUCER_REGS = 40, GEMM_CONSUMER_REGS = 232;

// Epilogue buffers of the fast kinds: per consumer warpgroup, EPI_BUFS subtiles of 64 rows x 128 bytes (32 fp32 or 64 fp16
// columns) in the TMA 128-byte swizzle: row r at r * 128, its 16-byte chunk c at chunk position c ^ (r % 8).  The quad of
// lanes holding one row of an 8-column group then writes 8 distinct chunk positions per 8 rows: no bank conflicts.
constexpr int EPI_BUFS = 2;
constexpr uint32_t EPI_SUB_BYTES = 64 * 128;

// Per-column operands of a tile in shared memory, [bias | gamma] x BN floats: the 256 consumer threads fetch them at the start
// of the tile, so that the latency hides behind its main loop, and store them once the main loop is done.
template <int BN>
__device__ __forceinline__ void load_tile_cols(const GemmParams& p, int n0, int ct, float (&v)[2 * BN / 256]) {
#pragma unroll
  for (int i = 0; i < 2 * BN / 256; ++i) {
    const int k = ct + 256 * i, n = n0 + k % BN;
    const float* src = k < BN ? p.bias : p.gamma;
    v[i] = src && n < p.N ? __ldg(src + n) : 0.f;
  }
}

// Fast epilogue kinds, on the 64 x BN half tile of one consumer warpgroup (rows row0 + [0, 64), columns n0 + [0, BN)):
// accumulators -> swizzled subtile in shared memory -> one TMA store per subtile, issued by the warpgroup's first thread.
// The stores drain while the next tile's main loop runs; the TMA map clips rows >= m_per_batch and columns >= N.
// Same arithmetic, in the same order, as epilogue_pair / epi_finish_scalar.
struct EpiCtx {
  uint8_t* buf;        // this warpgroup's EPI_BUFS subtile buffers
  uint64_t* rfull;     // one mbarrier per buffer: residual subtile landed
  uint32_t cols;       // shared address of the tile's [bias | gamma]
  int cw, b, row0, n0;
};

// 64-column fp16 subtiles, 128-byte rows.  Without a lo plane the subtiles alternate between the two buffers; with one, each
// subtile puts hi in the first buffer and lo in the second.  SwiGLU reduces each interleaved (gate, up) accumulator pair to one
// output column, 4 j + lane % 4 for the pair at columns 8 j + 2 (lane % 4): a 64 x BN half tile gives BN / 2 output columns.
// A hi plane alone with no activation or GELU is rounded as epilogue_pair's half2 branch rounds it; every other case through
// split_f16, as epi_finish_scalar.
template <int BN, bool SWIGLU>
__device__ __forceinline__ void epilogue_hi(const GemmParams& p, const CUtensorMap* tmHi, const CUtensorMap* tmLo, const EpiCtx& e,
                                                const float (&acc)[BN / 2]) {
  constexpr int NSUB = SWIGLU ? BN / 128 : BN / 64, JS = SWIGLU ? 16 : 8;      // subtiles; 8-column accumulator groups per subtile
  const __half2 hmax = __float2half2_rn(65504.f), hmin = __float2half2_rn(-65504.f);
  const int act = p.act;
  const bool lo = BN == 128 && p.olo.ptr != nullptr, leader = (threadIdx.x & 127) == 0;
  const bool rn_sat = BN == 256 || (!lo && (act == QB_ACT_NONE || act == QB_ACT_GELU));
  const int lane = threadIdx.x & 31;
  // rows r and r + 8 (r % 8 = lane / 4) at byte (SWIGLU ? 2 : 4) (lane % 4) of a 16-byte chunk c, stored at chunk c ^ (lane / 4)
  const uint32_t th = smem_u32(e.buf) + (((threadIdx.x >> 5) & 3) * 16 + (lane >> 2)) * 128 + (SWIGLU ? 2 : 4) * (lane & 3),
                 sw = (lane >> 2) << 4;
#pragma unroll
  for (int s = 0; s < NSUB; ++s) {
    const uint32_t bh = (lo ? 0 : s % EPI_BUFS) * EPI_SUB_BYTES, bl = EPI_SUB_BYTES;
    if (s == 0 || lo) {                        // the previous stores have read the buffers
      if (leader) bulk_wait_read<0>();
      named_bar_sync(2 + e.cw, 128);
    } else if (s >= EPI_BUFS) {                // the store of subtile s - EPI_BUFS has read this buffer
      if (leader) bulk_wait_read<EPI_BUFS - 1>();
      named_bar_sync(2 + e.cw, 128);
    }
#pragma unroll
    for (int jj = 0; jj < JS; ++jj) {
      const int j = JS * s + jj;
      const float2 bb = p.bias ? ld_shared_f32x2(e.cols + 4 * (8 * j + 2 * (lane & 3))) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (p.bias) { v0 += bb.x; v1 += bb.y; }
        if (SWIGLU) {                          // output column 4 jj + lane % 4: chunk jj / 2, byte 8 (jj % 2) + 2 (lane % 4)
          const uint32_t el = th + h * 1024 + ((16 * (jj >> 1)) ^ sw) + 8 * (jj & 1);
          __half hv, lv;
          split_f16(silu_f(v0) * v1, hv, lv);
          st_shared_b16(el + bh, hv);
          if (lo) st_shared_b16(el + bl, lv);
        } else {
          const uint32_t el = th + h * 1024 + ((16 * jj) ^ sw);
          if (act == QB_ACT_GELU) { v0 = gelu_fast(v0); v1 = gelu_fast(v1); }
          else if (BN == 128 && act == QB_ACT_ELU) { v0 = elu_f(v0); v1 = elu_f(v1); }
          if (rn_sat) {
            const __half2 o = __hmax2_nan(__hmin2_nan(__floats2half2_rn(v0, v1), hmax), hmin);
            st_shared_b32(el + bh, *reinterpret_cast<const uint32_t*>(&o));
          } else {
            __half2 hv, lv;
            split_f16(v0, hv.x, lv.x);
            split_f16(v1, hv.y, lv.y);
            st_shared_b32(el + bh, *reinterpret_cast<const uint32_t*>(&hv));
            if (lo) st_shared_b32(el + bl, *reinterpret_cast<const uint32_t*>(&lv));
          }
        }
      }
    }
    fence_proxy_async();
    named_bar_sync(2 + e.cw, 128);
    if (leader) {
      const int x = (SWIGLU ? e.n0 / 2 : e.n0) + 64 * s;
      tma_store_3d(tmHi, e.buf + bh, x, e.row0, e.b);
      if (lo) tma_store_3d(tmLo, e.buf + bl, x, e.row0, e.b);
      bulk_commit();
    }
  }
}

// 32-column fp32 subtiles.  The residual arrives by TMA into the subtile buffer the result is then written to.  Every element is
// read and then written by the same thread, so the residual may be the output buffer itself.
// Without planes the subtiles alternate between the two buffers: subtiles 0 .. EPI_BUFS - 1 of the residual were requested
// during the main loop, subtile s + EPI_BUFS as soon as the store of subtile s has read its buffer.
// With planes, (act2) -> split_f16 of the fp32 result: the first buffer holds each subtile's residual and result, the second its
// hi and lo planes as two 64-row x 64-byte boxes in the 64-byte swizzle (row r at r * 64, chunk c at c ^ (r / 2 % 4)); the
// residual of subtile s + 1 is requested once the stores of subtile s have read both.
template <int BN>
__device__ __forceinline__ void epilogue_f32(const GemmParams& p, const CUtensorMap* tmO, const CUtensorMap* tmR, const CUtensorMap* tmHi,
                                             const CUtensorMap* tmLo, const EpiCtx& e, const float (&acc)[BN / 2]) {
  constexpr int NSUB = BN / 32;
  constexpr uint32_t LO_OFF = EPI_SUB_BYTES / 2;
  static_assert(NSUB % (2 * EPI_BUFS) == 0, "each residual barrier completes an even number of phases per tile");
  const bool res = p.res.ptr != nullptr, planes = BN == 128 && p.ohi.ptr != nullptr, lo = p.olo.ptr != nullptr;
  const bool elu = p.act2 == QB_ACT_ELU;
  const bool leader = (threadIdx.x & 127) == 0;
  const int lane = threadIdx.x & 31, row = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  // rows r and r + 8 (r % 8 = lane / 4) at byte 8 (lane % 2) of chunk 2 jj + (lane % 4) / 2, stored at that chunk ^ (lane / 4);
  // 2 jj has no bit in common with (lane % 4) / 2, so the stored chunk is 2 jj ^ ((lane % 4) / 2 ^ lane / 4)
  const uint32_t th = smem_u32(e.buf) + row * 128 + 8 * (lane & 1), sw = (((lane >> 1) & 1) ^ (lane >> 2)) << 4;
  // planes: rows r and r + 8 at byte 4 (lane % 4) of chunk jj, stored at chunk jj ^ (r / 2 % 4) = jj ^ (lane / 8)
  const uint32_t tp = smem_u32(e.buf + EPI_SUB_BYTES) + row * 64 + 4 * (lane & 3), swp = ((lane >> 3) & 3) << 4;
#pragma unroll
  for (int s = 0; s < NSUB; ++s) {
    const int u = planes ? 0 : s % EPI_BUFS;
    uint8_t* buf = e.buf + u * EPI_SUB_BYTES;
    if (res) {
      mbar_wait(&e.rfull[u], (planes ? s : s / EPI_BUFS) & 1);
    } else if (s == 0 || planes) {             // the previous stores have read the buffers
      if (leader) bulk_wait_read<0>();
      named_bar_sync(2 + e.cw, 128);
    } else if (s >= EPI_BUFS) {                // the store of subtile s - EPI_BUFS has read this buffer
      if (leader) bulk_wait_read<EPI_BUFS - 1>();
      named_bar_sync(2 + e.cw, 128);
    }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * s + jj;
      const uint32_t col = e.cols + 4 * (8 * j + 2 * (lane & 3));
      const float2 bb = p.bias ? ld_shared_f32x2(col) : make_float2(0.f, 0.f);
      const float2 g = p.gamma ? ld_shared_f32x2(col + 4 * BN) : make_float2(1.f, 1.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t el = th + u * EPI_SUB_BYTES + h * 1024 + ((32 * jj) ^ sw);
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (p.bias) { v0 += bb.x; v1 += bb.y; }
        if (p.gamma) { v0 *= g.x; v1 *= g.y; }
        if (res) {
          const float2 rv = ld_shared_f32x2(el);
          v0 += rv.x; v1 += rv.y;
        }
        st_shared_f32x2(el, v0, v1);
        if (planes) {
          if (elu) { v0 = elu_f(v0); v1 = elu_f(v1); }
          const uint32_t ep = tp + h * 512 + ((16 * jj) ^ swp);
          __half2 hv, lv;
          split_f16(v0, hv.x, lv.x);
          split_f16(v1, hv.y, lv.y);
          st_shared_b32(ep, *reinterpret_cast<const uint32_t*>(&hv));
          if (lo) st_shared_b32(ep + LO_OFF, *reinterpret_cast<const uint32_t*>(&lv));
        }
      }
    }
    fence_proxy_async();
    named_bar_sync(2 + e.cw, 128);
    if (leader) {
      tma_store_3d(tmO, buf, e.n0 + 32 * s, e.row0, e.b);
      if (planes) {
        tma_store_3d(tmHi, e.buf + EPI_SUB_BYTES, e.n0 + 32 * s, e.row0, e.b);
        if (lo) tma_store_3d(tmLo, e.buf + EPI_SUB_BYTES + LO_OFF, e.n0 + 32 * s, e.row0, e.b);
      }
      bulk_commit();
      const int next = s + (planes ? 1 : EPI_BUFS);
      if (res && next < NSUB) {
        bulk_wait_read<0>();
        mbar_arrive_expect_tx(&e.rfull[u], EPI_SUB_BYTES);
        tma_load_3d(buf, tmR, &e.rfull[u], e.n0 + 32 * next, e.row0, e.b);
      }
    }
  }
}

// One kernel for every qb_gemm: BM x BN x 64 tiles, BN = 256 (wgmma m64n256k16, 128 accumulators per thread) or 128.
template <int NTERMS, int BN, int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo,
               const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmRes,
               const __grid_constant__ CUtensorMap tmHi, const __grid_constant__ CUtensorMap tmLo, const GemmParams p) {
  constexpr int BM = GEMM_BM, BK = GEMM_BK;
  constexpr int NPL = (NTERMS == 1) ? 1 : 2;
  constexpr uint32_t A_BYTES = BM * BK * 2, W_BYTES = BN * BK * 2;
  constexpr uint32_t STAGE_BYTES = NPL * (A_BYTES + W_BYTES);
  constexpr int CONSUMER_WARPS = 8;

  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* epi_smem = smem + STAGES * STAGE_BYTES;
  float* tile_cols = (float*)(epi_smem + 2 * EPI_BUFS * EPI_SUB_BYTES);      // [bias | gamma] x BN
  uint64_t* full = (uint64_t*)(tile_cols + 2 * BN);
  uint64_t* empty = full + STAGES;
  uint64_t* rfull = empty + STAGES;        // [2][EPI_BUFS]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const bool tma_epi = p.epi != EPI_GENERIC;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMER_WARPS); }
    for (int s = 0; s < 2 * EPI_BUFS; ++s) mbar_init(&rfull[s], 1);
    fence_mbar_init();
  }
  if (threadIdx.x == 32) {
    prefetch_tmap(&tmA_hi); prefetch_tmap(&tmW_hi);
    if (NPL == 2) { prefetch_tmap(&tmA_lo); prefetch_tmap(&tmW_lo); }
    if (p.epi == EPI_F32) { prefetch_tmap(&tmOut); if (p.res.ptr) prefetch_tmap(&tmRes); }
    if (tma_epi && p.ohi.ptr) { prefetch_tmap(&tmHi); if (p.olo.ptr) prefetch_tmap(&tmLo); }
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<GEMM_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int n_tile = tile % p.num_n_tiles, m_tile = tile / p.num_n_tiles;
        const int b = m_tile / p.tiles_per_batch, m0 = (m_tile % p.tiles_per_batch) * BM, n0 = n_tile * BN;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          const int tap = kb / p.cblocks, cb = kb - tap * p.cblocks;
          if (QB_PARK) mbar_wait_parked(&empty[stage], phase ^ 1); else mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);
          uint8_t* s = smem + stage * STAGE_BYTES;
          const int tt = tap * p.dil;      // input row of output row m: m * stride + tap * dilation
          const int ax = (tt % p.stride) * p.Cld + cb * BK, ay = m0 + tt / p.stride, wx = tap * p.C + cb * BK;
          tma_load_3d(s, &tmA_hi, &full[stage], ax, ay, b);
          if (NPL == 2) tma_load_3d(s + A_BYTES, &tmA_lo, &full[stage], ax, ay, b);
          tma_load_2d(s + NPL * A_BYTES, &tmW_hi, &full[stage], wx, n0);
          if (NPL == 2) tma_load_2d(s + NPL * A_BYTES + W_BYTES, &tmW_lo, &full[stage], wx, n0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<GEMM_CONSUMER_REGS>();
    const int cw = wg - 1, wq = warp & 3;      // consumer warpgroup: rows [cw * 64, +64) of the tile
    const bool leader = (threadIdx.x & 127) == 0, epi_res = p.epi == EPI_F32 && p.res.ptr;
    const int res_bufs = BN == 128 && p.ohi.ptr ? 1 : EPI_BUFS;      // EPI_F32 with planes keeps the second buffer for them
    const bool epi_cols = tma_epi && (p.bias || p.gamma);
    uint32_t stage = 0, phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int n_tile = tile % p.num_n_tiles, m_tile = tile / p.num_n_tiles;
      const int b = m_tile / p.tiles_per_batch, m0 = (m_tile % p.tiles_per_batch) * BM, n0 = n_tile * BN;
      float cols[2 * BN / 256];
      if (epi_cols) load_tile_cols<BN>(p, n0, threadIdx.x - 128, cols);
      uint32_t prev_stage = 0;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + cw * (A_BYTES / 2);
        const uint32_t sw = smem_u32(smem + stage * STAGE_BYTES) + NPL * A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t a_hi = make_wgmma_desc_sw128(sa + k * 32), w_hi = make_wgmma_desc_sw128(sw + k * 32);
          Wgmma<BN>::ss(acc, a_hi, w_hi, (kb | k) != 0 ? 1u : 0u);
          if (NTERMS == 3) {
            Wgmma<BN>::ss(acc, make_wgmma_desc_sw128(sa + A_BYTES + k * 32), w_hi, 1u);
            Wgmma<BN>::ss(acc, a_hi, make_wgmma_desc_sw128(sw + W_BYTES + k * 32), 1u);
          }
        }
        wgmma_commit();
        if (kb == 0 && epi_res && leader) {
          // while the first MMAs run: the previous tile's stores have left the epilogue buffers, which may now take the
          // first residual subtiles of this one
          bulk_wait_read<0>();
          for (int u = 0; u < res_bufs; ++u) {
            uint64_t* bar = rfull + cw * EPI_BUFS + u;
            mbar_arrive_expect_tx(bar, EPI_SUB_BYTES);
            tma_load_3d(epi_smem + (cw * EPI_BUFS + u) * EPI_SUB_BYTES, &tmRes, bar, n0 + 32 * u, m0 + cw * 64, b);
          }
        }
        wgmma_wait<1>();                          // the MMAs of K-block kb - 1 are done: release their stage
        if (kb > 0 && lane == 0) mbar_arrive(&empty[prev_stage]);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty[prev_stage]);
      if (epi_cols) {
        named_bar_sync(1, 256);                // both warpgroups are done with the previous tile's columns
#pragma unroll
        for (int i = 0; i < 2 * BN / 256; ++i) tile_cols[threadIdx.x - 128 + 256 * i] = cols[i];
        named_bar_sync(1, 256);
      }
      const EpiCtx ec{epi_smem + cw * EPI_BUFS * EPI_SUB_BYTES, rfull + cw * EPI_BUFS, smem_u32(tile_cols), cw, b, m0 + cw * 64, n0};
      if (p.epi == EPI_HI) {
        if constexpr (BN == 128) {
          if (p.act == QB_ACT_SWIGLU) epilogue_hi<BN, true>(p, &tmHi, &tmLo, ec, acc);
          else epilogue_hi<BN, false>(p, &tmHi, &tmLo, ec, acc);
        } else {
          epilogue_hi<BN, false>(p, &tmHi, &tmLo, ec, acc);
        }
      } else if (p.epi == EPI_F32) {
        epilogue_f32<BN>(p, &tmOut, &tmRes, &tmHi, &tmLo, ec, acc);
      } else {
        const int r = m0 + cw * 64 + wq * 16 + (lane >> 2), c = n0 + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          epilogue_pair(p, b, r, c + 8 * j, acc[4 * j], acc[4 * j + 1]);
          epilogue_pair(p, b, r + 8, c + 8 * j, acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
    }
    if (tma_epi && leader) bulk_wait<0>();      // the shared-memory sources of the last stores stay valid until read
  }
}

// ------------------------------------------------------------------ SIMT cross-check
__global__ void gemm_simt_kernel(const GemmParams p) {
  const int N_out = p.act == QB_ACT_SWIGLU ? p.N / 2 : p.N;
  long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)p.a_batch * p.m_per_batch * N_out;
  if (gid >= total) return;
  const int n = (int)(gid % N_out);
  const long long bm = gid / N_out;
  const int m = (int)(bm % p.m_per_batch), b = (int)(bm / p.m_per_batch);
  const long long K = (long long)p.taps * p.C;
  auto dot = [&](int col) {
    float acc = 0.f;
    for (int t = 0; t < p.taps; ++t) {
      long long row = (long long)m * p.stride + (long long)t * p.dil;
      if (row >= p.a_rpb) continue;
      const __half* ah = p.a_hi + ((long long)b * p.a_rpb + row) * p.Cld;
      const __half* al = p.a_lo ? p.a_lo + ((long long)b * p.a_rpb + row) * p.Cld : nullptr;
      const __half* wh = p.w_hi + (long long)col * K + (long long)t * p.C;
      const __half* wl = p.w_lo ? p.w_lo + (long long)col * K + (long long)t * p.C : nullptr;
      for (int c = 0; c < p.C; ++c) {
        float a = __half2float(ah[c]), w = __half2float(wh[c]);
        acc = fmaf(a, w, acc);
        if (al && wl) {
          acc = fmaf(__half2float(al[c]), w, acc);
          acc = fmaf(a, __half2float(wl[c]), acc);
        }
      }
    }
    return acc;
  };
  float v;
  if (p.act == QB_ACT_SWIGLU) {
    float g = dot(2 * n), u = dot(2 * n + 1);
    if (p.bias) { g += p.bias[2 * n]; u += p.bias[2 * n + 1]; }
    v = silu_f(g) * u;
  } else {
    v = dot(n);
    if (p.bias) v += p.bias[n];
    v = p.act == QB_ACT_SNAKE ? snake_f(v, p.act_p[n]) : apply_act(p.act, v);
  }
  epi_finish_scalar(p, b, m, n, v);
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

static int make_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                    const cuuint32_t* box, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                    CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode();
  QB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = enc(m, dtype, rank, const_cast<void*>(base), dims, strides_bytes, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  QB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed: %d (rank %d dims %llu %llu %llu)", (int)r, rank,
             (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0));
  return 0;
}

static RowMapD to_rm(const qb_rowmap& r) { return RowMapD{r.ptr, (long long)r.ld, (long long)r.rows_per_batch, (long long)r.row_off}; }

static bool aligned(const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; }

// Output columns of a launch: SwiGLU reduces each interleaved (gate, up) pair of the N GEMM columns to one.
static int out_cols(const GemmParams& p) { return p.act == QB_ACT_SWIGLU ? p.N / 2 : p.N; }

// A row map TMA can address as [batch][m_per_batch][out_cols] based at row `off`: 16-byte aligned base and row pitch, columns
// within the pitch, batches that do not overlap, and rows of whole 16-byte chunks.  The last condition is measured, not
// assumed: on an H100 a TMA store into a row that ends inside a 16-byte chunk wrote the pad columns of that chunk
// (tests/test_gemm_tma_planes_gpu.py, SwiGLU at 100 fp16 columns), so such rows, the decoder head's 1922 fp32 columns among
// them, stay on the generic epilogue.
static bool tma_rows(const RowMapD& r, long long esize, const GemmParams& p) {
  return r.ld >= out_cols(p) && (r.ld * esize) % 16 == 0 && (out_cols(p) * esize) % 16 == 0 && aligned(r.ptr, 16) &&
         (p.a_batch == 1 || r.rpb >= r.off + p.m_per_batch);
}

// The epilogues the fast kinds compute, when the TMA requirements hold for every buffer the kind reads or writes; each kind
// computes what epilogue_pair would.  The 128 x 256 tile holds 128 accumulators per thread: there the lo plane, ELU, SwiGLU and
// the planes of EPI_F32 would take the epilogue past the consumers' 232 registers (ptxas spills), so that tile keeps bias
// (GELU) -> hi and the fp32 kind without planes, and leaves the rest to the generic epilogue.
static int classify_epilogue(const GemmParams& p, int BN) {
  const bool wide = BN == 256;
  const bool planes_ok = !p.ohi.ptr || (tma_rows(p.ohi, 2, p) && (!p.olo.ptr || tma_rows(p.olo, 2, p)));
  if (p.ohi.ptr && !p.o32.ptr && !p.res.ptr && !p.gamma && p.act2 == QB_ACT_NONE && planes_ok &&
      (wide ? !p.olo.ptr && (p.act == QB_ACT_NONE || p.act == QB_ACT_GELU)
            : p.act == QB_ACT_NONE || p.act == QB_ACT_GELU || p.act == QB_ACT_ELU || p.act == QB_ACT_SWIGLU))
    return EPI_HI;
  if (p.o32.ptr && p.act == QB_ACT_NONE && (wide ? !p.ohi.ptr : p.act2 == QB_ACT_NONE || p.act2 == QB_ACT_ELU) && planes_ok &&
      tma_rows(p.o32, 4, p) && (!p.res.ptr || tma_rows(p.res, 4, p)))
    return EPI_F32;
  return EPI_GENERIC;
}

// Output / residual / planes map of the fast epilogue kinds: [batch][m_per_batch][out_cols] from row `off`, one 64-row box
// per subtile, 128 bytes wide (128-byte swizzle) or, for the planes of EPI_F32, 64 bytes (64-byte swizzle).
static int make_rows_map(CUtensorMap* m, const RowMapD& r, bool f32, int box_bytes, const GemmParams& p) {
  const cuuint64_t es = f32 ? 4 : 2, ld = (cuuint64_t)r.ld;
  const cuuint64_t rows = p.a_batch > 1 ? (cuuint64_t)r.rpb : (cuuint64_t)p.m_per_batch;
  cuuint64_t dims[3] = {(cuuint64_t)out_cols(p), (cuuint64_t)p.m_per_batch, (cuuint64_t)p.a_batch};
  cuuint64_t str[2] = {ld * es, rows * ld * es};
  cuuint32_t box[3] = {(cuuint32_t)(box_bytes / es), 64, 1};
  return make_map(m, (const char*)r.ptr + r.off * ld * es, 3, dims, str, box,
                  f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                  box_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
}

static int fill_params(const qb_gemm_desc* d, GemmParams* p, int BN) {
  QB_REQUIRE(d && d->a_hi && d->w_hi, "gemm: null operand");
  QB_REQUIRE((d->a_lo == nullptr) == (d->w_lo == nullptr), "gemm: a_lo and w_lo must both be given or both be NULL");
  QB_REQUIRE(d->taps >= 1 && d->stride >= 1, "gemm: bad taps/stride");
  QB_REQUIRE(d->a_ld % 64 == 0 && d->a_ld > 0, "gemm: a_ld (%lld) must be a positive multiple of 64", (long long)d->a_ld);
  QB_REQUIRE(d->a_rows_per_batch % d->stride == 0, "gemm: a_rows_per_batch must be a multiple of stride");
  QB_REQUIRE(d->a_batch >= 1 && d->m_per_batch >= 1 && d->n >= 1, "gemm: empty problem");
  QB_REQUIRE(d->act != QB_ACT_SWIGLU || d->n % 2 == 0, "gemm: SWIGLU needs even n");
  QB_REQUIRE(!d->out_lo.ptr || d->out_hi.ptr, "gemm: out_lo without out_hi");
  QB_REQUIRE(d->act != QB_ACT_SNAKE || d->act_param, "gemm: QB_ACT_SNAKE needs act_param (alpha[n])");
  QB_REQUIRE(d->act2 != QB_ACT_SNAKE || (d->act2_param && (reinterpret_cast<uintptr_t>(d->act2_param) & 7) == 0),
             "gemm: act2 = QB_ACT_SNAKE needs an 8-byte aligned act2_param (alpha[n])");
  memset(p, 0, sizeof(*p));
  p->tiles_per_batch = (int)ceil_div(d->m_per_batch, 128);
  p->num_n_tiles = (int)ceil_div(d->n, BN);
  p->num_tiles = (int)(d->a_batch * p->tiles_per_batch * p->num_n_tiles);
  const int64_t ck = d->a_cols > 0 ? d->a_cols : d->a_ld;
  QB_REQUIRE(ck % 64 == 0 && ck <= d->a_ld, "gemm: a_cols (%lld) must be a multiple of 64 and <= a_ld", (long long)ck);
  p->taps = d->taps; p->stride = d->stride; p->C = (int)ck; p->Cld = (int)d->a_ld; p->cblocks = (int)(ck / 64);
  p->dil = d->dilation > 0 ? d->dilation : 1;
  p->num_kb = p->taps * p->cblocks;
  p->m_per_batch = (int)d->m_per_batch; p->N = (int)d->n;
  p->bias = d->bias; p->gamma = d->gamma; p->act_p = d->act_param; p->act2_p = d->act2_param;
  p->res = to_rm(d->residual); p->o32 = to_rm(d->out_f32); p->ohi = to_rm(d->out_hi); p->olo = to_rm(d->out_lo);
  if (p->olo.ptr) { p->olo.ld = p->ohi.ld; p->olo.rpb = p->ohi.rpb; p->olo.off = p->ohi.off; }
  p->act = d->act; p->act2 = d->act2;
  p->a_hi = (const __half*)d->a_hi; p->a_lo = (const __half*)d->a_lo;
  p->w_hi = (const __half*)d->w_hi; p->w_lo = (const __half*)d->w_lo;
  p->a_rpb = d->a_rows_per_batch; p->a_batch = (int)d->a_batch;
  p->epi = classify_epilogue(*p, BN);
  return 0;
}

template <int NTERMS, int BN, int STAGES>
static int launch_tc(const qb_gemm_desc* d, cudaStream_t st, int num_sms) {
  GemmParams p;
  if (int e = fill_params(d, &p, BN)) return e;
  CUtensorMap mA_hi, mA_lo, mW_hi, mW_lo;
  const cuuint64_t C = (cuuint64_t)d->a_ld, s = (cuuint64_t)d->stride;
  cuuint64_t adims[3] = {s * C, (cuuint64_t)d->a_rows_per_batch / s, (cuuint64_t)d->a_batch};
  cuuint64_t astr[2] = {s * C * 2, (cuuint64_t)d->a_rows_per_batch * C * 2};
  cuuint32_t abox[3] = {64, 128, 1};
  const cuuint64_t Ck = (cuuint64_t)(d->a_cols > 0 ? d->a_cols : d->a_ld);
  cuuint64_t wdims[2] = {(cuuint64_t)d->taps * Ck, (cuuint64_t)d->n};
  cuuint64_t wstr[1] = {(cuuint64_t)d->taps * Ck * 2};
  cuuint32_t wbox[2] = {64, (cuuint32_t)BN};
  if (int e = make_map(&mA_hi, d->a_hi, 3, adims, astr, abox)) return e;
  if (int e = make_map(&mW_hi, d->w_hi, 2, wdims, wstr, wbox)) return e;
  if (NTERMS == 3) {
    if (int e = make_map(&mA_lo, d->a_lo, 3, adims, astr, abox)) return e;
    if (int e = make_map(&mW_lo, d->w_lo, 2, wdims, wstr, wbox)) return e;
  } else {
    mA_lo = mA_hi; mW_lo = mW_hi;
  }
  CUtensorMap mOut = mA_hi, mRes = mA_hi, mHi = mA_hi, mLo = mA_hi;             // used by the fast epilogue kinds only
  if (p.epi == EPI_F32) {
    if (int e = make_rows_map(&mOut, p.o32, true, 128, p)) return e;
    if (p.res.ptr)
      if (int e = make_rows_map(&mRes, p.res, true, 128, p)) return e;
  }
  if (p.epi != EPI_GENERIC && p.ohi.ptr) {
    const int box_bytes = p.epi == EPI_HI ? 128 : 64;
    if (int e = make_rows_map(&mHi, p.ohi, false, box_bytes, p)) return e;
    if (p.olo.ptr)
      if (int e = make_rows_map(&mLo, p.olo, false, box_bytes, p)) return e;
  }
  constexpr int NPL = NTERMS == 1 ? 1 : 2;
  // pipeline stages, epilogue subtile buffers, the tile's bias / gamma, mbarriers, and up to 896 bytes that align the
  // (128-byte aligned) base to 1024
  constexpr size_t smem = (size_t)STAGES * NPL * (GEMM_BM * 64 * 2 + BN * 64 * 2) + 2 * EPI_BUFS * EPI_SUB_BYTES + 2 * BN * 4 +
                          (2 * STAGES + 2 * EPI_BUFS) * 8 + 1024 - 128;
  static_assert(smem <= 227 * 1024, "GEMM pipeline and epilogue buffers exceed the 227 KB of shared memory a block may use");
  auto kern = gemm_tc_kernel<NTERMS, BN, STAGES>;
  static bool attr_set[QB_MAX_DEVICES] = {};          // the opt-in shared-memory limit is per-device state
  const int dev = current_device();
  if (!attr_set[dev]) {
    QB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[dev] = true;
  }
  int grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  kern<<<grid, GEMM_THREADS, smem, st>>>(mA_hi, mA_lo, mW_hi, mW_lo, mOut, mRes, mHi, mLo, p);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int num_sms_cached() {
  static int n[QB_MAX_DEVICES] = {};
  const int dev = current_device();
  if (!n[dev]) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (const char* e = getenv("QB_GEMM_SMS")) n[dev] = atoi(e);
  }
  return n[dev];
}

}  // namespace qb

using namespace qb;

extern "C" const char* qb_last_error(void) { return g_err; }
extern "C" int qb_version(void) { return 100; }
extern "C" int64_t qb_launch_count(void) { return (int64_t)g_launches.load(); }
extern "C" void qb_launch_count_reset(void) { g_launches = 0; }

// Three instantiations of one kernel, every stage 128 rows x 64 K, 192 KB of pipeline each (plus 32 KB of epilogue buffers):
//   single pass, n > 128:  128 x 256 tiles, 4 stages (48 KB)
//   single pass, n <= 128: 128 x 128 tiles, 6 stages (32 KB) - a 256-wide tile would be at least half padding
//   hi + lo split:         128 x 128 tiles, 3 stages (64 KB)
extern "C" const char* qb_gemm_kernel_name(int64_t m_per_batch, int64_t n, int32_t split) {
  (void)m_per_batch;
  if (split) return "gemm_tc_kernel<3,128,3>";
  return n > 128 ? "gemm_tc_kernel<1,256,4>" : "gemm_tc_kernel<1,128,6>";
}

extern "C" int qb_gemm(const qb_gemm_desc* d, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(d != nullptr, "gemm: null desc");
  const int sms = num_sms_cached();
  if (d->a_lo != nullptr) return launch_tc<3, 128, 3>(d, st, sms);
  return d->n > 128 ? launch_tc<1, 256, 4>(d, st, sms) : launch_tc<1, 128, 6>(d, st, sms);
}

extern "C" int qb_gemm_simt(const qb_gemm_desc* d, void* stream) {
  GemmParams p;
  if (int e = fill_params(d, &p, 128)) return e;
  const long long n_out = d->act == QB_ACT_SWIGLU ? d->n / 2 : d->n;
  const long long total = d->a_batch * d->m_per_batch * n_out;
  gemm_simt_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(p);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
