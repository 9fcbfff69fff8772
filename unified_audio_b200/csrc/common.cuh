// Shared device helpers for libquark_b200 (sm_90a).
// Raw PTX wrappers for mbarrier / TMA - no CUTLASS dependency (wgmma wrappers: wgmma.cuh).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace qb {

// ---------------------------------------------------------------- error plumbing (host)
void set_error(const char* fmt, ...);
#define QB_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      qb::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return -2;                                                                         \
    }                                                                                    \
  } while (0)
#define QB_REQUIRE(cond, ...)                                                            \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      qb::set_error(__VA_ARGS__);                                                        \
      return -1;                                                                         \
    }                                                                                    \
  } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------- small device math
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// GELU(x) = x * Phi(x) with erf from Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7, i.e. fp32-level):
// ~17 instructions, 2 MUFU - the epilogue of the ConvNeXt pwconv1 GEMM is otherwise erff-bound.
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  p *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z * z));
  const float erf_abs = fmaf(-p, e, 1.0f);           // erf(|x|/sqrt2)
  const float half_x = 0.5f * x;
  return fmaf(fabsf(half_x), erf_abs, half_x);        // 0.5x(1 + sign(x) erf(|z|))
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + __expf(-x)); }
__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }
// cached-decode attention: keys whose K / V rows one lane keeps in flight per trip (llm.cu lm_decode_attn2_kernel)
#ifndef LM_ATT_U_DEFAULT
#define LM_ATT_U_DEFAULT 8
#endif
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float elu_f(float x) { return x > 0.f ? x : expm1f(x); }

// fp32 -> fp16 rounded to nearest and saturated to +-65504 (infinities included), NaN kept as NaN: one cvt .satfinite.
// (A clamp with fminf / fmaxf, or __hmin2 / __hmax2, returns the non-NaN operand and would turn a NaN into a finite value; the
// half2 stores of the GEMM epilogue clamp with __hmin2_nan / __hmax2_nan.)
__device__ __forceinline__ __half f2h_sat(float x) {
  unsigned short h;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(x));
  return __ushort_as_half(h);
}
// fp32 -> (hi, lo) fp16 planes.  hi = rn(x) saturated to the fp16 range, lo = rn(x - hi).
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  hi = f2h_sat(x);
  lo = __float2half_rn(x - __half2float(hi));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------- PTX: mbarrier / TMA
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t elect.sync _|P, 0xffffffff;\n\t selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a mis-programmed pipeline traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) { asm volatile("trap;"); }
  }
}

// Same wait for warps that have slack (epilogue warps waiting for their accumulator tile, producers waiting for a free stage):
// try_wait with a suspend-time hint parks the thread in hardware until the phase completes (or the hint expires) instead of
// spinning on the barrier, so that waiting warps do not take issue slots from the ones doing the work.
__device__ __forceinline__ void mbar_wait_parked(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(200000u)
        : "memory");
    if (ok) return;
    if (++spins > (1u << 22)) { asm volatile("trap;"); }
  }
}

// Warpgroup register reallocation (sm_90a): every thread of the warpgroup executes it; the block's pool is fixed at launch by
// the kernel's register count, so the decreases of some warpgroups must free what the increases of the others take.
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(x), "r"(y)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
      : "memory");
}
// TMA store of one box from shared memory; elements outside the tensor map's bounds are not written.  Completion is tracked by
// bulk groups: commit after the store, then wait (.read: until the shared-memory source may be overwritten).
__device__ __forceinline__ void tma_store_3d(const void* tmap, const void* smem_src, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(tmap), "r"(smem_u32(smem_src)), "r"(x), "r"(y), "r"(z)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// shared-memory accesses by 32-bit address (a generic pointer takes two registers)
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y));
}
__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v));
}
__device__ __forceinline__ void st_shared_b16(uint32_t addr, __half v) {
  asm volatile("st.shared.b16 [%0], %1;" ::"r"(addr), "h"(__half_as_ushort(v)));
}
// barrier over `count` threads (a multiple of 32) under barrier id `id` (0 is __syncthreads')
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

}  // namespace qb
