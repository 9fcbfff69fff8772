// LSTM recurrence on the Hopper tensor cores (wgmma + TMA + mbarrier), persistent cooperative kernel.
// Reference: nn.LSTM(H,H,1,batch_first), HCodec-2.0/vq/encoder_modules/transformer.py:115,133.
//
// Each CTA keeps its W_hh slice [4U gate rows x H] resident in shared memory as the wgmma *B* operand (K-major, 128B swizzle,
// loaded once by TMA) and streams h_{t-1} (fp16, published by all CTAs) through a bulk-copy ring as the *A* operand; the gates
// accumulate in registers of the consumer warpgroups.
//
// The batch is split into GROUPS of 32 rows that are independent recurrences: group g is served by consumer warpgroup g (own
// accumulators, own flags).  The groups are software-pipelined: while group g waits for the grid-wide publication of its h_t
// (epilogue + fence + flag round trip), the TMA ring and the other warpgroups' MMAs carry the other groups' steps.  wgmma reads 64
// A rows: a group's 32 rows are rows 0..31 of the tile, rows 32..63 read whatever finite fp16 data follows the K-block in the ring
// (zeroed pad past its end) and only produce accumulators nobody reads (warps 2-3 of the warpgroup).
// W rows are pre-permuted by the host to unit-major order: row (4*j + g) of CTA c = gate g of unit c*U + j.
#include <atomic>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "quark_b200.h"
#include "wgmma.cuh"

namespace qb {
extern std::atomic<long long> g_launches;

constexpr int LT_GROUPS = 4, LT_THREADS = LT_GROUPS * 128 + 32;   // 4 consumer warpgroups + one producer warp
constexpr int LT_KG = 4;                          // K-blocks fetched by one bulk copy
constexpr int LT_STAGES = 4;                      // ring: 4 x (LT_KG x 4 KB) = 64 KB
constexpr uint32_t LT_KBLK = 32 * 128;            // one K-block of one group: 32 rows x 128 B
constexpr uint32_t LT_SLOT = LT_KBLK * LT_KG;
constexpr uint32_t LT_PAD = 4 * 1024;             // a 64-row A tile reads up to 4 KB past the last K-block of the ring

// flag polling: relaxed loads (the four of a lane are independent and in flight together - acquire loads would serialise
// into four L2 round trips per poll), one acquire fence once every flag has been seen
__device__ __forceinline__ unsigned lt_ld_relaxed(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// linear bulk copy global -> shared (no tensor map): the published h is stored tile-native (pre-swizzled)
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// Gate non-linearities of the epilogue: ex2.approx + rcp.approx (2^-21 relative on exp, 1 ulp on the reciprocal; absolute
// error < 3e-7 on sigmoid / tanh) - the epilogue sits on the step's critical chain.
__device__ __forceinline__ float lt_rcp(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float lt_sigmoid(float x) { return lt_rcp(1.0f + __expf(-x)); }
__device__ __forceinline__ float lt_tanh(float x) { return fmaf(-2.0f, lt_rcp(1.0f + __expf(2.0f * x)), 1.0f); }

template <int U>
__global__ void __launch_bounds__(LT_THREADS, 1)
lstm_tc_kernel(const __grid_constant__ CUtensorMap tmW,
               const float* __restrict__ xp, int B, int T, int H, __half* __restrict__ out_hi,
               __half* __restrict__ out_lo, __half* hbuf, unsigned* flags, int n_groups, int poll_ns) {
  constexpr int N = 4 * U;                      // gate rows of this CTA = wgmma N
  constexpr int UPT = N / 8;                    // units per epilogue thread
  static_assert(N % 16 == 0 && N <= 48, "unsupported slice width");
  constexpr uint32_t WBLK = N * 128;            // bytes of one [N x 64] K-block of W
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int KB = H / 64, SLOTS = KB / LT_KG;    // ring slots per group and step
  uint8_t* Wsm = smem;
  uint8_t* ring = smem + (size_t)KB * WBLK;     // KB*WBLK is a multiple of 1024 (N % 8 == 0)
  uint64_t* full = (uint64_t*)(ring + LT_STAGES * LT_SLOT + LT_PAD);
  uint64_t* empty = full + LT_STAGES;
  uint64_t* wbar = empty + LT_STAGES;
  // slot_tag[s]: index of the ring slot stage s currently holds (written by the producer once it owns the stage).  The groups share
  // the ring, so a warpgroup may wait for a slot whose stage is still several phases behind; a parity wait is only meaningful one
  // phase ahead, hence the tag is checked first.
  int* slot_tag = (int*)(wbar + 1);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int u0 = blockIdx.x * U, G = gridDim.x;

  if (tid == 0) {
    for (int s = 0; s < LT_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    mbar_init(wbar, 1);
    for (int s = 0; s < LT_STAGES; ++s) slot_tag[s] = -1;
    fence_mbar_init();
  }
  // ring + pad zeroed once: tile rows outside a group's K-block must be finite
  for (int i = tid; i < (int)((LT_STAGES * LT_SLOT + LT_PAD) / 16); i += LT_THREADS)
    reinterpret_cast<uint4*>(ring)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  if (warp == LT_GROUPS * 4) {
    // ===================== producer: flags -> bulk copies of h_{t-1} =====================
    if (lane == 0) {
      prefetch_tmap(&tmW);
      mbar_arrive_expect_tx(wbar, (uint32_t)KB * WBLK);
      for (int kb = 0; kb < KB; ++kb) tma_load_2d(Wsm + (size_t)kb * WBLK, &tmW, wbar, kb * 64, blockIdx.x * N);
    }
    uint32_t stage = 0, phase = 0;
    int slot = 0;
    for (int t = 1; t < T; ++t) {
      for (int g = 0; g < n_groups; ++g) {
        // wait until every CTA has published h_{t-1} of group g
        const unsigned* fl = flags + (size_t)g * G;
        unsigned spins = 0;
        for (;;) {
          bool ok = true;
          for (int c = lane; c < G; c += 32) ok = ok && (lt_ld_relaxed(fl + c) >= (unsigned)t);
          if (__all_sync(0xffffffffu, ok)) break;
          if (poll_ns) __nanosleep(poll_ns);                    // optional back-off (relaxed polls are cheap: none by default)
          if (++spins > (1u << 24)) asm volatile("trap;");
        }
        asm volatile("fence.acq_rel.gpu;" ::: "memory");        // acquire side of the flags every lane has just observed
        __syncwarp();
        if (lane == 0) {
          asm volatile("fence.proxy.async;" ::: "memory");    // generic-proxy writes of h -> async-proxy (bulk copy) reads
          const int buf = (t + 1) & 1;                          // h_{t-1} lives in buffer (t-1)&1
          for (int kb = 0; kb < KB; kb += LT_KG, ++slot) {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], LT_SLOT);
            __threadfence_block();
            *(volatile int*)(slot_tag + stage) = slot;
            bulk_load_1d(ring + stage * LT_SLOT, hbuf + (((size_t)buf * n_groups + g) * KB + kb) * (LT_KBLK / 2), LT_SLOT,
                         &full[stage]);
            if (++stage == LT_STAGES) { stage = 0; phase ^= 1; }
          }
        }
        __syncwarp();
      }
    }
  } else {
    // ===================== consumer warpgroup g: gates = h_{t-1} W^T, then the cell update of its 32 rows =====================
    const int g = warp >> 2, wq = warp & 3;
    if (g < n_groups) {
      // accumulator (row 16 wq + lane / 4 (+8), columns 8j + 2 (lane % 4) + {0, 1}): an even lane holds gates i, f and an odd lane
      // gates g, o of unit 2j + (lane / 2) % 2 for both rows; one exchange gives an even lane row +0 and an odd lane row +8
      const int rr = wq * 16 + (lane >> 2) + (lane & 1) * 8;     // row of the group this thread updates (wq < 2)
      const int n = g * 32 + rr;
      const bool act = wq < 2 && n < B;
      float c[UPT];
#pragma unroll
      for (int i = 0; i < UPT; ++i) c[i] = 0.f;
      mbar_wait(wbar, 0);
      for (int t = 0; t < T; ++t) {
        // tile-native layout [buf][group][K-block][32 rows][128 B], 16-byte chunks XOR-swizzled by (row & 7)
        __half* hcur = hbuf + ((size_t)(t & 1) * n_groups + g) * KB * (LT_KBLK / 2);
        float xg[4][UPT];
#pragma unroll
        for (int gg = 0; gg < 4; ++gg)
#pragma unroll
          for (int j = 0; j < UPT; ++j)
            xg[gg][j] = act ? xp[((long long)n * T + t) * 4 * H + (long long)gg * H + u0 + 2 * j + ((lane >> 1) & 1)] : 0.f;
        float acc[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        if (t > 0) {
          // ring slot index of this group's first slot of step t (the producer fills slots in (t, group, K) order)
          const long long s0 = ((long long)(t - 1) * n_groups + g) * SLOTS;
          for (int sidx = 0; sidx < SLOTS; ++sidx) {
            const long long q = s0 + sidx;
            const int stage = (int)(q % LT_STAGES);
            unsigned spins = 0;
            while (*(volatile int*)(slot_tag + stage) != (int)q)
              if (++spins > (1u << 26)) asm volatile("trap;");
            __threadfence_block();
            mbar_wait(&full[stage], (uint32_t)((q / LT_STAGES) & 1));
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < LT_KG; ++j) {
              const int kb = sidx * LT_KG + j;
              const uint32_t sa = smem_u32(ring + stage * LT_SLOT + j * LT_KBLK), sw = smem_u32(Wsm + (size_t)kb * WBLK);
#pragma unroll
              for (int k = 0; k < 4; ++k)
                Wgmma<N>::ss(acc, make_wgmma_desc_sw128(sa + k * 32), make_wgmma_desc_sw128(sw + k * 32), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(acc);
            if (lane == 0) mbar_arrive(&empty[stage]);
          }
        }
        if (wq < 2) {
          const bool odd = lane & 1;
#pragma unroll
          for (int j = 0; j < UPT; ++j) {
            const float s0 = odd ? acc[4 * j] : acc[4 * j + 2], s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
            const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
            const float a_i = odd ? r0 : acc[4 * j], a_f = odd ? r1 : acc[4 * j + 1];
            const float a_g = odd ? acc[4 * j + 2] : r0, a_o = odd ? acc[4 * j + 3] : r1;
            if (act) {
              const float ig = lt_sigmoid(a_i + xg[0][j]), fg = lt_sigmoid(a_f + xg[1][j]);
              const float cg = lt_tanh(a_g + xg[2][j]), og = lt_sigmoid(a_o + xg[3][j]);
              const float cn = fg * c[j] + ig * cg;
              c[j] = cn;
              __half hv, lv;
              split_f16(og * lt_tanh(cn), hv, lv);
              const int uu = u0 + 2 * j + ((lane >> 1) & 1), kbk = uu >> 6, col = uu & 63;
              hcur[kbk * (int)(LT_KBLK / 2) + rr * 64 + ((((col >> 3) ^ (rr & 7)) << 3) | (col & 7))] = hv;
              const long long o = ((long long)n * T + t) * H + uu;
              out_hi[o] = hv;
              if (out_lo) out_lo[o] = lv;
            }
          }
          // publish h_t of this group: both warps of the group done (h stores) -> flag
          asm volatile("bar.sync %0, 64;" ::"r"(1 + g) : "memory");
          if (wq == 0 && lane == 0) {   // release is cumulative over the group's h stores ordered before it by the bar.sync
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flags + (size_t)g * G + blockIdx.x), "r"((unsigned)(t + 1))
                         : "memory");
          }
        }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn lt_encode() {
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

static int lstm_tc_chunk(const float* xp, const qb_half* whh_perm, int U, int B, int64_t T, int64_t H, __half* oh, __half* ol,
                         void* workspace, cudaStream_t st) {
  const int N = 4 * U, grid = (int)(H / U), KB = (int)(H / 64);
  const int n_groups = (B + 31) / 32, Bp = n_groups * 32;
  EncodeTiledFn enc = lt_encode();
  QB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available");
  CUtensorMap tmW;
  {
    cuuint64_t dims[2] = {(cuuint64_t)H, (cuuint64_t)(4 * H)};
    cuuint64_t str[1] = {(cuuint64_t)H * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)N};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&tmW, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)whh_perm, dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    QB_REQUIRE(r == CUDA_SUCCESS, "lstm_tc: W tensor map failed (%d)", (int)r);
  }
  // published h: tile-native [buffer][group][K-block][32 rows][128 B] (pre-swizzled), read with linear bulk copies
  __half* hbuf = (__half*)workspace;
  const size_t smem = (size_t)KB * N * 128 + (size_t)LT_STAGES * LT_SLOT + LT_PAD + 1024 + 256;
  QB_REQUIRE(smem <= 227 * 1024, "lstm_tc: shared memory budget exceeded (%zu)", smem);
  const size_t hbytes = (size_t)2 * Bp * H * 2;
  QB_CHECK_CUDA(cudaMemsetAsync(workspace, 0, hbytes + 4096, st));
  unsigned* flags = (unsigned*)((uint8_t*)workspace + hbytes);
  int Bi = B, Ti = (int)T, Hi = (int)H, ng = n_groups;
  static int poll_ns = -1;
  if (poll_ns < 0) { const char* e = getenv("QB_LSTM_POLL_NS"); poll_ns = e ? atoi(e) : 0; }   // optional back-off of the flag polls
  void* args[] = {&tmW, &xp, &Bi, &Ti, &Hi, &oh, &ol, &hbuf, &flags, &ng, &poll_ns};
  const void* fn = U == 4 ? (const void*)lstm_tc_kernel<4> : U == 8 ? (const void*)lstm_tc_kernel<8> : (const void*)lstm_tc_kernel<12>;
  QB_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  QB_CHECK_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(LT_THREADS), args, smem, st));
  g_launches++;
  return 0;
}

}  // namespace qb
using namespace qb;

extern "C" int32_t qb_lstm_tc_units(int64_t H) {
  // units per CTA: H/U CTAs must be co-resident (<= SM count) and 4U a multiple of 16
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    sms = 132;
  for (int U : {4, 8, 12}) if (H % U == 0 && H / U <= sms) return U;
  return 0;
}

extern "C" int64_t qb_lstm_tc_workspace_bytes(int64_t B, int64_t H) {
  const int64_t Bc = B < 128 ? B : 128;                 // rows processed by one launch
  const int64_t Bp = ceil_div(Bc, 32) * 32;
  return 2 * Bp * H * 2 + 4096;
}

extern "C" int qb_lstm_tc(const float* xp, const qb_half* whh_perm, int32_t units, int64_t B, int64_t T, int64_t H,
                          qb_half* out_hi, qb_half* out_lo, void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(xp && whh_perm && out_hi && workspace, "lstm_tc: bad args");
  QB_REQUIRE(H % (64 * LT_KG) == 0 && (units == 4 || units == 8 || units == 12) && H % units == 0, "lstm_tc: unsupported H / units");
  QB_REQUIRE(B >= 1, "lstm_tc: empty batch");
  for (int64_t b0 = 0; b0 < B; b0 += 128) {              // <= 4 groups of 32 rows per launch
    const int bc = (int)(B - b0 < 128 ? B - b0 : 128);
    if (int e = lstm_tc_chunk(xp + b0 * T * 4 * H, whh_perm, units, bc, T, H, (__half*)out_hi + b0 * T * H,
                              out_lo ? (__half*)out_lo + b0 * T * H : nullptr, workspace, st))
      return e;
  }
  return 0;
}
