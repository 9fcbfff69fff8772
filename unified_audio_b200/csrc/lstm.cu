// Single-layer LSTM recurrence as ONE persistent cooperative kernel
// (reference: nn.LSTM(H,H,1,batch_first) inside every attention block,
//  HCodec-2.0/vq/encoder_modules/transformer.py:115,133).
//
// The input projection x W_ih^T + b_ih + b_hh is done beforehand by the wgmma GEMM (xp).  Here:
//  * hidden units are sharded over CTAs (U = 4*MT units -> 16*MT gate rows i|f|g|o per CTA);
//    the CTA's fp16 W_hh slice stays resident in shared memory for all T steps;
//  * per step every CTA computes gates[16*MT x B] = W_slice . h_{t-1}^T with mma.sync m16n8k16
//    (fp16 in, fp32 accumulate); h_{t-1} (fp16, [B][H], double buffered in global/L2) is loaded
//    straight into B-fragments with 64-bit L2 loads - W's K order is permuted once at load so
//    that each thread's 4 fragment halves are contiguous in memory;
//  * 8 warps = 2 batch halves x 4 K quarters, partial sums reduced through shared memory;
//  * cell state c stays in shared memory (fp32); h_t is published as fp16 and a grid-wide
//    monotonic-counter barrier separates the steps.
#include <atomic>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

constexpr int LSTM_THREADS = 256;
constexpr int LSTM_NB = 64;       // batch columns per chunk
constexpr int LSTM_REDP = 68;     // padded row pitch (floats) of the reduction buffer
constexpr int LSTM_REP = 1;       // replicas of the published h (spreads the all-CTA broadcast reads over L2)

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&a)[4], const void* smem_ptr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3])
               : "r"(smem_u32(smem_ptr)));
}
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int MT>
__global__ void __launch_bounds__(LSTM_THREADS, 1)
lstm_kernel(const float* __restrict__ xp, const __half* __restrict__ whh, int B, int T, int H,
            __half* __restrict__ out_hi, __half* __restrict__ out_lo, __half* hbuf, unsigned* counter, int Bp,
            long long* prof) {
  constexpr int ROWS = 16 * MT, U = 4 * MT;
  extern __shared__ __align__(16) uint8_t sm[];
  const int pitch = H + 8;  // halves; +16 B per row keeps ldmatrix conflict-free
  __half* Wsm = reinterpret_cast<__half*>(sm);
  float* red = reinterpret_cast<float*>(sm + (size_t)ROWS * pitch * 2);
  float* cs = red + 4 * ROWS * LSTM_REDP;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int u0 = blockIdx.x * U;
  const int G = gridDim.x;

  // one-time: W_hh slice -> smem, K order permuted inside every 32-block so that the 8 consecutive
  // memory halves a thread fetches with one 128-bit load are its B-fragment registers of two k16 steps:
  // logical 32-bit word wl (0..15) of a block <- memory word 4*(wl&3) + ((wl>>2)&1) + 2*(wl>>3)
  const int wpr = H / 2;  // 32-bit words per row
  for (int idx = tid; idx < ROWS * wpr; idx += LSTM_THREADS) {
    const int r = idx / wpr, wl = idx - r * wpr;
    const int kb = wl >> 4, w16 = wl & 15;
    const int memw = 4 * (w16 & 3) + ((w16 >> 2) & 1) + 2 * (w16 >> 3);
    const int g = r / U, j = r - g * U;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(whh + ((long long)g * H + u0 + j) * H);
    reinterpret_cast<uint32_t*>(Wsm + (size_t)r * pitch)[wl] = src[kb * 16 + memw];
  }
  for (int i = tid; i < Bp * U; i += LSTM_THREADS) cs[i] = 0.f;
  __syncthreads();

  const int nh = warp & 1, kq = warp >> 1;
  const int kb32_per_q = H / 128;  // 32-wide K blocks per K quarter
  const int n_chunks = Bp / LSTM_NB;

  long long pc[4] = {0, 0, 0, 0};
  for (int t = 0; t < T; ++t) {
    long long c0 = clock64();
    if (t > 0) {  // wait until every CTA has published h_{t-1}: per-CTA flags (no atomic serialisation)
      if (warp == 0) {
        unsigned spins = 0;
        for (;;) {
          bool ok = true;
          for (int c = lane; c < G; c += 32) ok = ok && (ld_acquire_u32(counter + c) >= (unsigned)t);
          if (__all_sync(0xffffffffu, ok)) break;
          if (++spins > (1u << 26)) asm volatile("trap;");
        }
      }
      __syncthreads();
    }
    long long c1 = clock64();
    pc[0] += c1 - c0;
    const __half* hprev = hbuf + ((size_t)((t + 1) & 1) * LSTM_REP + (blockIdx.x % LSTM_REP)) * Bp * H;
    __half* hcur = hbuf + (size_t)(t & 1) * LSTM_REP * Bp * H;

    for (int ch = 0; ch < n_chunks; ++ch) {
      const int nb0 = ch * LSTM_NB;
      // ---- prefetch this chunk's xp gate pre-activations (independent of the recurrence)
      constexpr int PAIRS = (U * LSTM_NB + LSTM_THREADS - 1) / LSTM_THREADS;
      float xg[PAIRS][4];
#pragma unroll
      for (int i = 0; i < PAIRS; ++i) {
        const int p = tid + i * LSTM_THREADS;
        const int j = p / LSTM_NB, n = nb0 + (p % LSTM_NB);
#pragma unroll
        for (int g = 0; g < 4; ++g)
          xg[i][g] = (p < U * LSTM_NB && n < B) ? xp[((long long)n * T + t) * 4 * H + (long long)g * H + u0 + j] : 0.f;
      }
      // ---- gates partial sums on the tensor cores
      float acc[MT][4][4];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
      if (t > 0) {
        const __half* hb = hprev + (size_t)(nb0 + nh * 32 + (lane >> 2)) * H + (lane & 3) * 8;
        const int kb_beg = kq * kb32_per_q, kb_end = kb_beg + kb32_per_q;   // 32-wide K blocks of this quarter
        for (int g0 = kb_beg; g0 < kb_end; g0 += 12) {
          uint4 bf[2][4][4];
          auto load_group = [&](int buf, int kb0) {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
              for (int nt = 0; nt < 4; ++nt)
                bf[buf][kk][nt] = (kb0 + kk < kb_end)
                                      ? __ldcg(reinterpret_cast<const uint4*>(hb + (size_t)nt * 8 * H + (kb0 + kk) * 32))
                                      : make_uint4(0u, 0u, 0u, 0u);
          };
          load_group(0, g0);
#pragma unroll
          for (int gi = 0; gi < 3; ++gi) {
            const int kb0 = g0 + gi * 4;
            if (gi + 1 < 3 && kb0 + 4 < kb_end) load_group((gi + 1) & 1, kb0 + 4);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
              if (kb0 + kk < kb_end) {
#pragma unroll
                for (int half = 0; half < 2; ++half) {
#pragma unroll
                  for (int mt = 0; mt < MT; ++mt) {
                    uint32_t a[4];
                    ldmatrix_x4(a, Wsm + (size_t)(mt * 16 + (lane & 15)) * pitch + (kb0 + kk) * 32 + half * 16 + (lane >> 4) * 8);
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                      const uint4 v = bf[gi & 1][kk][nt];
                      mma_16816(acc[mt][nt], a, half ? v.z : v.x, half ? v.w : v.y);
                    }
                  }
                }
              }
            }
          }
        }
      }
      long long c2 = clock64();
      pc[1] += c2 - c1;
      // ---- K-quarter partials -> smem
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int r = mt * 16 + (lane >> 2), c = nh * 32 + nt * 8 + (lane & 3) * 2;
          float* d0 = red + ((size_t)kq * ROWS + r) * LSTM_REDP + c;
          float* d1 = red + ((size_t)kq * ROWS + r + 8) * LSTM_REDP + c;
          d0[0] = acc[mt][nt][0]; d0[1] = acc[mt][nt][1];
          d1[0] = acc[mt][nt][2]; d1[1] = acc[mt][nt][3];
        }
      __syncthreads();
      // ---- pointwise cell update for (unit j, batch n) pairs
#pragma unroll
      for (int i = 0; i < PAIRS; ++i) {
        const int p = tid + i * LSTM_THREADS;
        if (p < U * LSTM_NB) {
          const int j = p / LSTM_NB, nl = p % LSTM_NB, n = nb0 + nl;
          float gsum[4];
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            float s = xg[i][g];
#pragma unroll
            for (int q4 = 0; q4 < 4; ++q4) s += red[((size_t)q4 * ROWS + g * U + j) * LSTM_REDP + nl];
            gsum[g] = s;
          }
          const float ig = sigmoid_acc(gsum[0]), fg = sigmoid_acc(gsum[1]), gg = tanhf(gsum[2]), og = sigmoid_acc(gsum[3]);
          const float c = fg * cs[(size_t)n * U + j] + ig * gg;
          cs[(size_t)n * U + j] = c;
          const float h = og * tanhf(c);
          __half hh, hl;
          split_f16(h, hh, hl);
#pragma unroll
          for (int rp = 0; rp < LSTM_REP; ++rp) hcur[((size_t)rp * Bp + n) * H + u0 + j] = hh;
          if (n < B) {
            const long long o = ((long long)n * T + t) * H + u0 + j;
            out_hi[o] = hh;
            if (out_lo) out_lo[o] = hl;
          }
        }
      }
      __syncthreads();  // red / cs reuse by the next chunk
      c1 = clock64();
      pc[2] += c1 - c2;
    }
    // ---- publish h_t
    if (tid == 0) {
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(counter + blockIdx.x), "r"((unsigned)(t + 1)) : "memory");
    }
    pc[3] += clock64() - c1;
  }
  if (prof && tid == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) {
    const int o = blockIdx.x == 0 ? 0 : 4;
    for (int i = 0; i < 4; ++i) prof[o + i] = pc[i];
  }
}

static int pick_mt(int64_t H, int sms) {
  for (int mt = 1; mt <= 3; ++mt) {
    const int64_t U = 4 * mt;
    if (H % U == 0 && H / U <= sms) return mt;
  }
  return 0;
}

}  // namespace qb
using namespace qb;

extern "C" int64_t qb_lstm_workspace_bytes(int64_t B, int64_t H) {
  const int64_t Bp = ceil_div(B, LSTM_NB) * LSTM_NB;
  return 2 * LSTM_REP * Bp * H * 2 + 4096;
}

extern "C" int qb_lstm(const float* xp, const qb_half* whh_hi, const qb_half* whh_lo, int64_t B, int64_t T, int64_t H,
                       qb_half* out_hi, qb_half* out_lo, void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(xp && whh_hi && out_hi && workspace, "lstm: bad args");
  QB_REQUIRE(whh_lo == nullptr, "lstm: split-precision recurrent weights are not supported (single-pass fp16 policy)");
  QB_REQUIRE(H % 128 == 0, "lstm: H must be a multiple of 128");
  int dev = 0, sms = 0;
  QB_CHECK_CUDA(cudaGetDevice(&dev));
  QB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int mt = pick_mt(H, sms);
  QB_REQUIRE(mt != 0, "lstm: cannot shard H=%lld over %d SMs", (long long)H, sms);
  const int Bp = (int)(ceil_div(B, LSTM_NB) * LSTM_NB);
  const int rows = 16 * mt, U = 4 * mt, grid = (int)(H / U);
  const size_t smem = (size_t)rows * (H + 8) * 2 + (size_t)4 * rows * LSTM_REDP * 4 + (size_t)Bp * U * 4;
  QB_REQUIRE(smem <= 227 * 1024, "lstm: shared memory budget exceeded (%zu bytes; B too large?)", smem);
  QB_CHECK_CUDA(cudaMemsetAsync(workspace, 0, (size_t)qb_lstm_workspace_bytes(B, H), st));
  __half* hbuf = (__half*)workspace;
  unsigned* counter = (unsigned*)((uint8_t*)workspace + (size_t)2 * LSTM_REP * Bp * H * 2);
  const __half* w = (const __half*)whh_hi;
  __half* oh = (__half*)out_hi;
  __half* ol = (__half*)out_lo;
  int Bi = (int)B, Ti = (int)T, Hi = (int)H, Bpi = Bp;
  static long long* prof = nullptr;
  if (!prof && getenv("QB_LSTM_PROF")) cudaMalloc(&prof, 64);
  void* args[] = {&xp, &w, &Bi, &Ti, &Hi, &oh, &ol, &hbuf, &counter, &Bpi, &prof};
  const void* fn = mt == 1 ? (const void*)lstm_kernel<1> : mt == 2 ? (const void*)lstm_kernel<2> : (const void*)lstm_kernel<3>;
  QB_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  QB_CHECK_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(LSTM_THREADS), args, smem, st));
  g_launches++;
  if (prof) {
    long long h[8];
    cudaStreamSynchronize(st);
    cudaMemcpy(h, prof, 64, cudaMemcpyDeviceToHost);
    fprintf(stderr, "[lstm prof] T=%d cycles/step cta0: wait %.0f mma %.0f reduce+pointwise %.0f publish %.0f | ctaN: wait %.0f mma %.0f rp %.0f pub %.0f\n", Ti,
            h[0] / (double)Ti, h[1] / (double)Ti, h[2] / (double)Ti, h[3] / (double)Ti, h[4] / (double)Ti, h[5] / (double)Ti, h[6] / (double)Ti, h[7] / (double)Ti);
  }
  return 0;
}
