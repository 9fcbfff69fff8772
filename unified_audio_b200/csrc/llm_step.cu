// UniSE AR-LM cached decode as ONE persistent cooperative kernel (QuarkAudio-UniSE/model/llm/llm_sft.py:137-193, greedy).
//
// The per-kernel decode step (llm.cu: 5 kernels per layer + 2 for the head = 62 dependent launches per token) is bound by
// launch-to-launch dependency latency rather than by its HBM traffic.  Here the
// whole generation loop runs inside one kernel of one CTA per SM: the 62 stages of a step are separated by a device-side grid
// barrier (one atomic arrive + one polled word) instead of a kernel boundary, every worker issues the weight loads of its
// next tile BEFORE it waits at the barrier (weights do not depend on activations), and all step state (position, output slot)
// lives in registers.  The arithmetic of every tile is the tile arithmetic of lm_skinny_kernel / lm_decode_attn2_kernel /
// lm_argmax_embed_kernel (same packed fp16 {hi,lo} weights, same 3-term mma.sync products, same fixed-order reductions), so
// the tokens are bit-identical to the per-kernel path.
//
// Work decomposition (CTA = 512 threads = two 256-thread workers; W = 2 x #CTAs workers):
//   QKV     3*heads*4 tiles of 16 columns (RMSNorm scale, RoPE, K/V cache append)      256-thread workers
//   ATT     heads*B items (flash-decoding over the fp32 cache)                          256-thread workers
//   OPROJ   hidden/8 tiles (+ residual)                                                 256-thread workers
//   GATEUP  inter/8 tiles (RMSNorm scale, SwiGLU)                                       256-thread workers
//   DOWN    hidden/8 tiles, K = inter (+ residual)                                      whole CTA (16 warps split K)
//   HEAD    range/16 tiles (final RMSNorm scale, arg-max partials)                      256-thread workers
//   ARGMAX  B items (token, next input embedding)                                       256-thread workers
// Activations written by other SMs are read with ld.global.cg (L1 is not coherent across SMs inside a kernel).
#include <atomic>
#include <cstdio>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

constexpr int LM_ATT_U = LM_ATT_U_DEFAULT;      // same key grouping as lm_decode_attn2_kernel: bit-identical tokens
constexpr int ST_MAX_LAYERS = 16, ST_THREADS = 512, ST_WSMEM = 4608;       // floats of shared memory per 256-thread worker

struct StepLayer {
  const uint4 *wqkv, *wo, *wg, *wu, *wd;
  float *kc, *vc;
};
struct StepParams {
  int B, hidden, heads, inter, layers, Lmax, n_steps, out_stride;
  StepLayer L[ST_MAX_LAYERS];
  const uint4* whead;
  float *x, *q_buf, *attn_buf, *mlp_buf;
  const float *rcos, *rsin, *emb;
  int *pos, *slot;
  const int* range;
  float* part_val;
  int* part_idx;
  int64_t* out_ids;
  unsigned* bar;
  float eps;
  int dbg;       // bit 0: skip the grid barriers, bit 1: skip the tile arithmetic (timing aids, QB_LM_STEP_DBG)
};

enum { TK_QKV = 0, TK_RESID = 1, TK_GATEUP = 2, TK_HEAD = 3 };

__device__ __forceinline__ void st_mma(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void worker_sync(int bar_id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// all CTAs of the (cooperative) grid; `epoch` counts arrivals expected so far (thread 0 of every CTA keeps it in a register).
// Arrive: one release reduction (cumulative over the CTA's stores ordered before it by the bar.sync); wait: relaxed polls of
// the one word, then ONE acquire fence (an acquire load per poll costs a fence per iteration).
__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned& epoch, unsigned n_ctas, int dbg) {
  if (dbg & 1) { __syncthreads(); return; }      // timing aid only (results undefined)
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += n_ctas;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
    unsigned spins = 0;
    while (ld_relaxed_u32(ctr) < epoch) {
      if (++spins > (1u << 28)) asm volatile("trap;");
    }
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------- skinny projection tiles
// One tile = 8 (RESID) or 16 output columns x 32 batch rows x K; NW warps split K (SPW k-steps of 16 each) and sum through
// shared memory in a fixed order - the body of lm_skinny_kernel with (bid, tid) explicit.
template <int MODE, int SPW, int NW>
struct SkTile {
  static constexpr int NT = MODE == TK_RESID ? 1 : 2;
  struct Info {
    const uint4* wrow[NT];
    bool active;
    int row0, dd0, hh, sec;
  };
  __device__ static __forceinline__ void locate(const StepParams& p, const uint4* W, const uint4* W2, int K, int bid, int tid, Info& ti) {
    const int lane = tid & 31, g = lane >> 2, K4 = K >> 2;
    ti.active = true; ti.row0 = 0; ti.dd0 = 0; ti.hh = 0; ti.sec = 0;
    if (MODE == TK_QKV) {
      ti.dd0 = (bid & 3) * 8; ti.hh = (bid >> 2) % p.heads; ti.sec = bid / (4 * p.heads);
      ti.row0 = ti.sec * p.heads * 64 + ti.hh * 64 + ti.dd0;
      ti.wrow[0] = W + (size_t)(ti.row0 + g) * K4;
      if (NT > 1) ti.wrow[NT - 1] = W + (size_t)(ti.row0 + 32 + g) * K4;
    } else if (MODE == TK_RESID) {
      ti.row0 = bid * 8;
      ti.wrow[0] = W + (size_t)(ti.row0 + g) * K4;
    } else if (MODE == TK_GATEUP) {
      ti.row0 = bid * 8;
      ti.wrow[0] = W + (size_t)(ti.row0 + g) * K4;
      if (NT > 1) ti.wrow[NT - 1] = W2 + (size_t)(ti.row0 + g) * K4;
    } else {
      const int lo = p.range[0], ncol = p.range[1] - lo;
      ti.active = bid * 16 < ncol;
      ti.row0 = lo + (ti.active ? bid * 16 : 0);
      ti.wrow[0] = W + (size_t)(ti.row0 + g) * K4;
      if (NT > 1) ti.wrow[NT - 1] = W + (size_t)(ti.row0 + 8 + g) * K4;
    }
  }
  __device__ static __forceinline__ void load_w(const Info& ti, int K, int tid, uint4 (&wv)[NT][SPW]) {
    const int lane = tid & 31, warp = tid >> 5, t = lane & 3, steps_total = K >> 4;
#pragma unroll
    for (int s = 0; s < SPW; ++s) {
      const int step = warp * SPW + s;
      const bool ok = step < steps_total && ti.active;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) wv[nt][s] = ok ? __ldg(ti.wrow[nt] + step * 4 + t) : make_uint4(0u, 0u, 0u, 0u);
    }
  }
  // x [B,K] activations (other SMs' writes: ld.cg); smem: red [NW][NT][32][8] then ssq [NW][32]
  __device__ static __forceinline__ void compute(const StepParams& p, const Info& ti, const float* x, int K, float* out, int N, int pos,
                                                 float* kc, float* vc, int bid, int tid, const uint4 (&wv)[NT][SPW], float* smem,
                                                 int bar_id) {
    float(*red)[NT][32][8] = reinterpret_cast<float(*)[NT][32][8]>(smem);
    float(*ssq)[32] = reinterpret_cast<float(*)[32]>(smem + NW * NT * 32 * 8);
    const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int steps_total = K >> 4;
    float acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
    float ss[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int s0 = 0; s0 < SPW; s0 += 4) {
      float4 xv[4][4];
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const int step = warp * SPW + s0 + s;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int row = r * 8 + g;
          xv[s][r] = (step < steps_total && row < p.B && ti.active)
                         ? __ldcg(reinterpret_cast<const float4*>(x + (size_t)row * K + step * 16 + 4 * t))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        uint32_t ah[4][2], al[4][2];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float4 v = xv[s][r];
          if (MODE != TK_RESID) ss[r] = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, ss[r]))));
          const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
          const float2 b0 = __half22float2(h0), b1 = __half22float2(h1);
          const __half2 l0 = __floats2half2_rn(v.x - b0.x, v.y - b0.y), l1 = __floats2half2_rn(v.z - b1.x, v.w - b1.y);
          ah[r][0] = *reinterpret_cast<const uint32_t*>(&h0); ah[r][1] = *reinterpret_cast<const uint32_t*>(&h1);
          al[r][0] = *reinterpret_cast<const uint32_t*>(&l0); al[r][1] = *reinterpret_cast<const uint32_t*>(&l1);
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const uint4 w = wv[nt][s0 + s];
            st_mma(acc[mt][nt], al[2 * mt][0], al[2 * mt + 1][0], al[2 * mt][1], al[2 * mt + 1][1], w.x, w.y);
            st_mma(acc[mt][nt], ah[2 * mt][0], ah[2 * mt + 1][0], ah[2 * mt][1], ah[2 * mt + 1][1], w.z, w.w);
            st_mma(acc[mt][nt], ah[2 * mt][0], ah[2 * mt + 1][0], ah[2 * mt][1], ah[2 * mt + 1][1], w.x, w.y);
          }
      }
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        *reinterpret_cast<float2*>(&red[warp][nt][mt * 16 + g][2 * t]) = make_float2(acc[mt][nt][0], acc[mt][nt][1]);
        *reinterpret_cast<float2*>(&red[warp][nt][mt * 16 + g + 8][2 * t]) = make_float2(acc[mt][nt][2], acc[mt][nt][3]);
      }
    if (MODE != TK_RESID) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        float q = ss[r];
        q += __shfl_xor_sync(0xffffffffu, q, 1);
        q += __shfl_xor_sync(0xffffffffu, q, 2);
        if (t == 0) ssq[warp][r * 8 + g] = q;
      }
    }
    worker_sync(bar_id, NW * 32);
    if (tid < 256) {
      const int b = tid >> 3, c = tid & 7;
      float v0 = 0.f, v1 = 0.f, q = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        v0 += red[w][0][b][c];
        if (NT > 1) v1 += red[w][NT - 1][b][c];
        if (MODE != TK_RESID) q += ssq[w][b];
      }
      if (MODE != TK_RESID) {
        const float rs = rsqrtf(q / K + p.eps);
        v0 *= rs;
        v1 *= rs;
      }
      if (MODE == TK_HEAD) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        if (ti.active && b < p.B) {
          bv = v0; bi = ti.row0 + c;
          if (v1 > bv) { bv = v1; bi = ti.row0 + 8 + c; }
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (c == 0) {
          p.part_val[(size_t)bid * 32 + b] = bv;
          p.part_idx[(size_t)bid * 32 + b] = bi;
        }
      } else if (b < p.B) {
        if (MODE == TK_RESID) {
          float* o = out + (size_t)b * N + ti.row0 + c;
          *o = __ldcg(o) + v0;
        } else if (MODE == TK_GATEUP) {
          out[(size_t)b * N + ti.row0 + c] = silu_f(v0) * v1;
        } else {  // TK_QKV
          const int dd = ti.dd0 + c, hh = ti.hh;
          if (ti.sec < 2) {
            const float c1 = p.rcos[pos * 64 + dd], s1 = p.rsin[pos * 64 + dd];
            const float c2 = p.rcos[pos * 64 + dd + 32], s2 = p.rsin[pos * 64 + dd + 32];
            const float y0 = v0 * c1 - v1 * s1, y1 = v1 * c2 + v0 * s2;
            if (ti.sec == 0) {
              out[(size_t)b * p.heads * 64 + hh * 64 + dd] = y0 * 0.125f;
              out[(size_t)b * p.heads * 64 + hh * 64 + dd + 32] = y1 * 0.125f;
            } else {
              const size_t o = (((size_t)b * p.heads + hh) * p.Lmax + pos) * 64 + dd;
              kc[o] = y0;
              kc[o + 32] = y1;
            }
          } else {
            const size_t o = (((size_t)b * p.heads + hh) * p.Lmax + pos) * 64 + dd;
            vc[o] = v0;
            vc[o + 32] = v1;
          }
        }
      }
    }
    worker_sync(bar_id, NW * 32);      // the worker's shared memory is reused by its next tile
  }
};


// ---------------------------------------------------------------------------------------------- flash-decoding attention
// item = (head h, batch row b): 16 half-warps walk keys hw, hw+16, ... with an online softmax (lm_decode_attn2_kernel body);
// smem: sacc [16][64], sm [16], sl [16]
__device__ __forceinline__ void attn_item(const float* __restrict__ q, const float* __restrict__ kc, const float* __restrict__ vc, int H,
                                          int Lmax, int n, float* __restrict__ out, int h, int b, int tid, float* smem, int bar_id) {
  float(*sacc)[64] = reinterpret_cast<float(*)[64]>(smem);
  float* sm = smem + 16 * 64;
  float* sl = sm + 16;
  const int lane = tid & 31, warp = tid >> 5;
  const int c = lane & 15, hw = warp * 2 + (lane >> 4);
  const float4 qv = __ldcg(reinterpret_cast<const float4*>(q + (size_t)b * H * 64 + h * 64 + 4 * c));
  const float4* kb = reinterpret_cast<const float4*>(kc + ((size_t)b * H + h) * Lmax * 64) + c;
  const float4* vb = reinterpret_cast<const float4*>(vc + ((size_t)b * H + h) * Lmax * 64) + c;
  float m = -INFINITY, l = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int base = warp * 2; base < n; base += 16 * LM_ATT_U) {
    const int j0 = base + (lane >> 4);
    float4 kv[LM_ATT_U], vv[LM_ATT_U];
    float s[LM_ATT_U];
#pragma unroll
    for (int u = 0; u < LM_ATT_U; ++u) {
      const int j = j0 + 16 * u;
      const bool ok = j < n;
      kv[u] = ok ? __ldcg(kb + (size_t)j * 16) : make_float4(0.f, 0.f, 0.f, 0.f);
      vv[u] = ok ? __ldcg(vb + (size_t)j * 16) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < LM_ATT_U; ++u) {
      float d = fmaf(qv.x, kv[u].x, fmaf(qv.y, kv[u].y, fmaf(qv.z, kv[u].z, qv.w * kv[u].w)));
      d += __shfl_xor_sync(0xffffffffu, d, 8);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      s[u] = (j0 + 16 * u < n) ? d : -INFINITY;
    }
    float mn = m;
#pragma unroll
    for (int u = 0; u < LM_ATT_U; ++u) mn = fmaxf(mn, s[u]);
    if (mn > -INFINITY) {
      const float corr = expf(m - mn);
      l *= corr;
      acc.x *= corr; acc.y *= corr; acc.z *= corr; acc.w *= corr;
#pragma unroll
      for (int u = 0; u < LM_ATT_U; ++u) {
        const float pr = expf(s[u] - mn);
        l += pr;
        acc.x = fmaf(pr, vv[u].x, acc.x); acc.y = fmaf(pr, vv[u].y, acc.y);
        acc.z = fmaf(pr, vv[u].z, acc.z); acc.w = fmaf(pr, vv[u].w, acc.w);
      }
      m = mn;
    }
  }
  *reinterpret_cast<float4*>(&sacc[hw][4 * c]) = acc;
  if (c == 0) { sm[hw] = m; sl[hw] = l; }
  worker_sync(bar_id, 256);
  if (tid < 64) {
    float M = sm[0];
#pragma unroll
    for (int i = 1; i < 16; ++i) M = fmaxf(M, sm[i]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float e = expf(sm[i] - M);
      num = fmaf(e, sacc[i][tid], num);
      den = fmaf(e, sl[i], den);
    }
    out[(size_t)b * H * 64 + h * 64 + tid] = num / den;
  }
  worker_sync(bar_id, 256);
}

// ---------------------------------------------------------------------------------------------- greedy token of one batch row
// (lm_argmax_embed_kernel body for a 256-thread worker): partials [n_part][32] -> token, out_ids, next input embedding
__device__ __forceinline__ void argmax_item(const StepParams& p, int n_part, int b, int slot, int tid, float* smem, int bar_id) {
  float* sv = smem;
  int* si = reinterpret_cast<int*>(smem + 32);
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = tid; i < n_part; i += 256) {
    const float v = __ldcg(p.part_val + (size_t)i * 32 + b);
    const int ix = __ldcg(p.part_idx + (size_t)i * 32 + b);
    if (v > bv || (v == bv && ix < bi)) { bv = v; bi = ix; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if ((tid & 31) == 0) { sv[tid >> 5] = bv; si[tid >> 5] = bi; }
  worker_sync(bar_id, 256);
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (sv[w] > bv || (sv[w] == bv && si[w] < bi)) { bv = sv[w]; bi = si[w]; }
    if (bi == 0x7fffffff || bi < 0) bi = p.range[0];          // all-NaN row: first column of the range
    si[0] = bi;
    p.out_ids[(size_t)b * p.out_stride + slot] = (int64_t)bi;
  }
  worker_sync(bar_id, 256);
  const int tok = si[0];
  for (int k = tid; k < p.hidden; k += 256) p.x[(size_t)b * p.hidden + k] = p.emb[(size_t)tok * p.hidden + k];
  worker_sync(bar_id, 256);
}

// ---------------------------------------------------------------------------------------------- the persistent kernel
__global__ void __launch_bounds__(ST_THREADS, 1) lm_decode_steps_kernel(const StepParams p) {
  __shared__ __align__(16) float smem_all[2 * ST_WSMEM];
  const int tid = threadIdx.x, wk = tid >> 8, wt = tid & 255;
  const int w = blockIdx.x * 2 + wk, NWK = gridDim.x * 2;                 // 256-thread workers
  float* wsm = smem_all + wk * ST_WSMEM;
  const int wbar = 1 + wk;
  unsigned epoch = 0;
  const unsigned n_ctas = gridDim.x;
  const int pos0 = *p.pos, slot0 = *p.slot;
  const int H = p.hidden, I = p.inter, heads = p.heads;
  const int n_qkv = 3 * heads * 4, n_att = heads * p.B, n_o = H / 8, n_gu = I / 8;
  using QKV = SkTile<TK_QKV, 4, 8>;
  using OPJ = SkTile<TK_RESID, 4, 8>;
  using GUP = SkTile<TK_GATEUP, 4, 8>;
  using DWN = SkTile<TK_RESID, 8, 16>;
  using HED = SkTile<TK_HEAD, 4, 8>;

  for (int s = 0; s < p.n_steps; ++s) {
    const int pos = pos0 + s, slot = slot0 + s;
    for (int li = 0; li < p.layers; ++li) {
      const StepLayer& L = p.L[li];
      {  // ---- RMSNorm + QKV + RoPE + cache append
        QKV::Info ti;
        uint4 wv[2][4];
        int item = w;
        if (item < n_qkv) { QKV::locate(p, L.wqkv, nullptr, H, item, wt, ti); QKV::load_w(ti, H, wt, wv); }
        grid_barrier(p.bar, epoch, n_ctas, p.dbg);
        for (; item < n_qkv; item += NWK) {
          if (item != w) { QKV::locate(p, L.wqkv, nullptr, H, item, wt, ti); QKV::load_w(ti, H, wt, wv); }
          if (!(p.dbg & 2)) QKV::compute(p, ti, p.x, H, p.q_buf, 0, pos, L.kc, L.vc, item, wt, wv, wsm, wbar);
        }
      }
      {  // ---- attention over the cache (keys 0..pos)
        grid_barrier(p.bar, epoch, n_ctas, p.dbg);
        for (int item = w; item < n_att; item += NWK)
          if (!(p.dbg & 2)) attn_item(p.q_buf, L.kc, L.vc, heads, p.Lmax, pos + 1, p.attn_buf, item % heads, item / heads, wt, wsm, wbar);
      }
      {  // ---- o_proj + residual
        OPJ::Info ti;
        uint4 wv[1][4];
        int item = w;
        if (item < n_o) { OPJ::locate(p, L.wo, nullptr, H, item, wt, ti); OPJ::load_w(ti, H, wt, wv); }
        grid_barrier(p.bar, epoch, n_ctas, p.dbg);
        for (; item < n_o; item += NWK) {
          if (item != w) { OPJ::locate(p, L.wo, nullptr, H, item, wt, ti); OPJ::load_w(ti, H, wt, wv); }
          if (!(p.dbg & 2)) OPJ::compute(p, ti, p.attn_buf, H, p.x, H, pos, nullptr, nullptr, item, wt, wv, wsm, wbar);
        }
      }
      {  // ---- RMSNorm + gate / up + SwiGLU
        GUP::Info ti;
        uint4 wv[2][4];
        int item = w;
        if (item < n_gu) { GUP::locate(p, L.wg, L.wu, H, item, wt, ti); GUP::load_w(ti, H, wt, wv); }
        grid_barrier(p.bar, epoch, n_ctas, p.dbg);
        for (; item < n_gu; item += NWK) {
          if (item != w) { GUP::locate(p, L.wg, L.wu, H, item, wt, ti); GUP::load_w(ti, H, wt, wv); }
          if (!(p.dbg & 2)) GUP::compute(p, ti, p.x, H, p.mlp_buf, I, pos, nullptr, nullptr, item, wt, wv, wsm, wbar);
        }
      }
      {  // ---- down + residual: K = inter, the whole CTA (16 warps) per tile
        DWN::Info ti;
        uint4 wv[1][8];
        int item = blockIdx.x;
        if (item < n_o) { DWN::locate(p, L.wd, nullptr, I, item, tid, ti); DWN::load_w(ti, I, tid, wv); }
        grid_barrier(p.bar, epoch, n_ctas, p.dbg);
        for (; item < n_o; item += (int)gridDim.x) {
          if (item != (int)blockIdx.x) { DWN::locate(p, L.wd, nullptr, I, item, tid, ti); DWN::load_w(ti, I, tid, wv); }
          if (!(p.dbg & 2)) DWN::compute(p, ti, p.mlp_buf, I, p.x, H, pos, nullptr, nullptr, item, tid, wv, smem_all, 0);
        }
      }
    }
    {  // ---- final RMSNorm (folded) + head restricted to the token range -> arg-max partials per 16 columns
      const int n_head = (p.range[1] - p.range[0]) / 16;
      HED::Info ti;
      uint4 wv[2][4];
      int item = w;
      if (item < n_head) { HED::locate(p, p.whead, nullptr, H, item, wt, ti); HED::load_w(ti, H, wt, wv); }
      grid_barrier(p.bar, epoch, n_ctas, p.dbg);
      for (; item < n_head; item += NWK) {
        if (item != w) { HED::locate(p, p.whead, nullptr, H, item, wt, ti); HED::load_w(ti, H, wt, wv); }
        if (!(p.dbg & 2)) HED::compute(p, ti, p.x, H, nullptr, 0, pos, nullptr, nullptr, item, wt, wv, wsm, wbar);
      }
      grid_barrier(p.bar, epoch, n_ctas, p.dbg);
      for (int b = w; b < p.B; b += NWK) if (!(p.dbg & 2)) argmax_item(p, n_head, b, slot, wt, wsm, wbar);
    }
  }
  grid_barrier(p.bar, epoch, n_ctas, p.dbg);
  if (blockIdx.x == 0 && tid == 0) { *p.pos = pos0 + p.n_steps; *p.slot = slot0 + p.n_steps; }
}

}  // namespace qb
using namespace qb;

// n_steps cached greedy steps in ONE cooperative launch.  Pointers as for qb_lm_decode_layer_tc / qb_lm_head_argmax_tc, per layer
// arrays of `layers` device pointers given on the HOST.  x [B, hidden] holds the embedding of the first input token on entry and
// of the last produced token on exit; *pos / *slot (device ints) advance by n_steps; out_ids[b*out_stride + slot..] receive the
// tokens.  barrier: device uint32 (zeroed by this call).  Replaces llm_sft.py:137-164 / 166-193 for do_sample=False.
extern "C" int qb_lm_decode_steps(float* x, int64_t B, int32_t hidden, int32_t heads, int32_t inter, int32_t layers,
                                  const qb_half* const* wqkv, const qb_half* const* wo, const qb_half* const* wgate,
                                  const qb_half* const* wup, const qb_half* const* wdown, float* const* k_cache, float* const* v_cache,
                                  int32_t Lmax, const qb_half* w_head, const int32_t* range, int32_t max_cols, const float* embedding,
                                  const float* rope_cos, const float* rope_sin, float* q_buf, float* attn_buf, float* mlp_buf,
                                  float* part_val, int32_t* part_idx, int64_t* out_ids, int32_t out_stride, int32_t* pos, int32_t* slot,
                                  int32_t n_steps, uint32_t* barrier, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(x && wqkv && wo && wgate && wup && wdown && k_cache && v_cache && w_head && range && embedding && rope_cos && rope_sin &&
                 q_buf && attn_buf && mlp_buf && part_val && part_idx && out_ids && pos && slot && barrier, "lm_decode_steps: null argument");
  QB_REQUIRE(B >= 1 && B <= 32 && layers >= 1 && layers <= ST_MAX_LAYERS && n_steps >= 1, "lm_decode_steps: 1 <= B <= 32, 1 <= layers <= %d", ST_MAX_LAYERS);
  QB_REQUIRE(hidden == heads * 64 && hidden == 512 && inter == 2048 && max_cols % 16 == 0,
             "lm_decode_steps: the persistent kernel is built for the shipped LM (hidden 512 = 8 x 64, FFN 2048)");
  StepParams p = {};
  p.B = (int)B; p.hidden = hidden; p.heads = heads; p.inter = inter; p.layers = layers; p.Lmax = Lmax; p.n_steps = n_steps;
  p.out_stride = out_stride;
  for (int i = 0; i < layers; ++i) {
    p.L[i].wqkv = (const uint4*)wqkv[i]; p.L[i].wo = (const uint4*)wo[i]; p.L[i].wg = (const uint4*)wgate[i];
    p.L[i].wu = (const uint4*)wup[i]; p.L[i].wd = (const uint4*)wdown[i]; p.L[i].kc = k_cache[i]; p.L[i].vc = v_cache[i];
  }
  p.whead = (const uint4*)w_head; p.x = x; p.q_buf = q_buf; p.attn_buf = attn_buf; p.mlp_buf = mlp_buf;
  p.rcos = rope_cos; p.rsin = rope_sin; p.emb = embedding; p.pos = pos; p.slot = slot; p.range = range;
  p.part_val = part_val; p.part_idx = part_idx; p.out_ids = out_ids; p.bar = barrier; p.eps = 1e-6f;
  int dev = 0, sms = 0, per_sm = 0;
  QB_CHECK_CUDA(cudaGetDevice(&dev));
  QB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  QB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lm_decode_steps_kernel, ST_THREADS, 0));
  QB_REQUIRE(per_sm >= 1, "lm_decode_steps: kernel does not fit on an SM");
  if (const char* e = getenv("QB_LM_STEP_DBG")) p.dbg = atoi(e);
  int grid = sms;
  if (const char* e = getenv("QB_LM_STEP_CTAS")) grid = atoi(e) > 0 && atoi(e) < sms ? atoi(e) : sms;
  QB_CHECK_CUDA(cudaMemsetAsync(barrier, 0, sizeof(uint32_t), st));
  void* args[] = {&p};
  QB_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)lm_decode_steps_kernel, dim3((unsigned)grid), dim3(ST_THREADS), args, 0, st));
  g_launches++;
  return 0;
}
