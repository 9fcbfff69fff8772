// UniSE AR-LM kernels (reference: QuarkAudio-UniSE/model/llm/llm.py:150-228, llm_sft.py:93-195; HF Llama
// decoder layers: RMSNorm(1e-6) -> q/k/v (no bias) -> RoPE -> causal attention -> o_proj -> +res ->
// RMSNorm -> SwiGLU MLP -> +res).
//
// Prefill / teacher-forced forward (L > 1) runs on the wgmma GEMM (gemm.cu) plus the two kernels here:
//   lm_qkv_prep   RoPE at absolute positions, 1/sqrt(d) folded into q, K/V appended to the static fp32 cache
//   lm_flash_attn causal flash attention (mma.sync m16n8k16, 3-term fp16 split of Q/K/P/V) over the cache
// KV-cache decode (L == 1, B <= 32) is HBM-bound (weights + cache streamed once per step), each stage launched as a
// programmatic dependent of the previous one:
//   lm_skinny<MODE>   fused RMSNorm -> projection -> {RoPE + cache append | residual | SwiGLU | arg-max partials},
//                     3-term fp16-split mma.sync over pre-packed weights
//   lm_decode_attn2   one CTA per (head, batch row), online softmax over the fp32 cache
//   lm_argmax_embed   range-restricted greedy token + next input embedding + position bump
//   lm_sample_embed   top-k / top-p / temperature draw instead of the arg-max (sampled decoding)
// All decode state (position, token range, output slot) lives in device memory so that one decode step is a
// fixed launch sequence that can be captured in a CUDA graph and replayed.
#include <atomic>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

// ------------------------------------------------------------------------------------------ prefill
__global__ void lm_qkv_prep_kernel(const float* __restrict__ qkv, int L, int H, int pos0, const float* __restrict__ rcos,
                                   const float* __restrict__ rsin, float* __restrict__ q32, float* __restrict__ kc,
                                   float* __restrict__ vc, int Lmax, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int d = (int)(i & 31);
  long long r = i >> 5;
  const int h = (int)(r % H);
  r /= H;
  const int t = (int)(r % L);
  const long long b = r / L;
  const int pos = pos0 + t;
  const float* base = qkv + (b * L + t) * 3LL * H * 64 + h * 64;
  const float c1 = rcos[pos * 64 + d], s1 = rsin[pos * 64 + d], c2 = rcos[pos * 64 + d + 32], s2 = rsin[pos * 64 + d + 32];
  const long long oq = ((b * H + h) * L + t) * 64 + d;
  const long long oc = ((b * H + h) * (long long)Lmax + pos) * 64 + d;
  {
    const float x1 = base[d], x2 = base[d + 32];
    q32[oq] = (x1 * c1 - x2 * s1) * 0.125f;
    q32[oq + 32] = (x2 * c2 + x1 * s2) * 0.125f;
  }
  {
    const float x1 = base[H * 64 + d], x2 = base[H * 64 + d + 32];
    kc[oc] = x1 * c1 - x2 * s1;
    kc[oc + 32] = x2 * c2 + x1 * s2;
  }
  vc[oc] = base[2 * H * 64 + d];
  vc[oc + 32] = base[2 * H * 64 + d + 32];
}

constexpr int LF_BQ = 64, LF_BK = 64, LF_D = 64, LF_P = 72;

__device__ __forceinline__ void l_ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void l_ldsm_x4_t(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void l_mma(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t l_pack(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// q32 [B,H,L,64] (RoPE'd, pre-scaled); fp32 cache kc/vc [B,H,Lmax,64]; query t sits at absolute position
// pos0 + t and sees keys <= it.  Operands are split into fp16 hi/lo planes while being staged into shared
// memory and both products run as 3-term split MMAs (hi*hi + lo*hi + hi*lo): ~2^-21 relative, which the
// 1e-3 logit tolerance needs once attention scores are O(10) (single-pass fp16 gives ~|s| * 2^-11).
__device__ __forceinline__ void stage_split8(const float* __restrict__ src, bool ok, __half* dst_hi, __half* dst_lo) {
  float v[8];
  if (ok) {
    const float4 a = *reinterpret_cast<const float4*>(src), c = *reinterpret_cast<const float4*>(src + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
  }
  __half2 h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    const float2 bk = __half22float2(h[i]);
    l[i] = __floats2half2_rn(v[2 * i] - bk.x, v[2 * i + 1] - bk.y);
  }
  *reinterpret_cast<uint4*>(dst_hi) = *reinterpret_cast<uint4*>(h);
  *reinterpret_cast<uint4*>(dst_lo) = *reinterpret_cast<uint4*>(l);
}

__global__ void __launch_bounds__(128)
lm_flash_attn_kernel(const float* __restrict__ q32, const float* __restrict__ kc, const float* __restrict__ vc, int L,
                     int H, int pos0, int Lmax, __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  extern __shared__ __align__(16) __half lsm[];
  __half* sqh = lsm;
  __half* sql = sqh + LF_BQ * LF_P;
  __half* skh = sql + LF_BQ * LF_P;
  __half* skl = skh + LF_BK * LF_P;
  __half* svh = skl + LF_BK * LF_P;
  __half* svl = svh + LF_BK * LF_P;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.x * LF_BQ, h = blockIdx.y, b = blockIdx.z;
  const long long qhead = ((long long)b * H + h) * L * LF_D;
  const long long chead = ((long long)b * H + h) * (long long)Lmax * LF_D;
  for (int c = tid; c < LF_BQ * 8; c += 128) {
    const int r = c >> 3, ch = c & 7;
    stage_split8(q32 + qhead + (long long)(q0 + r) * LF_D + ch * 8, q0 + r < L, sqh + r * LF_P + ch * 8, sql + r * LF_P + ch * 8);
  }
  __syncthreads();
  uint32_t qh[4][4], ql[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const int off = (warp * 16 + (lane & 15)) * LF_P + ks * 16 + (lane >> 4) * 8;
    l_ldsm_x4(qh[ks][0], qh[ks][1], qh[ks][2], qh[ks][3], sqh + off);
    l_ldsm_x4(ql[ks][0], ql[ks][1], ql[ks][2], ql[ks][3], sql + off);
  }
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[j][e] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const float LOG2E = 1.4426950408889634f;
  const int qa = q0 + warp * 16 + (lane >> 2), qb = qa + 8;     // this thread's two query rows
  const int kv_end = min(pos0 + L, pos0 + q0 + LF_BQ);           // causal: no key beyond the tile's last query
  for (int k0 = 0; k0 < kv_end; k0 += LF_BK) {
    __syncthreads();
    for (int c = tid; c < LF_BK * 8; c += 128) {
      const int r = c >> 3, ch = c & 7;
      const bool ok = k0 + r < kv_end;
      const long long g = chead + (long long)(k0 + r) * LF_D + ch * 8;
      stage_split8(kc + g, ok, skh + r * LF_P + ch * 8, skl + r * LF_P + ch * 8);
      stage_split8(vc + g, ok, svh + r * LF_P + ch * 8, svl + r * LF_P + ch * 8);
    }
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[j][e] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {
        const int off = (j * 8 + (lane & 7)) * LF_P + kp * 32 + (lane >> 3) * 8;
        uint32_t b0, b1, b2, b3, c0, c1, c2, c3;
        l_ldsm_x4(b0, b1, b2, b3, skh + off);
        l_ldsm_x4(c0, c1, c2, c3, skl + off);
        l_mma(s[j], qh[2 * kp][0], qh[2 * kp][1], qh[2 * kp][2], qh[2 * kp][3], b0, b1);
        l_mma(s[j], ql[2 * kp][0], ql[2 * kp][1], ql[2 * kp][2], ql[2 * kp][3], b0, b1);
        l_mma(s[j], qh[2 * kp][0], qh[2 * kp][1], qh[2 * kp][2], qh[2 * kp][3], c0, c1);
        l_mma(s[j], qh[2 * kp + 1][0], qh[2 * kp + 1][1], qh[2 * kp + 1][2], qh[2 * kp + 1][3], b2, b3);
        l_mma(s[j], ql[2 * kp + 1][0], ql[2 * kp + 1][1], ql[2 * kp + 1][2], ql[2 * kp + 1][3], b2, b3);
        l_mma(s[j], qh[2 * kp + 1][0], qh[2 * kp + 1][1], qh[2 * kp + 1][2], qh[2 * kp + 1][3], c2, c3);
      }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int key = k0 + j * 8 + (lane & 3) * 2;
      if (key > pos0 + qa) s[j][0] = -INFINITY;
      if (key + 1 > pos0 + qa) s[j][1] = -INFINITY;
      if (key > pos0 + qb) s[j][2] = -INFINITY;
      if (key + 1 > pos0 + qb) s[j][3] = -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    // rows beyond L (tail tile) may see no valid key: keep them finite
    const float e0 = (mn0 == -INFINITY) ? 0.f : mn0, e1 = (mn1 == -INFINITY) ? 0.f : mn1;
    const float c0 = exp2f((m0 - e0) * LOG2E), c1 = exp2f((m1 - e1) * LOG2E);
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = exp2f((s[j][0] - e0) * LOG2E);
      s[j][1] = exp2f((s[j][1] - e0) * LOG2E);
      s[j][2] = exp2f((s[j][2] - e1) * LOG2E);
      s[j][3] = exp2f((s[j][3] - e1) * LOG2E);
      rs0 += s[j][0] + s[j][1];
      rs1 += s[j][2] + s[j][3];
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
    m0 = mn0;
    m1 = mn1;
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] *= c0; o[j][1] *= c0; o[j][2] *= c1; o[j][3] *= c1; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t ah[4], al[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // e: (tile 2ks | 2ks+1) x (cols 0,1 | 2,3) in A-fragment order
        const int jj = 2 * ks + (e >> 1), cc = (e & 1) * 2;
        const __half2 hh = __floats2half2_rn(s[jj][cc], s[jj][cc + 1]);
        const float2 bk = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(s[jj][cc] - bk.x, s[jj][cc + 1] - bk.y);
        ah[e] = *reinterpret_cast<const uint32_t*>(&hh);
        al[e] = *reinterpret_cast<const uint32_t*>(&ll);
      }
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        const int off = (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LF_P + jp * 16 + (lane >> 4) * 8;
        uint32_t b0, b1, b2, b3, d0, d1, d2, d3;
        l_ldsm_x4_t(b0, b1, b2, b3, svh + off);
        l_ldsm_x4_t(d0, d1, d2, d3, svl + off);
        l_mma(o[2 * jp], ah[0], ah[1], ah[2], ah[3], b0, b1);
        l_mma(o[2 * jp], al[0], al[1], al[2], al[3], b0, b1);
        l_mma(o[2 * jp], ah[0], ah[1], ah[2], ah[3], d0, d1);
        l_mma(o[2 * jp + 1], ah[0], ah[1], ah[2], ah[3], b2, b3);
        l_mma(o[2 * jp + 1], al[0], al[1], al[2], al[3], b2, b3);
        l_mma(o[2 * jp + 1], ah[0], ah[1], ah[2], ah[3], d2, d3);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = j * 8 + (lane & 3) * 2;
    if (qa < L) {
      const long long off = ((long long)b * L + qa) * (long long)(H * LF_D) + h * LF_D + d;
      __half ha, hb, la, lb;
      split_f16(o[j][0] * i0, ha, la);
      split_f16(o[j][1] * i0, hb, lb);
      *reinterpret_cast<__half2*>(out_hi + off) = __halves2half2(ha, hb);
      if (out_lo) *reinterpret_cast<__half2*>(out_lo + off) = __halves2half2(la, lb);
    }
    if (qb < L) {
      const long long off = ((long long)b * L + qb) * (long long)(H * LF_D) + h * LF_D + d;
      __half ha, hb, la, lb;
      split_f16(o[j][2] * i1, ha, la);
      split_f16(o[j][3] * i1, hb, lb);
      *reinterpret_cast<__half2*>(out_hi + off) = __halves2half2(ha, hb);
      if (out_lo) *reinterpret_cast<__half2*>(out_lo + off) = __halves2half2(la, lb);
    }
  }
}

// ------------------------------------------------------------------------------------------ decode step
// Positions of the decode step: row b reads pos[b] (rows whose prefixes differ in length sit at different positions).  The head's
// block of row b bumps pos[b] after its dependency wait: every kernel of the step that reads positions has finished by then, and
// the next step reads them after its own wait.

// greedy token from the head partials, next input embedding, position / slot bump
__global__ void lm_argmax_embed_kernel(const float* __restrict__ part_val, const int* __restrict__ part_idx, int n_part,
                                       int B, const float* __restrict__ emb, int Hd, float* __restrict__ x_next,
                                       int64_t* __restrict__ out_ids, int out_stride, int* __restrict__ pos,
                                       int* __restrict__ slot, const int* __restrict__ range, int vocab) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");          // no-ops unless launched as a programmatic dependent
  const int b = blockIdx.x;
  const int range_lo = range[0];
  __shared__ float sv[32];
  __shared__ int si[32];
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n_part; i += blockDim.x) {
    const float v = part_val[(size_t)i * 32 + b];
    const int ix = part_idx[(size_t)i * 32 + b];
    if (v > bv || (v == bv && ix < bi)) { bv = v; bi = ix; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (sv[w] > bv || (sv[w] == bv && si[w] < bi)) { bv = sv[w]; bi = si[w]; }
    // an all-NaN logit row never wins a comparison (bi stays at its sentinel): fall back to the first column of the
    // range like torch.argmax returning a valid index, instead of gathering emb[0x7fffffff]
    if ((unsigned)bi >= (unsigned)vocab) bi = range_lo;
    si[0] = bi;
    out_ids[(size_t)b * out_stride + *slot] = (int64_t)bi;
    pos[b] += 1;
  }
  __syncthreads();
  const int tok = si[0];
  for (int k = threadIdx.x; k < Hd; k += blockDim.x) x_next[(size_t)b * Hd + k] = emb[(size_t)tok * Hd + k];
  // every block has read *slot before any block can finish? no: use a grid-wide last-block bump instead
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int done = atomicAdd(slot + 1, 1);          // slot[1] = arrival counter
    if (done == B - 1) { slot[1] = 0; *slot += 1; }
  }
}


// ------------------------------------------------------------------------------------------ teacher-forced loss + accuracy
// CustomLlamaModel.loss_function (QuarkAudio-UniSE/model/llm/llm.py:87-104): label-smoothed KL (batchmean) between
// log_softmax(logits) and the smoothed one-hot target, plus arg-max accuracy.  One pass over the logits: per row the
// log-sum-exp, the target logit, the plain sum and the arg-max; with t = 1 - ls on the target and u = ls / (V - 1) elsewhere
//   KL_row = t log t + ls log u - t logp_target - u (sum_c logit_c - logit_target - (V - 1) lse)
// A second single-block kernel sums the rows in a fixed order (deterministic).
__global__ void __launch_bounds__(256)
lm_loss_rows_kernel(const float* __restrict__ logits, long long ld, int V, const int64_t* __restrict__ targets, float ls,
                    float* __restrict__ row_loss, int* __restrict__ row_hit) {
  const long long row = blockIdx.x;
  const float* x = logits + row * ld;
  float m = -INFINITY, sum = 0.f;
  int am = 0;
  for (int c = threadIdx.x; c < V; c += 256) {
    const float v = x[c];
    sum += v;
    if (v > m) { m = v; am = c; }
  }
  __shared__ float sm[256], ss[256];
  __shared__ int si[256];
  sm[threadIdx.x] = m; ss[threadIdx.x] = sum; si[threadIdx.x] = am;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const float mo = sm[threadIdx.x + o];
      const int io = si[threadIdx.x + o];
      if (mo > sm[threadIdx.x] || (mo == sm[threadIdx.x] && io < si[threadIdx.x])) { sm[threadIdx.x] = mo; si[threadIdx.x] = io; }
      ss[threadIdx.x] += ss[threadIdx.x + o];
    }
    __syncthreads();
  }
  const float M = sm[0];
  float e = 0.f;
  for (int c = threadIdx.x; c < V; c += 256) e += expf(x[c] - M);
  __shared__ float se[256];
  se[threadIdx.x] = e;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) se[threadIdx.x] += se[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float lse = M + logf(se[0]);
    const int tg = (int)targets[row];
    const float lt = x[tg];
    const float t = 1.f - ls, u = ls / (float)(V - 1);
    const float ent = (t > 0.f ? t * logf(t) : 0.f) + (ls > 0.f ? ls * logf(u) : 0.f);
    row_loss[row] = ent - t * (lt - lse) - u * ((ss[0] - lt) - (float)(V - 1) * lse);
    row_hit[row] = si[0] == tg;
  }
}
__global__ void lm_loss_reduce_kernel(const float* __restrict__ row_loss, const int* __restrict__ row_hit, long long M,
                                      float* __restrict__ out) {
  __shared__ double sl[256];
  __shared__ long long sh[256];
  double l = 0.0;
  long long h = 0;
  for (long long i = threadIdx.x; i < M; i += 256) { l += row_loss[i]; h += row_hit[i]; }
  sl[threadIdx.x] = l; sh[threadIdx.x] = h;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { sl[threadIdx.x] += sl[threadIdx.x + o]; sh[threadIdx.x] += sh[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[0] = (float)(sl[0] / (double)M); out[1] = (float)((double)sh[0] / (double)M); }
}

// ------------------------------------------------------------------------------------------ sampled decoding
// CustomLlamaModel.sample_logits (QuarkAudio-UniSE/model/llm/llm.py:253-289) for one row per CTA, on the range-restricted
// logits the head kernel wrote: top-k (threshold = k-th largest value, ties kept: `logits < topk[-1]` is what is removed)
// -> top-p over softmax of the SURVIVORS sorted descending (a token is removed when the cumulative probability of the
// tokens BEFORE it already exceeds top_p; the first one always stays) -> / temperature -> softmax -> one multinomial
// draw.  torch.multinomial's generator cannot be reproduced bit for bit, so the draw is defined here as the inverse CDF
// over the kept tokens in descending-logit order (ties: ascending id) at u = Philox4x32-10(key = seed, counter =
// {step, row, call, 0}).x * 2^-32 truncated to 24 bits: same distribution, replayable from (seed, call, step, row).
// With per-row keys (row_keys != NULL) row b's uniform is Philox4x32-10(key = row_keys[b], counter = {step, 0, 0, 0}): a
// function of its key and the step only, so a row draws the same tokens wherever it sits in whichever batch.
// Two kernels: lm_sample_embed for 1 <= top_k <= LS_MAX (the survivors above the k-th value fit LS_MAX slots, one thread
// walks them), lm_sample_full_embed for top_k = 0 (no filter) or above LS_MAX, up to the whole range: every survivor is
// stored and sorted, and the top-p cut, the normaliser and the inverse-CDF search are fixed-order block-wide scans.
constexpr int LS_MAX = 1024;             // survivors above the threshold kept (< top_k) by lm_sample_embed_kernel
__device__ __forceinline__ uint32_t ls_key(float v) {     // monotone float -> uint32 (NaN sorts lowest)
  if (v != v) return 0u;
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ls_val(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ uint32_t philox_u32(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}
__device__ __forceinline__ float ls_uniform(const unsigned* seed, const unsigned* row_keys, int step, int b) {
  const uint32_t r = row_keys ? philox_u32(row_keys[2 * b], row_keys[2 * b + 1], (uint32_t)step, 0u, 0u, 0u)
                              : philox_u32(seed[0], seed[1], (uint32_t)step, (uint32_t)b, seed[2], 0u);
  return (float)(r >> 8) * (1.0f / 16777216.0f);
}

// The need-th largest of keys[0..n) (1 <= need <= n) by radix select, one byte per pass from the top, with NT threads; the
// caller has stored keys and synchronised.  Returns the key; n_gt = the keys strictly above it, n_eq = the keys equal to it.
template <int NT>
__device__ __forceinline__ uint32_t ls_radix_select(const uint32_t* keys, int n, int need, int* hist, int& n_gt, int& n_eq) {
  __shared__ uint32_t s_prefix;
  __shared__ int s_need, s_eq;
  const int tid = threadIdx.x;
  if (tid == 0) { s_prefix = 0u; s_need = need; }
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += NT) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix, himask = shift == 24 ? 0u : (0xFFFFFFFFu << (shift + 8));
    for (int i = tid; i < n; i += NT) {
      const uint32_t k = keys[i];
      if ((k & himask) == prefix) atomicAdd(&hist[(k >> shift) & 255], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int nd = s_need, bin = 255;
      for (; bin > 0; --bin) {
        if (hist[bin] >= nd) break;
        nd -= hist[bin];
      }
      s_need = nd;
      s_prefix = prefix | ((uint32_t)bin << shift);
      if (shift == 0) s_eq = hist[bin];          // keys equal to the threshold
    }
    __syncthreads();
  }
  n_gt = need - s_need;
  n_eq = s_eq;
  return s_prefix;
}

__global__ void __launch_bounds__(256)
lm_sample_embed_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ range, int B, float inv_temp,
                       int top_k, float top_p, const unsigned* __restrict__ seed /* {seed_lo, seed_hi, call, 0} */,
                       const unsigned* __restrict__ row_keys /* [B][2] or NULL */, const float* __restrict__ emb, int Hd,
                       float* __restrict__ x_next, int64_t* __restrict__ out_ids, int out_stride, int* __restrict__ pos,
                       int* __restrict__ slot, float* __restrict__ dbg) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  extern __shared__ uint32_t ls_smem[];
  const int lo = range[0], n = range[1] - lo, b = blockIdx.x, tid = threadIdx.x;
  uint32_t* keys = ls_smem;                       // [n]
  uint32_t* skey = keys + ((n + 3) & ~3);         // [LS_MAX] survivors: key
  int* sidx = (int*)(skey + LS_MAX);              // [LS_MAX] survivors: column
  __shared__ int hist[256];
  __shared__ int sh_cnt, sh_tok, sh_rank;
  for (int i = tid; i < n; i += 256) keys[i] = ls_key(logits[(size_t)b * ld + i]);
  if (tid == 0) sh_cnt = 0;
  __syncthreads();
  // ---- radix select of the top_k-th largest key
  int n_gt, n_eq;
  const uint32_t thr = ls_radix_select<256>(keys, n, top_k < n ? top_k : n, hist, n_gt, n_eq);
  // ---- survivors: every key >= threshold (ties at the k-th value stay, llm.py:263-264).  Those strictly above it (at most
  // top_k - 1) are collected and bitonic-sorted descending; the n_eq tied ones, however many, share one value and follow them
  // in ascending column order, so they are counted rather than stored.
  for (int i = tid; i < n; i += 256) {
    const uint32_t k = keys[i];
    if (k > thr) {
      const int s = atomicAdd(&sh_cnt, 1);
      skey[s] = k; sidx[s] = i;
    }
  }
  __syncthreads();
  const int cnt = n_gt;
  int P = 1;
  while (P < cnt) P <<= 1;
  for (int i = cnt + tid; i < P; i += 256) { skey[i] = 0u; sidx[i] = 0x7fffffff; }
  __syncthreads();
  for (int k2 = 2; k2 <= P; k2 <<= 1)
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += 256) {
        const int l = i ^ j;
        if (l > i) {
          const uint32_t ka = skey[i], kb = skey[l];
          const int ia = sidx[i], ib = sidx[l];
          const bool a_first = ka > kb || (ka == kb && ia < ib);       // descending by key, ascending by column on ties
          const bool up = (i & k2) == 0;
          if (up != a_first) { skey[i] = kb; skey[l] = ka; sidx[i] = ib; sidx[l] = ia; }
        }
      }
      __syncthreads();
    }
  // ---- top-p cut, temperature, inverse-CDF draw over the survivors in order: the cnt sorted ones one by one (sequential fp32 adds,
  // like torch.cumsum on a row), then the tied tail in closed form (j tied tokens add j * their common term)
  if (tid == 0) {
    const float v = ls_val(thr), m = cnt > 0 ? ls_val(skey[0]) : v;
    const int n_all = cnt + n_eq;
    int nk = n_all;
    if (top_p < 1.0f) {
      const float q = expf(v - m);
      float Z = 0.f;
      for (int i = 0; i < cnt; ++i) Z += expf(ls_val(skey[i]) - m);
      Z += (float)n_eq * q;
      float cum = 0.f;
      nk = 0;
      for (int i = 1; i <= cnt; ++i) {               // a token goes once the mass before it exceeds top_p
        cum += expf(ls_val(skey[i - 1]) - m) / Z;
        if (cum > top_p) { nk = i; break; }
      }
      if (nk == 0) {                                 // the cut falls in the tied tail: keep the first j of it, j >= 1
        const float qz = q / Z;
        int j = qz > 0.f ? (int)fminf(fmaxf(floorf((top_p - cum) / qz), 0.f), (float)n_eq) : n_eq;
        while (j > 1 && cum + (float)(j - 1) * qz > top_p) --j;
        while (j < n_eq && !(cum + (float)j * qz > top_p)) ++j;
        nk = cnt + (j > 1 ? j : 1);
      }
    }
    const int k_gt = nk < cnt ? nk : cnt, k_eq = nk - k_gt;
    const float et = expf((v - m) * inv_temp);
    float S = 0.f;
    for (int i = 0; i < k_gt; ++i) S += expf((ls_val(skey[i]) - m) * inv_temp);
    S += (float)k_eq * et;
    const float u = ls_uniform(seed, row_keys, *slot, b);
    const float target = u * S;
    float run = 0.f;
    int pick = -1;
    for (int i = 0; i < k_gt; ++i) {
      run += expf((ls_val(skey[i]) - m) * inv_temp);
      if (run > target) { pick = i; break; }
    }
    sh_rank = -1;
    if (pick >= 0) {
      sh_tok = lo + sidx[pick];
    } else if (k_eq > 0) {                           // j-th tied token (0-based): the first j with run + (j + 1) et > target
      int j = et > 0.f ? (int)fminf(fmaxf(floorf((target - run) / et), 0.f), (float)(k_eq - 1)) : k_eq - 1;
      while (j > 0 && run + (float)j * et > target) --j;
      while (j < k_eq - 1 && !(run + (float)(j + 1) * et > target)) ++j;
      sh_rank = j;
    } else {
      sh_tok = lo + sidx[k_gt - 1];
    }
    if (m != m) { sh_tok = lo; sh_rank = -1; }      // all-NaN row: first column of the range (see arg-max kernel)
    if (dbg) { dbg[b * 4 + 0] = u; dbg[b * 4 + 1] = (float)n_all; dbg[b * 4 + 2] = (float)nk; dbg[b * 4 + 3] = S; }
  }
  __syncthreads();
  if (sh_rank >= 0) {                               // column of the rank-th tied key: block-wide prefix count over the row
    int* cnt_of = hist;
    const int per = (n + 255) / 256, i0 = tid * per, i1 = min(n, i0 + per);
    int c = 0;
    for (int i = i0; i < i1; ++i) c += keys[i] == thr;
    cnt_of[tid] = c;
    __syncthreads();
    if (tid == 0)
      for (int i = 0, s = 0; i < 256; ++i) { const int ci = cnt_of[i]; cnt_of[i] = s; s += ci; }
    __syncthreads();
    int rank = sh_rank - cnt_of[tid];
    if (rank >= 0 && rank < c)
      for (int i = i0; i < i1; ++i)
        if (keys[i] == thr && rank-- == 0) { sh_tok = lo + i; break; }
    __syncthreads();
  }
  const int tok = sh_tok;
  if (tid == 0) { out_ids[(size_t)b * out_stride + *slot] = (int64_t)tok; pos[b] += 1; }
  for (int k = tid; k < Hd; k += 256) x_next[(size_t)b * Hd + k] = emb[(size_t)tok * Hd + k];
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const int done = atomicAdd(slot + 1, 1);
    if (done == B - 1) { slot[1] = 0; *slot += 1; }
  }
}

// Fixed-order scan over w[0..n) by LSF_NT threads, thread t owning the contiguous slice [i0, i1): per-slice sums, a warp scan of
// them, a scan of the warp totals.  Returns the sum of the slices before this thread's; total = the sum of all of them.
constexpr int LSF_NT = 1024;
__device__ __forceinline__ float lsf_scan(const float* w, int i0, int i1, float* red /* [32] */, float& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float s = 0.f;
  for (int i = i0; i < i1; ++i) s += w[i];
  float inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  float ex = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) ex = 0.f;
  __syncthreads();                                  // red may still be read by the previous scan
  if (lane == 31) red[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    float v = red[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float y = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += y;
    }
    red[lane] = v;
  }
  __syncthreads();
  total = red[31];
  return (warp > 0 ? red[warp - 1] : 0.f) + ex;
}

// The index of the first element whose running sum (the scan above, then this slice in order) exceeds `limit`, or n if none.
__device__ __forceinline__ int lsf_first_above(const float* w, int n, int per, float limit, float* red, int* first) {
  const int i0 = min(n, (int)threadIdx.x * per), i1 = min(n, i0 + per);
  if (threadIdx.x == 0) *first = n;
  float total;
  float run = lsf_scan(w, i0, i1, red, total);
  for (int i = i0; i < i1; ++i) {
    run += w[i];
    if (run > limit) { atomicMin(first, i); break; }
  }
  __syncthreads();
  return *first;
}

__global__ void __launch_bounds__(LSF_NT, 1)
lm_sample_full_embed_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ range, int B, float inv_temp,
                            int top_k, float top_p, const unsigned* __restrict__ seed, const unsigned* __restrict__ row_keys,
                            const float* __restrict__ emb, int Hd, float* __restrict__ x_next, int64_t* __restrict__ out_ids,
                            int out_stride, int* __restrict__ pos, int* __restrict__ slot, float* __restrict__ dbg) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  extern __shared__ uint32_t ls_smem[];
  const int lo = range[0], n = range[1] - lo, b = blockIdx.x, tid = threadIdx.x;
  int cap = 1;
  while (cap < ld) cap <<= 1;
  uint32_t* keys = ls_smem;                       // [ld] keys of the row; after the sort, float scratch
  uint32_t* skey = keys + ((ld + 3) & ~3);        // [cap] survivors: key
  int* sidx = (int*)(skey + cap);                 // [cap] survivors: column
  float* w = reinterpret_cast<float*>(keys);
  __shared__ int hist[256];
  __shared__ float red[32];
  __shared__ int sh_cnt, sh_first;
  for (int i = tid; i < n; i += LSF_NT) keys[i] = ls_key(logits[(size_t)b * ld + i]);
  if (tid == 0) sh_cnt = 0;
  __syncthreads();
  // ---- top-k threshold (top_k <= 0 or >= n: every key, the radix select then returns the smallest), every survivor stored
  int n_gt, n_eq;
  const uint32_t thr = ls_radix_select<LSF_NT>(keys, n, top_k >= 1 && top_k < n ? top_k : n, hist, n_gt, n_eq);
  const int cnt = n_gt + n_eq;
  for (int i = tid; i < n; i += LSF_NT) {
    const uint32_t k = keys[i];
    if (k >= thr) {
      const int s = atomicAdd(&sh_cnt, 1);
      skey[s] = k; sidx[s] = i;
    }
  }
  int P = 1;
  while (P < cnt) P <<= 1;
  for (int i = cnt + tid; i < P; i += LSF_NT) { skey[i] = 0u; sidx[i] = 0x7fffffff; }
  __syncthreads();
  // ---- bitonic sort, descending by key, ascending by column on ties: a total order, so the atomic slots above do not matter
  for (int k2 = 2; k2 <= P; k2 <<= 1)
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int q = tid; q < (P >> 1); q += LSF_NT) {
        const int i = ((q & ~(j - 1)) << 1) | (q & (j - 1)), l = i + j;
        const uint32_t ka = skey[i], kb = skey[l];
        const int ia = sidx[i], ib = sidx[l];
        const bool a_first = ka > kb || (ka == kb && ia < ib);
        const bool up = (i & k2) == 0;
        if (up != a_first) { skey[i] = kb; skey[l] = ka; sidx[i] = ib; sidx[l] = ia; }
      }
      __syncthreads();
    }
  // ---- top-p: a token goes once the softmax mass of the tokens before it exceeds top_p (the first always stays)
  const float m = ls_val(skey[0]);
  const int per = (cnt + LSF_NT - 1) / LSF_NT, i0 = min(cnt, tid * per), i1 = min(cnt, i0 + per);
  int nk = cnt;
  if (top_p < 1.0f) {
    for (int i = i0; i < i1; ++i) w[i] = expf(ls_val(skey[i]) - m);
    float Z;
    lsf_scan(w, i0, i1, red, Z);
    for (int i = i0; i < i1; ++i) w[i] = w[i] / Z;        // each thread rescales the slice it summed
    const int f = lsf_first_above(w, cnt, per, top_p, red, &sh_first);
    nk = f < cnt ? f + 1 : cnt;
  }
  // ---- temperature, normaliser, inverse-CDF draw over the nk kept tokens
  const int per_k = (nk + LSF_NT - 1) / LSF_NT, j0 = min(nk, tid * per_k), j1 = min(nk, j0 + per_k);
  __syncthreads();                                        // every thread is past its reads of w
  for (int i = j0; i < j1; ++i) w[i] = expf((ls_val(skey[i]) - m) * inv_temp);
  float S;
  lsf_scan(w, j0, j1, red, S);
  const float u = ls_uniform(seed, row_keys, *slot, b);
  int pick = lsf_first_above(w, nk, per_k, u * S, red, &sh_first);
  if (pick >= nk) pick = nk - 1;
  const int tok = m != m ? lo : lo + sidx[pick];          // all-NaN row: first column of the range (see arg-max kernel)
  if (tid == 0) {
    if (dbg) { dbg[b * 4 + 0] = u; dbg[b * 4 + 1] = (float)cnt; dbg[b * 4 + 2] = (float)nk; dbg[b * 4 + 3] = S; }
    out_ids[(size_t)b * out_stride + *slot] = (int64_t)tok;
    pos[b] += 1;
  }
  for (int k = tid; k < Hd; k += LSF_NT) x_next[(size_t)b * Hd + k] = emb[(size_t)tok * Hd + k];
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const int done = atomicAdd(slot + 1, 1);
    if (done == B - 1) { slot[1] = 0; *slot += 1; }
  }
}

// ------------------------------------------------------------------------------------------ decode step, projections and attention
// fp32 SIMT dot products spend their time in shared-memory reads (every warp re-reads the whole x tile for one or
// two output columns) and in 32-way shuffle reductions.  These kernels fuse the same way (RMSNorm folded into W,
// RoPE + cache append / residual / SwiGLU / arg-max partials in the epilogue) but run the [32 x K] . [K x 8]
// products as 3-term fp16-split mma.sync tiles:
//   * weights are pre-packed once (qb_lm_pack_weight) as uint4 {hi[4], lo[4]} per 4 consecutive k of a row:
//     the same 4 bytes / parameter as fp32, zero conversion work on the streaming side, one 16-byte load per lane
//     that is directly the B fragment of two MMA k-slots (k-slot order inside an MMA is free as long as A agrees);
//   * each warp owns a contiguous K slice and issues ALL of its weight loads before `griddepcontrol.wait`, so under
//     programmatic dependent launch the HBM latency of step n+1's weights overlaps the tail of kernel n;
//   * x is read straight from global/L2 into A fragments (no shared-memory staging), split hi/lo in registers;
//   * partial tiles of the warps are summed through shared memory in a fixed order (deterministic).
enum { SK_QKV = 0, SK_RESID = 1, SK_GATEUP = 2, SK_HEAD = 3 };

struct SkParams {
  const float* x;        // [B,K]
  int B, K;
  const uint4* W;        // packed rows [N][K/4]
  const uint4* W2;       // GATEUP: up-proj rows
  float eps;
  float* out;            // RESID: x [B,N] updated in place; GATEUP: [B,N]; QKV: q [B,H*64]
  int N;
  int H, Lmax;
  const int* pos;        // QKV: row b's position is pos[b]
  const float* rcos;
  const float* rsin;
  float* kc;
  float* vc;
  const int* range;
  float* part_val;
  int* part_idx;
  float* logits;        // HEAD: optional full logits of the range [B][logits_ld] (sampled decoding); NULL = arg-max partials only
  int logits_ld;
};

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__global__ void lm_pack_weight_kernel(const float* __restrict__ w, long long total4, uint4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const float4 v = reinterpret_cast<const float4*>(w)[i];
  const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  const float2 b0 = __half22float2(h0), b1 = __half22float2(h1);
  const __half2 l0 = __floats2half2_rn(v.x - b0.x, v.y - b0.y), l1 = __floats2half2_rn(v.z - b1.x, v.w - b1.y);
  uint4 o;
  o.x = *reinterpret_cast<const uint32_t*>(&h0); o.y = *reinterpret_cast<const uint32_t*>(&h1);
  o.z = *reinterpret_cast<const uint32_t*>(&l0); o.w = *reinterpret_cast<const uint32_t*>(&l1);
  out[i] = o;
}

// 256-thread variants are capped at 128 registers so that TWO CTAs fit an SM: the gate/up projection (inter/8 = 256 CTAs) and the
// head (256 / 512 CTAs) then run in one / two waves on 132 SMs instead of two / four.
template <int MODE, int SPW, int NW>
__global__ void __launch_bounds__(NW * 32, NW == 8 ? 2 : 1)
lm_skinny_kernel(const SkParams p) {
  constexpr int NT = MODE == SK_RESID ? 1 : 2;       // 8-column tiles per CTA
  __shared__ __align__(16) float red[NW][NT][32][8];
  __shared__ float ssq[NW][32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int K = p.K, K4 = K >> 2, steps_total = K >> 4;
  // ---- which weight rows
  const uint4* wrow[NT];
  bool cta_active = true;
  int row0 = 0, dd0 = 0, hh = 0, sec = 0;
  int row_end = 1 << 30;        // HEAD: rows >= row0 + row_end lie past the range: no load, no candidate, no logit
  if (MODE == SK_QKV) {
    dd0 = (blockIdx.x & 3) * 8; hh = (blockIdx.x >> 2) % p.H; sec = blockIdx.x / (4 * p.H);
    row0 = sec * p.H * 64 + hh * 64 + dd0;
    wrow[0] = p.W + (size_t)(row0 + g) * K4;
    if (NT > 1) wrow[NT - 1] = p.W + (size_t)(row0 + 32 + g) * K4;
  } else if (MODE == SK_RESID) {
    row0 = blockIdx.x * 8;
    wrow[0] = p.W + (size_t)(row0 + g) * K4;
  } else if (MODE == SK_GATEUP) {
    row0 = blockIdx.x * 8;
    wrow[0] = p.W + (size_t)(row0 + g) * K4;
    if (NT > 1) wrow[NT - 1] = p.W2 + (size_t)(row0 + g) * K4;
  } else {
    const int lo = p.range[0], ncol = p.range[1] - lo;      // host-written before the graph launch, not by a kernel
    cta_active = (int)blockIdx.x * 16 < ncol;
    row0 = lo + (cta_active ? blockIdx.x * 16 : 0);
    row_end = p.range[1] - row0;       // the last CTA of a range whose width is not a multiple of 16 owns fewer rows
    wrow[0] = p.W + (size_t)(row0 + g) * K4;
    if (NT > 1) wrow[NT - 1] = p.W + (size_t)(row0 + 8 + g) * K4;
  }
  // ---- all of this warp's weight fragments in flight before the dependency wait
  uint4 wv[NT][SPW];
#pragma unroll
  for (int s = 0; s < SPW; ++s) {
    const int step = warp * SPW + s;
    const bool ok = step < steps_total && cta_active;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
      wv[nt][s] = ok && nt * 8 + g < row_end ? __ldg(wrow[nt] + step * 4 + t) : make_uint4(0u, 0u, 0u, 0u);
  }
  pdl_wait();
  float acc[2][NT][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
  float ss[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int s0 = 0; s0 < SPW; s0 += 4) {       // 4 k-steps of x (16 float4 per lane) in flight at a time
    float4 xv[4][4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int step = warp * SPW + s0 + s;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = r * 8 + g;
        xv[s][r] = (step < steps_total && row < p.B && cta_active)
                       ? *reinterpret_cast<const float4*>(p.x + (size_t)row * K + step * 16 + 4 * t)
                       : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      uint32_t ah[4][2], al[4][2];      // [row group r][k pair]
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float4 v = xv[s][r];
        if (MODE != SK_RESID) ss[r] = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, ss[r]))));
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
          // A regs: {row g k-lo pair, row g+8 k-lo pair, row g k-hi pair, row g+8 k-hi pair}; small terms first
          l_mma(acc[mt][nt], al[2 * mt][0], al[2 * mt + 1][0], al[2 * mt][1], al[2 * mt + 1][1], w.x, w.y);
          l_mma(acc[mt][nt], ah[2 * mt][0], ah[2 * mt + 1][0], ah[2 * mt][1], ah[2 * mt + 1][1], w.z, w.w);
          l_mma(acc[mt][nt], ah[2 * mt][0], ah[2 * mt + 1][0], ah[2 * mt][1], ah[2 * mt + 1][1], w.x, w.y);
        }
    }
  }
  // the dependent grid may start (and prefetch its weights) while this one reduces, stores and drains.  Not before the dependency
  // wait: the dependent's L1 would be invalidated at its launch and then refilled with stale x by an older co-resident kernel.
  pdl_launch_dependents();
  // ---- cross-warp reduction (fixed order)
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      *reinterpret_cast<float2*>(&red[warp][nt][mt * 16 + g][2 * t]) = make_float2(acc[mt][nt][0], acc[mt][nt][1]);
      *reinterpret_cast<float2*>(&red[warp][nt][mt * 16 + g + 8][2 * t]) = make_float2(acc[mt][nt][2], acc[mt][nt][3]);
    }
  if (MODE != SK_RESID) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float q = ss[r];
      q += __shfl_xor_sync(0xffffffffu, q, 1);
      q += __shfl_xor_sync(0xffffffffu, q, 2);
      if (t == 0) ssq[warp][r * 8 + g] = q;
    }
  }
  __syncthreads();
  if (tid >= 256) return;
  const int b = tid >> 3, c = tid & 7;
  float v0 = 0.f, v1 = 0.f, q = 0.f;
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    v0 += red[w][0][b][c];
    if (NT > 1) v1 += red[w][NT - 1][b][c];
    if (MODE != SK_RESID) q += ssq[w][b];
  }
  if (MODE != SK_RESID) {
    const float rs = rsqrtf(q / K + p.eps);
    v0 *= rs;
    v1 *= rs;
  }
  if (MODE == SK_HEAD) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    if (cta_active && b < p.B && c < row_end) {
      bv = v0; bi = row0 + c;
      if (8 + c < row_end && v1 > bv) { bv = v1; bi = row0 + 8 + c; }
      if (p.logits) {
        float* lg = p.logits + (size_t)b * p.logits_ld + (row0 - p.range[0]);
        lg[c] = v0;
        if (8 + c < row_end) lg[8 + c] = v1;
      }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (c == 0) {
      p.part_val[(size_t)blockIdx.x * 32 + b] = bv;
      p.part_idx[(size_t)blockIdx.x * 32 + b] = bi;
    }
    return;
  }
  if (b >= p.B) return;
  if (MODE == SK_RESID) {
    p.out[(size_t)b * p.N + row0 + c] += v0;
  } else if (MODE == SK_GATEUP) {
    p.out[(size_t)b * p.N + row0 + c] = silu_f(v0) * v1;
  } else {  // SK_QKV
    const int pos = p.pos[b], dd = dd0 + c;
    if (sec < 2) {
      const float c1 = p.rcos[pos * 64 + dd], s1 = p.rsin[pos * 64 + dd];
      const float c2 = p.rcos[pos * 64 + dd + 32], s2 = p.rsin[pos * 64 + dd + 32];
      const float y0 = v0 * c1 - v1 * s1, y1 = v1 * c2 + v0 * s2;
      if (sec == 0) {
        p.out[(size_t)b * p.H * 64 + hh * 64 + dd] = y0 * 0.125f;
        p.out[(size_t)b * p.H * 64 + hh * 64 + dd + 32] = y1 * 0.125f;
      } else {
        const size_t o = (((size_t)b * p.H + hh) * p.Lmax + pos) * 64 + dd;
        p.kc[o] = y0;
        p.kc[o + 32] = y1;
      }
    } else {
      const size_t o = (((size_t)b * p.H + hh) * p.Lmax + pos) * 64 + dd;
      p.vc[o] = v0;
      p.vc[o + 32] = v1;
    }
  }
}

// one CTA per (head, batch row), 16 half-warps each walking keys hw, hw+16, ... with an online softmax; a key row
// (64 fp32) is one coalesced 256-byte read by 16 lanes, K and V of 4 keys in flight per lane; the 16 partial
// (max, sum, acc) triples are merged through shared memory in a fixed order.  No score buffer: any cache length.
template <int LM_ATT_U>
__global__ void __launch_bounds__(256)
lm_decode_attn2_kernel(const float* __restrict__ q, const float* __restrict__ kc, const float* __restrict__ vc, int H,
                       int Lmax, const int* __restrict__ posp, float* __restrict__ out) {
  __shared__ __align__(16) float sacc[16][64];
  __shared__ float sm[16], sl[16];
  pdl_wait();
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = lane & 15, hw = warp * 2 + (lane >> 4);
  const int n = posp[b] + 1;                     // keys 0..pos of this row (its K / V at pos were appended by lm_skinny<QKV>)
  const float4 qv = *reinterpret_cast<const float4*>(q + (size_t)b * H * 64 + h * 64 + 4 * c);
  const float4* kb = reinterpret_cast<const float4*>(kc + ((size_t)b * H + h) * Lmax * 64) + c;
  const float4* vb = reinterpret_cast<const float4*>(vc + ((size_t)b * H + h) * Lmax * 64) + c;
  float m = -INFINITY, l = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int base = warp * 2; base < n; base += 16 * LM_ATT_U) {       // warp-uniform trip count (full-mask shuffles inside)
    const int j0 = base + (lane >> 4);
    float4 kv[LM_ATT_U], vv[LM_ATT_U];
    float s[LM_ATT_U];
#pragma unroll
    for (int u = 0; u < LM_ATT_U; ++u) {
      const int j = j0 + 16 * u;
      const bool ok = j < n;
      kv[u] = ok ? kb[(size_t)j * 16] : make_float4(0.f, 0.f, 0.f, 0.f);
      vv[u] = ok ? vb[(size_t)j * 16] : make_float4(0.f, 0.f, 0.f, 0.f);
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
    if (mn > -INFINITY) {                       // (the odd half-warp can run out of keys one trip early)
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
  pdl_launch_dependents();      // after the main loop, as in lm_skinny_kernel
  *reinterpret_cast<float4*>(&sacc[hw][4 * c]) = acc;
  if (c == 0) { sm[hw] = m; sl[hw] = l; }
  __syncthreads();
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
}

}  // namespace qb
using namespace qb;

extern "C" int qb_lm_qkv_prep(const float* qkv, int64_t B, int64_t L, int32_t heads, int32_t pos0, const float* rope_cos,
                              const float* rope_sin, float* q32, float* k_cache, float* v_cache, int32_t Lmax,
                              void* stream) {
  QB_REQUIRE(qkv && rope_cos && rope_sin && q32 && k_cache && v_cache && pos0 + L <= Lmax, "lm_qkv_prep: bad args");
  const long long total = B * L * heads * 32;
  lm_qkv_prep_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
      qkv, (int)L, heads, pos0, rope_cos, rope_sin, q32, k_cache, v_cache, Lmax, total);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_lm_flash_attn(const float* q32, const float* k_cache, const float* v_cache, int64_t B, int64_t L,
                                int32_t heads, int32_t pos0, int32_t Lmax, qb_half* out_hi, qb_half* out_lo, void* stream) {
  QB_REQUIRE(q32 && k_cache && v_cache && out_hi && L > 0, "lm_flash_attn: bad args");
  dim3 grid((unsigned)ceil_div(L, LF_BQ), (unsigned)heads, (unsigned)B);
  const size_t smem = (size_t)(2 * LF_BQ + 4 * LF_BK) * LF_P * sizeof(__half);
    QB_CHECK_CUDA(cudaFuncSetAttribute(lm_flash_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // per-device state: set on every launch (cheap)
  lm_flash_attn_kernel<<<grid, 128, smem, (cudaStream_t)stream>>>(q32, k_cache, v_cache, (int)L, heads, pos0, Lmax,
                                                                 (__half*)out_hi, (__half*)out_lo);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------ decode step, host side
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  g_launches++;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

template <int MODE>
static int launch_skinny(const SkParams& p, int n_ctas, cudaStream_t st) {
  QB_REQUIRE(p.K % 16 == 0 && p.K <= 2048, "lm decode: K = %d unsupported (multiple of 16, <= 2048)", p.K);
  cudaError_t e;
  if (p.K <= 512) e = launch_pdl(lm_skinny_kernel<MODE, 4, 8>, dim3((unsigned)n_ctas), dim3(256), 0, st, p);
  else if (p.K <= 1024) e = launch_pdl(lm_skinny_kernel<MODE, 4, 16>, dim3((unsigned)n_ctas), dim3(512), 0, st, p);
  else e = launch_pdl(lm_skinny_kernel<MODE, 8, 16>, dim3((unsigned)n_ctas), dim3(512), 0, st, p);
  QB_CHECK_CUDA(e);
  return 0;
}

extern "C" int qb_lm_pack_weight(const float* w, int64_t n, int64_t k, qb_half* out, void* stream) {
  QB_REQUIRE(w && out && k % 4 == 0, "lm_pack_weight: bad args");
  const long long total4 = n * k / 4;
  lm_pack_weight_kernel<<<(unsigned)ceil_div(total4, 256), 256, 0, (cudaStream_t)stream>>>(w, total4, (uint4*)out);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int g_lm_att_unroll = LM_ATT_U_DEFAULT;
extern "C" int qb_lm_set_att_unroll(int32_t keys_per_lane) {
  QB_REQUIRE(keys_per_lane == 4 || keys_per_lane == 8, "lm_set_att_unroll: 4 or 8 (got %d)", (int)keys_per_lane);
  g_lm_att_unroll = keys_per_lane;
  return 0;
}

extern "C" int qb_lm_decode_layer_tc(float* x, int64_t B, int32_t hidden, int32_t heads, int32_t inter, const qb_half* wqkv,
                                     const qb_half* wo, const qb_half* wgate, const qb_half* wup, const qb_half* wdown,
                                     float* k_cache, float* v_cache, int32_t Lmax, const int32_t* pos, const float* rope_cos,
                                     const float* rope_sin, float* q_buf, float* attn_buf, float* mlp_buf, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(B >= 1 && B <= 32, "lm_decode_layer_tc: batch must be 1..32 (got %lld)", (long long)B);
  QB_REQUIRE(hidden == heads * 64 && hidden % 16 == 0 && inter % 16 == 0, "lm_decode_layer_tc: unsupported dims");
  SkParams p = {};
  p.B = (int)B; p.eps = 1e-6f; p.H = heads; p.Lmax = Lmax; p.pos = pos;
  p.rcos = rope_cos; p.rsin = rope_sin;
  p.kc = k_cache; p.vc = v_cache;
  // RMSNorm + QKV + RoPE + cache append
  p.x = x; p.K = hidden; p.W = (const uint4*)wqkv; p.out = q_buf;
  if (int e = launch_skinny<SK_QKV>(p, 3 * heads * 4, st)) return e;
  // keys in flight per half-warp trip (K and V rows of LM_ATT_U keys per lane), qb_lm_set_att_unroll: 8 for a single decode chain
  // (latency-bound), 4 when several chains share the GPU (throughput-bound)
  auto att = g_lm_att_unroll == 4 ? lm_decode_attn2_kernel<4> : lm_decode_attn2_kernel<8>;
  QB_CHECK_CUDA(launch_pdl(att, dim3((unsigned)heads, (unsigned)B), dim3(256), 0, st, (const float*)q_buf,
                           (const float*)k_cache, (const float*)v_cache, (int)heads, (int)Lmax, (const int*)pos, attn_buf));
  // o_proj + residual
  p.x = attn_buf; p.K = hidden; p.W = (const uint4*)wo; p.out = x; p.N = hidden;
  if (int e = launch_skinny<SK_RESID>(p, hidden / 8, st)) return e;
  // RMSNorm + gate/up + SwiGLU
  p.x = x; p.K = hidden; p.W = (const uint4*)wgate; p.W2 = (const uint4*)wup; p.out = mlp_buf; p.N = inter;
  if (int e = launch_skinny<SK_GATEUP>(p, inter / 8, st)) return e;
  // down + residual
  p.x = mlp_buf; p.K = inter; p.W = (const uint4*)wdown; p.W2 = nullptr; p.out = x; p.N = hidden;
  if (int e = launch_skinny<SK_RESID>(p, hidden / 8, st)) return e;
  return 0;
}

extern "C" int qb_lm_head_argmax_tc(const float* x, int64_t B, int32_t hidden, const qb_half* w_head, const int32_t* range,
                                    int32_t max_cols, const float* embedding, float* x_next, int64_t* out_ids,
                                    int32_t out_stride, int32_t* pos, int32_t* slot, float* part_val, int32_t* part_idx,
                                    void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(B >= 1 && B <= 32 && max_cols % 16 == 0, "lm_head_argmax_tc: bad args (max_cols must be a multiple of 16)");
  SkParams p = {};
  p.B = (int)B; p.eps = 1e-6f; p.x = x; p.K = hidden; p.W = (const uint4*)w_head; p.range = range;
  p.part_val = part_val; p.part_idx = part_idx;
  if (int e = launch_skinny<SK_HEAD>(p, max_cols / 16, st)) return e;
  QB_CHECK_CUDA(launch_pdl(lm_argmax_embed_kernel, dim3((unsigned)B), dim3(128), 0, st, (const float*)part_val,
                           (const int*)part_idx, (int)(max_cols / 16), (int)B, embedding, (int)hidden, x_next, out_ids,
                           (int)out_stride, (int*)pos, (int*)slot, (const int*)range, 0x7ffffffe));
  return 0;
}

// Sampled decoding step: as qb_lm_head_argmax_tc, but the head writes the full range logits [B][max_cols] and the token is
// drawn by lm_sample_embed_kernel (1 <= top_k <= LS_MAX) or lm_sample_full_embed_kernel (any other top_k) (top-k -> top-p ->
// temperature -> multinomial, llm.py:253-289).  Exactly one of seed (one stream for the call) and row_keys (one per row).
static int head_sample(const char* name, const float* x, int64_t B, int32_t hidden, const qb_half* w_head, const int32_t* range,
                       int32_t max_cols, const float* embedding, float* x_next, int64_t* out_ids, int32_t out_stride, int32_t* pos,
                       int32_t* slot, float* part_val, int32_t* part_idx, float* logits, float temperature, int32_t top_k,
                       float top_p, const uint32_t* seed, const uint32_t* row_keys, float* debug, cudaStream_t st) {
  QB_REQUIRE(B >= 1 && B <= 32 && max_cols % 16 == 0, "%s: bad args (max_cols must be a multiple of 16)", name);
  QB_REQUIRE(logits && (seed || row_keys), "%s: logits / seed buffers required", name);
  QB_REQUIRE(temperature > 0.f && temperature <= 1.0f, "%s: temperature must be in (0, 1] (llm.py:278)", name);
  SkParams p = {};
  p.B = (int)B; p.eps = 1e-6f; p.x = x; p.K = hidden; p.W = (const uint4*)w_head; p.range = range;
  p.part_val = part_val; p.part_idx = part_idx; p.logits = logits; p.logits_ld = max_cols;
  if (int e = launch_skinny<SK_HEAD>(p, max_cols / 16, st)) return e;
  const size_t smem_cap = 160 * 1024;
  if (top_k >= 1 && top_k <= LS_MAX) {
    const size_t smem = ((size_t)((max_cols + 3) & ~3) + 2 * LS_MAX) * 4;
    QB_CHECK_CUDA(cudaFuncSetAttribute(lm_sample_embed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap));   // per-device state: set on every launch (cheap)
    QB_REQUIRE(smem <= smem_cap, "%s: range too wide (%d columns)", name, max_cols);
    QB_CHECK_CUDA(launch_pdl(lm_sample_embed_kernel, dim3((unsigned)B), dim3(256), smem, st, (const float*)logits, (int)max_cols,
                             (const int*)range, (int)B, 1.0f / temperature, (int)top_k, top_p, (const unsigned*)seed,
                             (const unsigned*)row_keys, embedding, (int)hidden, x_next, out_ids, (int)out_stride, (int*)pos, (int*)slot,
                             debug));
    return 0;
  }
  size_t cap = 1;
  while (cap < (size_t)max_cols) cap <<= 1;
  const size_t smem = ((size_t)((max_cols + 3) & ~3) + 2 * cap) * 4;      // row keys + every column as a survivor (key, id)
  QB_CHECK_CUDA(cudaFuncSetAttribute(lm_sample_full_embed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap));
  QB_REQUIRE(smem <= smem_cap, "%s: range too wide for top_k = %d (%d columns)", name, (int)top_k, max_cols);
  QB_CHECK_CUDA(launch_pdl(lm_sample_full_embed_kernel, dim3((unsigned)B), dim3(LSF_NT), smem, st, (const float*)logits,
                           (int)max_cols, (const int*)range, (int)B, 1.0f / temperature, (int)top_k, top_p, (const unsigned*)seed,
                           (const unsigned*)row_keys, embedding, (int)hidden, x_next, out_ids, (int)out_stride, (int*)pos, (int*)slot,
                           debug));
  return 0;
}

extern "C" int qb_lm_head_sample_tc(const float* x, int64_t B, int32_t hidden, const qb_half* w_head, const int32_t* range,
                                    int32_t max_cols, const float* embedding, float* x_next, int64_t* out_ids,
                                    int32_t out_stride, int32_t* pos, int32_t* slot, float* part_val, int32_t* part_idx,
                                    float* logits, float temperature, int32_t top_k, float top_p, const uint32_t* seed,
                                    float* debug, void* stream) {
  QB_REQUIRE(seed, "lm_head_sample_tc: seed buffer required");
  return head_sample("lm_head_sample_tc", x, B, hidden, w_head, range, max_cols, embedding, x_next, out_ids, out_stride, pos, slot,
                     part_val, part_idx, logits, temperature, top_k, top_p, seed, nullptr, debug, (cudaStream_t)stream);
}

extern "C" int qb_lm_head_sample_rows_tc(const float* x, int64_t B, int32_t hidden, const qb_half* w_head, const int32_t* range,
                                         int32_t max_cols, const float* embedding, float* x_next, int64_t* out_ids,
                                         int32_t out_stride, int32_t* pos, int32_t* slot, float* part_val, int32_t* part_idx,
                                         float* logits, float temperature, int32_t top_k, float top_p, const uint32_t* row_keys,
                                         float* debug, void* stream) {
  QB_REQUIRE(row_keys, "lm_head_sample_rows_tc: row_keys buffer required");
  return head_sample("lm_head_sample_rows_tc", x, B, hidden, w_head, range, max_cols, embedding, x_next, out_ids, out_stride, pos,
                     slot, part_val, part_idx, logits, temperature, top_k, top_p, nullptr, row_keys, debug, (cudaStream_t)stream);
}

extern "C" int qb_lm_loss(const float* logits, int64_t ld, int64_t M, int32_t V, const int64_t* targets, float label_smoothing,
                          float* workspace /* [2*M] */, float* out /* {loss, accuracy} */, void* stream) {
  QB_REQUIRE(logits && targets && workspace && out && M >= 1 && V >= 2 && ld >= V, "lm_loss: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  float* row_loss = workspace;
  int* row_hit = (int*)(workspace + M);
  lm_loss_rows_kernel<<<(unsigned)M, 256, 0, st>>>(logits, ld, V, targets, label_smoothing, row_loss, row_hit);
  lm_loss_reduce_kernel<<<1, 256, 0, st>>>(row_loss, row_hit, M, out);
  g_launches += 2;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
