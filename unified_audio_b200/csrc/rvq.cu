// Residual vector quantiser (reference call sites HCodec-2.0/vq/codec.py:81-82, 94-95; arithmetic
// template HCodec-2.0/vq/core_vq.py:223-238, 394-412; upstream vector-quantize-pytorch 1.22.15).
//
// Encode, per layer q (strictly sequential - the residual chain):
//   1. scores[m,j] = |e_j|^2 - 2 r_m.e_j  on the tensor cores: the wgmma GEMM with 3-term fp16
//      split operands (~2^-21 relative), bias = -|e|^2/2 and gamma = -2 folded into its epilogue;
//   2. rvq_select (this file): warp per token - arg-min over the K scores; every candidate whose
//      score lies within `tol` of the minimum is re-ranked by its EXACT squared distance in fp64
//      (lowest index wins exact ties), so the chosen index equals the exact-arithmetic arg-min of
//      the fp32 residual path irrespective of tensor-core rounding;
//   3. the same kernel updates the residual in fp32 (r -= e_idx, as the reference), accumulates
//      the quantised sum and emits the next layer's fp16 planes.
#include <atomic>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

__global__ void rvq_select_kernel(const float* __restrict__ scores, float* __restrict__ resid,
                                  const float* __restrict__ cb /*[K,D] layer q*/, long long M, int D, int K,
                                  float tol_rel, float e2max, int64_t* __restrict__ idx, int nq, int q,
                                  float* __restrict__ quant, __half* __restrict__ hi, __half* __restrict__ lo) {
  const int lane = threadIdx.x & 31;
  const long long m = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= M) return;
  const float* sr = scores + m * K;
  float* r = resid + m * D;
  // |r|^2 for the tolerance scale
  float r2 = 0.f;
  for (int d = lane; d < D; d += 32) r2 = fmaf(r[d], r[d], r2);
  r2 = warp_sum(r2);
  // pass 1: fp32 arg-min, lowest index on ties
  float best = INFINITY;
  int bi = 0x7fffffff;
  for (int j = lane; j < K; j += 32) {
    const float s = sr[j];
    if (s < best) { best = s; bi = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  // pass 2: near-ties -> exact fp64 re-rank
  const float thr = best + tol_rel * (r2 + e2max);
  int cnt = 0;
  for (int j = lane; j < K; j += 32) cnt += (sr[j] <= thr) ? 1 : 0;
  cnt = (int)warp_sum((float)cnt);
  if (cnt > 1) {
    double dbest = 1e300;
    int di = 0x7fffffff;
    for (int j0 = 0; j0 < K; j0 += 32) {
      const int j = j0 + lane;
      unsigned mask = __ballot_sync(0xffffffffu, j < K && sr[j] <= thr);
      while (mask) {
        const int cand = j0 + __ffs(mask) - 1;
        mask &= mask - 1;
        const float* e = cb + (long long)cand * D;
        double acc = 0.0;
        for (int d = lane; d < D; d += 32) {
          const double df = (double)r[d] - (double)e[d];
          acc += df * df;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (acc < dbest) { dbest = acc; di = cand; }  // candidates visited in ascending index order
      }
    }
    bi = di;
  }
  if (lane == 0) idx[m * nq + q] = (int64_t)bi;
  const float* e = cb + (long long)bi * D;
  for (int d = lane; d < D; d += 32) {
    const float ev = e[d];
    const float rn = r[d] - ev;
    r[d] = rn;
    if (quant) quant[m * D + d] = (q == 0 ? 0.f : quant[m * D + d]) + ev;
    if (hi) {
      __half h, l;
      split_f16(rn, h, l);
      hi[m * D + d] = h;
      lo[m * D + d] = l;
    }
  }
}

__global__ void rvq_init_kernel(const float* __restrict__ x, float* __restrict__ resid, __half* __restrict__ hi,
                                __half* __restrict__ lo, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i];
  resid[i] = v;
  __half h, l;
  split_f16(v, h, l);
  hi[i] = h;
  lo[i] = l;
}

__global__ void rvq_decode_kernel(const int64_t* __restrict__ idx, const float* __restrict__ cb, int D, int K, int nq,
                                  float* __restrict__ out, long long out_ld, long long col_off) {
  const long long m = blockIdx.x;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    for (int q = 0; q < nq; ++q) {
      const int64_t i = idx[m * nq + q];
      if (i >= 0) acc += cb[((long long)q * K + i) * D + d];
    }
    out[m * out_ld + col_off + d] = acc;
  }
}

// Factorised VQ tokenize (BiCodec's semantic quantiser, factorized_vector_quantize.py:148-152,169-187), all in fp64: the
// codebook is 8-wide, so the whole scan is ~1 G fp64 FMA at the largest batches and needs no shortlist / re-rank.
//   phase 1: a warp per row: z_e = W_in z + b_in (fp64 sums over D_in), e = z_e / max(|z_e|, 1e-12) -> shared memory;
//   phase 2: the codebook streams through shared memory in tiles; warp w scans its slice of every tile with lane = row, so
//            every lane of a warp reads the same code (broadcast); score 2 e.c - |c|^2 (-dist without the row constant |e|^2);
//   then the FVQ_SLICES per-row winners are merged: highest score, lowest index on exact ties.
constexpr int FVQ_ROWS = 32, FVQ_SLICES = 8, FVQ_TILE = 256;

template <int CD>
__global__ void __launch_bounds__(FVQ_ROWS * FVQ_SLICES)
fvq_tokenize_kernel(const float* __restrict__ z, long long M, int D, const float* __restrict__ w_in, const float* __restrict__ b_in,
                    const double* __restrict__ cb, int K, int cdim, int64_t* __restrict__ idx, float* __restrict__ z_e) {
  __shared__ double e_s[FVQ_ROWS][CD];
  __shared__ double c_s[FVQ_TILE][CD];
  __shared__ double c2_s[FVQ_TILE];
  __shared__ double best_s[FVQ_SLICES][FVQ_ROWS];
  __shared__ int bi_s[FVQ_SLICES][FVQ_ROWS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long row0 = (long long)blockIdx.x * FVQ_ROWS;
  for (int r = warp; r < FVQ_ROWS; r += FVQ_SLICES) {
    const long long m = row0 + r;
    double acc[CD];
#pragma unroll
    for (int j = 0; j < CD; ++j) acc[j] = 0.0;
    if (m < M) {
      const float* zr = z + m * D;
      for (int c = lane; c < D; c += 32) {
        const double v = (double)zr[c];
#pragma unroll
        for (int j = 0; j < CD; ++j)
          if (j < cdim) acc[j] = fma((double)w_in[(long long)j * D + c], v, acc[j]);
      }
    }
    double n2 = 0.0;
#pragma unroll
    for (int j = 0; j < CD; ++j) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
      if (j < cdim && m < M) {
        acc[j] += (double)b_in[j];
        n2 = fma(acc[j], acc[j], n2);
        if (z_e && lane == 0) z_e[m * cdim + j] = (float)acc[j];
      }
    }
    const double inv = 1.0 / fmax(sqrt(n2), 1e-12);               // F.normalize
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < CD; ++j) e_s[r][j] = (j < cdim && m < M) ? acc[j] * inv : 0.0;
    }
  }
  __syncthreads();
  double e[CD];
#pragma unroll
  for (int j = 0; j < CD; ++j) e[j] = e_s[lane][j];
  double best = -INFINITY;
  int bi = 0x7fffffff;
  constexpr int PER = FVQ_TILE / FVQ_SLICES;
  for (int k0 = 0; k0 < K; k0 += FVQ_TILE) {
    const int nk = min(FVQ_TILE, K - k0);
    for (int i = threadIdx.x; i < FVQ_TILE * CD; i += blockDim.x) {
      const int k = i / CD, j = i % CD;
      c_s[k][j] = (k < nk && j < cdim) ? cb[(long long)(k0 + k) * cdim + j] : 0.0;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < nk; k += blockDim.x) {
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < CD; ++j) s = fma(c_s[k][j], c_s[k][j], s);
      c2_s[k] = s;
    }
    __syncthreads();
    const int kb = warp * PER, ke = min(kb + PER, nk);
    for (int k = kb; k < ke; ++k) {                                  // ascending: strict > keeps the lowest index
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < CD; ++j) s = fma(e[j], c_s[k][j], s);
      const double score = 2.0 * s - c2_s[k];
      if (score > best) { best = score; bi = k0 + k; }
    }
    __syncthreads();
  }
  best_s[warp][lane] = best;
  bi_s[warp][lane] = bi;
  __syncthreads();
  if (warp == 0) {
    const long long m = row0 + lane;
    double b = best_s[0][lane];
    int id = bi_s[0][lane];
    for (int w = 1; w < FVQ_SLICES; ++w) {
      const double o = best_s[w][lane];
      const int oi = bi_s[w][lane];
      if (o > b || (o == b && oi < id)) { b = o; id = oi; }
    }
    if (m < M) idx[m] = id == 0x7fffffff ? 0 : (int64_t)id;        // an all-NaN row: index 0, as torch.max
  }
}


// FactorizedVectorQuantize.forward's usage statistics (factorized_vector_quantize.py:97-103): an int32 histogram of the indices
// (integer atomics: the counts do not depend on the order), then one block reduces the K bins in a fixed order in fp64.
constexpr int FVQ_USAGE_THREADS = 256;

__global__ void fvq_histogram_kernel(const int64_t* __restrict__ idx, long long n, int K, int32_t* __restrict__ counts) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int64_t k = idx[i];
    if (k >= 0 && k < K) atomicAdd(counts + k, 1);
  }
}

__global__ void fvq_usage_kernel(const int32_t* __restrict__ counts, int K, long long n, float* __restrict__ perplexity,
                                 float* __restrict__ active) {
  __shared__ double s_h[FVQ_USAGE_THREADS];
  __shared__ int s_a[FVQ_USAGE_THREADS];
  double h = 0.0;
  int a = 0;
  for (int k = threadIdx.x; k < K; k += FVQ_USAGE_THREADS) {
    const double p = (double)counts[k] / (double)n;
    h += p * log(p + 1e-10);
    a += counts[k] > 0;
  }
  s_h[threadIdx.x] = h;
  s_a[threadIdx.x] = a;
  __syncthreads();
  for (int o = FVQ_USAGE_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s_h[threadIdx.x] += s_h[threadIdx.x + o];
      s_a[threadIdx.x] += s_a[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *perplexity = (float)exp(-s_h[0]);
    *active = (float)s_a[0];
  }
}

}  // namespace qb
using namespace qb;

extern "C" int qb_fvq_tokenize(const float* z, int64_t M, int32_t D_in, const float* w_in, const float* b_in, const double* codebook_n,
                               int32_t K, int32_t cdim, int64_t* idx, float* z_e, void* stream) {
  QB_REQUIRE(z && w_in && b_in && codebook_n && idx && M >= 0 && D_in >= 1 && K >= 1, "fvq_tokenize: bad args");
  QB_REQUIRE(cdim >= 1 && cdim <= 16, "fvq_tokenize: codebook_dim must be 1..16 (got %d)", cdim);
  if (M == 0) return 0;
  const unsigned grid = (unsigned)ceil_div(M, FVQ_ROWS);
  if (cdim <= 8)
    fvq_tokenize_kernel<8><<<grid, FVQ_ROWS * FVQ_SLICES, 0, (cudaStream_t)stream>>>(z, M, D_in, w_in, b_in, codebook_n, K, cdim, idx, z_e);
  else
    fvq_tokenize_kernel<16><<<grid, FVQ_ROWS * FVQ_SLICES, 0, (cudaStream_t)stream>>>(z, M, D_in, w_in, b_in, codebook_n, K, cdim, idx, z_e);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int64_t qb_rvq_workspace_bytes(int64_t M, int32_t D, int32_t K) {
  return M * D * 4 + 2 * M * D * 2 + M * (int64_t)K * 4 + 1024;
}

extern "C" int qb_rvq_encode(const float* x, const float* codebooks, const qb_half* cb_hi, const qb_half* cb_lo,
                             const float* neg_half_e2, float e2max, int64_t M, int32_t D, int32_t K, int32_t nq,
                             int64_t* idx, float* quantized, void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  QB_REQUIRE(x && codebooks && cb_hi && cb_lo && neg_half_e2 && idx && workspace, "rvq_encode: bad args");
  QB_REQUIRE(D % 64 == 0, "rvq_encode: D must be a multiple of 64");
  if (M == 0) return 0;
  uint8_t* ws = (uint8_t*)workspace;
  float* resid = (float*)ws; ws += (size_t)M * D * 4;
  __half* hi = (__half*)ws; ws += (size_t)M * D * 2;
  __half* lo = (__half*)ws; ws += (size_t)M * D * 2;
  ws = (uint8_t*)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
  float* scores = (float*)ws;
  const long long n = (long long)M * D;
  rvq_init_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(x, resid, hi, lo, n);
  g_launches++;
  for (int q = 0; q < nq; ++q) {
    qb_gemm_desc g = {};
    g.a_hi = (const qb_half*)hi; g.a_lo = (const qb_half*)lo;
    g.a_batch = 1; g.a_rows_per_batch = M; g.a_ld = D; g.taps = 1; g.stride = 1; g.m_per_batch = M;
    g.w_hi = cb_hi + (size_t)q * K * D; g.w_lo = cb_lo + (size_t)q * K * D; g.n = K;
    g.bias = neg_half_e2 + (size_t)q * K;            // v = (acc - |e|^2/2) ...
    g.gamma = neg_half_e2 + (size_t)nq * K;           // ... * (-2): K-vector of -2 appended by the caller
    g.act = QB_ACT_NONE; g.act2 = QB_ACT_NONE;
    g.out_f32.ptr = scores; g.out_f32.ld = K; g.out_f32.rows_per_batch = M; g.out_f32.row_off = 0;
    if (int e = qb_gemm(&g, stream)) return e;
    rvq_select_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, st>>>(scores, resid, codebooks + (size_t)q * K * D, M, D, K,
                                                                1e-4f, e2max, idx, nq, q, quantized,
                                                                q + 1 < nq ? hi : nullptr, lo);
    g_launches++;
  }
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_rvq_decode(const int64_t* idx, const float* codebooks, int64_t M, int32_t D, int32_t K, int32_t nq,
                             float* out, int64_t out_ld, int64_t col_off, void* stream) {
  QB_REQUIRE(idx && codebooks && out, "rvq_decode: bad args");
  if (M == 0) return 0;
  rvq_decode_kernel<<<(unsigned)M, 128, 0, (cudaStream_t)stream>>>(idx, codebooks, D, K, nq, out, out_ld, col_off);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_fvq_usage(const int64_t* idx, int64_t n, int32_t K, int32_t* counts, float* perplexity, float* active, void* stream) {
  QB_REQUIRE(idx && counts && perplexity && active, "fvq_usage: bad args");
  QB_REQUIRE(n >= 1 && K >= 1, "fvq_usage: needs at least one index and one code (n %lld, K %d)", (long long)n, K);
  cudaStream_t st = (cudaStream_t)stream;
  QB_CHECK_CUDA(cudaMemsetAsync(counts, 0, (size_t)K * sizeof(int32_t), st));
  const long long g = ceil_div(n, 256);
  fvq_histogram_kernel<<<(unsigned)(g < 132 * 16 ? g : 132 * 16), 256, 0, st>>>(idx, n, K, counts);
  fvq_usage_kernel<<<1, FVQ_USAGE_THREADS, 0, st>>>(counts, K, n, perplexity, active);
  g_launches += 2;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
