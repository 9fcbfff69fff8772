// Data-dependent primitives of H-Codec-1.5's adaptive frame-rate path (SURVEY.md 8f.4), on the device:
//   FlexiCodec._perform_similarity_alignment_vectorized   QuarkAudio-HCodec/HCodec-1.5/adaptive/modeling_flexicodec_new.py:828-921
//   Codec._inject_length_to_codes_index / _extract_length_from_codes_index   HCodec-1.5/vq/codec_adaptive.py:68-80
//   FlexiCodec._deaggregate_features_from_token_lengths   modeling_flexicodec_new.py:1007-1041
// The reference builds a dense [B, G, T] alignment matrix with cummax / cumsum / scatter and repeat_interleave in a Python loop; here
// a clip is one CTA: cosine similarities of consecutive frames (warp per pair), then one in-CTA scan that emits the frame -> token
// map and the token lengths directly (the alignment matrix is a one-hot of that map: produced on request for the callers that want it).
#include <atomic>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

// h [B, T, D] fp32 (channel-last).  sim [B, T-1]; seg [B, T] int32 (frame -> token); lengths [B, T] int32 (frames per token, 0 past
// the clip's last token); n_groups [B] int32.
__global__ void __launch_bounds__(256)
similarity_alignment_kernel(const float* __restrict__ h, int T, int D, float threshold, int max_per_group, float* __restrict__ sim,
                            int* __restrict__ seg, int* __restrict__ lengths, int* __restrict__ n_groups) {
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* hb = h + (size_t)b * T * D;
  float* sb = sim + (size_t)b * (T - 1);
  // F.cosine_similarity(x, y, dim, eps = 1e-8): x.y / (max(|x|, eps) * max(|y|, eps))
  for (int t = warp; t < T - 1; t += nw) {
    const float* x = hb + (size_t)t * D;
    const float* y = x + D;
    float xy = 0.f, xx = 0.f, yy = 0.f;
    for (int d = lane; d < D; d += 32) {
      const float a = x[d], c = y[d];
      xy = fmaf(a, c, xy); xx = fmaf(a, a, xx); yy = fmaf(c, c, yy);
    }
    xy = warp_sum(xy); xx = warp_sum(xx); yy = warp_sum(yy);
    if (lane == 0) sb[t] = xy / (fmaxf(sqrtf(xx), 1e-8f) * fmaxf(sqrtf(yy), 1e-8f));
  }
  __syncthreads();
  // sequential scan (T is a few hundred to a few thousand frames): similarity boundary or length cap opens a new token
  if (threadIdx.x == 0) {
    int* sg = seg + (size_t)b * T;
    int* ln = lengths + (size_t)b * T;
    int g = -1, in_seg = 0;
    for (int t = 0; t < T; ++t) {
      const bool boundary = t == 0 || sb[t - 1] <= threshold;
      if (boundary) in_seg = 0;
      const bool split = max_per_group > 0 ? (in_seg % max_per_group) == 0 : boundary;
      if (split) { ++g; ln[g] = 0; }
      sg[t] = g;
      ln[g] += 1;
      ++in_seg;
    }
    for (int i = g + 1; i < T; ++i) ln[i] = 0;
    n_groups[b] = g + 1;
  }
}
// alignment matrix [B, G, T] float 0/1 from the frame -> token map
__global__ void alignment_matrix_kernel(const int* __restrict__ seg, int T, int G, float* __restrict__ align, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const int g = (int)((i / T) % G);
    const long long b = i / ((long long)T * G);
    align[i] = seg[b * T + t] == g ? 1.f : 0.f;
  }
}
// codes [B, nq, G] int64, lengths [B, G] int32: inject  -> (len - 1) * K + code;  extract -> code % K, len = code / K + 1 (row 0)
__global__ void pack_lengths_kernel(const int64_t* __restrict__ codes, const int* __restrict__ lengths, int nq, int G, int K,
                                    int64_t* __restrict__ out, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const long long b = i / ((long long)G * nq);
    out[i] = ((int64_t)lengths[b * G + g] - 1) * K + codes[i];
  }
}
__global__ void unpack_lengths_kernel(const int64_t* __restrict__ codes, int nq, int G, int K, int64_t* __restrict__ plain,
                                      int* __restrict__ lengths, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int q = (int)((i / G) % nq);
    const long long b = i / ((long long)G * nq);
    const int64_t c = codes[i];
    // torch.div(codes, K, rounding_mode="floor") and python-style % for negative codes
    int64_t fl = c / K;
    if ((c % K != 0) && ((c < 0) != (K < 0))) --fl;
    plain[i] = c - fl * K;
    if (q == 0) lengths[b * G + g] = (int)(fl + 1);
  }
}
// x [B, C, G] (channel-first, any 8-byte element type viewed as int64 or fp32 via elem_bytes), lengths [B, G] -> out [B, C, T_out]
// repeat_interleave per clip, zero padded to T_out; offsets [B, G] = exclusive prefix sums of the lengths (computed by offsets_kernel)
__global__ void length_offsets_kernel(const int* __restrict__ lengths, int G, int* __restrict__ offsets, int* __restrict__ totals) {
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int g = 0; g < G; ++g) { offsets[(size_t)b * G + g] = acc; acc += max(lengths[(size_t)b * G + g], 0); }
    totals[b] = acc;
  }
}
template <typename T>
__global__ void deaggregate_kernel(const T* __restrict__ x, const int* __restrict__ lengths, const int* __restrict__ offsets, int C, int G,
                                   int T_out, T* __restrict__ out, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % G);
    const int c = (int)((i / G) % C);
    const long long b = i / ((long long)G * C);
    const int o = offsets[b * G + g], n = lengths[b * G + g];
    const T v = x[i];
    T* dst = out + (b * C + c) * (long long)T_out + o;
    for (int r = 0; r < n && o + r < T_out; ++r) dst[r] = v;
  }
}
// QueryTokenAggregator input (adaptive/model_blocks/mimi/transformer.py:760-805): the T frames of a clip and one query token per group
// in one sequence of T + G rows - frame t sits at t + seg[t] (one query has been inserted behind every earlier group), the query of
// group g right behind the group's last frame (offset + length + g) and holds mean(frames of g) + query_embedding; padded groups
// (g >= n_groups[b]) fill the tail T + g with the bare embedding.  grid (T + G, B); qpos [B, G] = row of each query.
__global__ void __launch_bounds__(128)
agg_interleave_kernel(const float* __restrict__ feats, const int* __restrict__ seg, const int* __restrict__ lengths,
                      const int* __restrict__ offsets, const int* __restrict__ n_groups, const float* __restrict__ qemb, int T, int G,
                      int D, float* __restrict__ out, int* __restrict__ qpos) {
  const int s = blockIdx.x, b = blockIdx.y, L = T + G;
  const float* fb = feats + (size_t)b * T * D;
  float* ob = out + (size_t)b * L * D;
  if (s < T) {
    const int pos = s + seg[(size_t)b * T + s];
    for (int d = threadIdx.x; d < D; d += blockDim.x) ob[(size_t)pos * D + d] = fb[(size_t)s * D + d];
    return;
  }
  const int g = s - T;
  if (g >= n_groups[b]) {
    for (int d = threadIdx.x; d < D; d += blockDim.x) ob[(size_t)(T + g) * D + d] = qemb[d];
    if (threadIdx.x == 0) qpos[(size_t)b * G + g] = T + g;
    return;
  }
  const int st = offsets[(size_t)b * G + g], len = lengths[(size_t)b * G + g];
  const int pos = st + len + g;
  const float inv = 1.f / (float)max(len, 1);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < len; ++r) acc += fb[(size_t)(st + r) * D + d];
    ob[(size_t)pos * D + d] = acc * inv + qemb[d];
  }
  if (threadIdx.x == 0) qpos[(size_t)b * G + g] = pos;
}
// tokens [B*G, D] = rows qpos of x [B, L, D]; zero for padded groups (transformer.py:817-824)
__global__ void __launch_bounds__(128)
agg_gather_kernel(const float* __restrict__ x, const int* __restrict__ qpos, const int* __restrict__ n_groups, int L, int G, int D,
                  float* __restrict__ out) {
  const int g = blockIdx.x, b = blockIdx.y;
  const bool live = g < n_groups[b];
  const float* src = x + ((size_t)b * L + (live ? qpos[(size_t)b * G + g] : 0)) * D;
  float* dst = out + ((size_t)b * G + g) * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) dst[d] = live ? src[d] : 0.f;
}
static inline unsigned ad_grid(long long total) {
  long long g = (total + 255) / 256;
  return (unsigned)(g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g));
}
}  // namespace qb
using namespace qb;

extern "C" int qb_similarity_alignment(const float* h, int64_t B, int64_t T, int32_t D, float threshold, int32_t max_tokens_per_group,
                                       float* sim, int32_t* seg, int32_t* lengths, int32_t* n_groups, void* stream) {
  QB_REQUIRE(h && sim && seg && lengths && n_groups && B >= 1 && T >= 2 && D >= 1, "similarity_alignment: bad args (T >= 2)");
  similarity_alignment_kernel<<<(unsigned)B, 256, 0, (cudaStream_t)stream>>>(h, (int)T, D, threshold, max_tokens_per_group, sim, seg, lengths,
                                                                              n_groups);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int qb_alignment_matrix(const int32_t* seg, int64_t B, int64_t T, int64_t G, float* align, void* stream) {
  QB_REQUIRE(seg && align && G >= 1, "alignment_matrix: bad args");
  const long long total = B * G * T;
  alignment_matrix_kernel<<<ad_grid(total), 256, 0, (cudaStream_t)stream>>>(seg, (int)T, (int)G, align, total);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int qb_pack_lengths(const int64_t* codes, const int32_t* lengths, int64_t B, int32_t nq, int64_t G, int32_t codebook_size,
                               int64_t* out, void* stream) {
  QB_REQUIRE(codes && lengths && out && codebook_size >= 1, "pack_lengths: bad args");
  const long long total = B * nq * G;
  if (!total) return 0;
  pack_lengths_kernel<<<ad_grid(total), 256, 0, (cudaStream_t)stream>>>(codes, lengths, nq, (int)G, codebook_size, out, total);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int qb_unpack_lengths(const int64_t* codes, int64_t B, int32_t nq, int64_t G, int32_t codebook_size, int64_t* plain,
                                 int32_t* lengths, void* stream) {
  QB_REQUIRE(codes && plain && lengths && codebook_size >= 1, "unpack_lengths: bad args");
  const long long total = B * nq * G;
  if (!total) return 0;
  unpack_lengths_kernel<<<ad_grid(total), 256, 0, (cudaStream_t)stream>>>(codes, nq, (int)G, codebook_size, plain, lengths, total);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int qb_length_offsets(const int32_t* lengths, int64_t B, int64_t G, int32_t* offsets, int32_t* totals, void* stream) {
  QB_REQUIRE(lengths && offsets && totals, "length_offsets: bad args");
  length_offsets_kernel<<<(unsigned)B, 32, 0, (cudaStream_t)stream>>>(lengths, (int)G, offsets, totals);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int qb_deaggregate(const void* x, int32_t elem_bytes, const int32_t* lengths, const int32_t* offsets, int64_t B, int64_t C,
                              int64_t G, int64_t T_out, void* out, void* stream) {
  QB_REQUIRE(x && lengths && offsets && out && (elem_bytes == 4 || elem_bytes == 8), "deaggregate: bad args (4- or 8-byte elements)");
  const long long total = B * C * G;
  if (!total) return 0;
  QB_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)B * C * T_out * elem_bytes, (cudaStream_t)stream));
  if (elem_bytes == 4)
    deaggregate_kernel<float><<<ad_grid(total), 256, 0, (cudaStream_t)stream>>>((const float*)x, lengths, offsets, (int)C, (int)G, (int)T_out,
                                                                               (float*)out, total);
  else
    deaggregate_kernel<int64_t><<<ad_grid(total), 256, 0, (cudaStream_t)stream>>>((const int64_t*)x, lengths, offsets, (int)C, (int)G,
                                                                                 (int)T_out, (int64_t*)out, total);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_agg_interleave(const float* feats, const int32_t* seg, const int32_t* lengths, const int32_t* offsets,
                                 const int32_t* n_groups, const float* query_embedding, int64_t B, int64_t T, int64_t G, int32_t D,
                                 float* out, int32_t* qpos, void* stream) {
  QB_REQUIRE(feats && seg && lengths && offsets && n_groups && query_embedding && out && qpos && B >= 1 && T >= 1 && G >= 1 && D >= 1,
             "agg_interleave: bad args");
  agg_interleave_kernel<<<dim3((unsigned)(T + G), (unsigned)B), 128, 0, (cudaStream_t)stream>>>(feats, seg, lengths, offsets, n_groups,
                                                                                               query_embedding, (int)T, (int)G, D, out, qpos);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int qb_agg_gather(const float* x, const int32_t* qpos, const int32_t* n_groups, int64_t B, int64_t L, int64_t G, int32_t D,
                             float* out, void* stream) {
  QB_REQUIRE(x && qpos && n_groups && out && B >= 1 && G >= 1 && L >= G && D >= 1, "agg_gather: bad args");
  agg_gather_kernel<<<dim3((unsigned)G, (unsigned)B), 128, 0, (cudaStream_t)stream>>>(x, qpos, n_groups, (int)L, (int)G, D, out);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
