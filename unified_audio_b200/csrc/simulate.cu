// UniSE's training-data simulation (QuarkAudio-UniSE/dataloader/simulation/simulate.py:10-192, rir_utils.py:340-517,
// detect_non_silence.py:1-98, dataloader/data_module.py:106-140,217-233) on packed ragged rows: one concatenated fp32 buffer per
// signal and int64 row offsets [rows + 1], so utterances of any lengths share each launch.  Every random parameter is drawn on
// the host (unified_audio_b200/simulate.py) and arrives as per-row arrays; a row whose stage is off is skipped (or copied, for the
// out-of-place convolution).  Every reduction runs in a fixed order with fp64 partials and there are no floating-point atomics,
// so a batch is bit-reproducible.
#include <atomic>
#include <cmath>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

#define QB_SIM_LAUNCHED(n)           \
  g_launches += (n);                 \
  QB_CHECK_CUDA(cudaGetLastError()); \
  return 0

constexpr int SIM_FRAME = 1024, SIM_SHIFT = 512;
constexpr int RT = 1024;                       // threads of the one-block-per-row kernels
constexpr int EW = 256, EW_PER = 4;            // elementwise kernels: 256 threads x 4 samples per block and row

// ------------------------------------------------------------------------------------------ fixed-order block reductions
template <int NT>
__device__ double block_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = NT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

template <int NT>
__device__ float block_max(float v, float* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = NT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] = fmaxf(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  const float r = sh[0];
  __syncthreads();
  return r;
}

template <int NT>
__device__ long long block_min_ll(long long v, long long* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = NT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] = min(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  const long long r = sh[0];
  __syncthreads();
  return r;
}

// ------------------------------------------------------------------------------------------ 1. non-silence detection, active RMS
// power[frame_off[r] + f] = variance of x_r[512 f .. 512 f + 1023] (zero past the row's end: framing(padded=True)), fp64, two-pass.
__global__ void frame_power_kernel(const float* __restrict__ x, const int64_t* __restrict__ offs, const int64_t* __restrict__ frame_off,
                                   double* __restrict__ power) {
  __shared__ double sh[256];
  const int r = blockIdx.y;
  const long long f = blockIdx.x;
  if (f >= frame_off[r + 1] - frame_off[r]) return;
  const float* xr = x + offs[r];
  const long long L = offs[r + 1] - offs[r], s0 = f * SIM_SHIFT;
  float v[4];
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long n = s0 + threadIdx.x + 256 * j;
    v[j] = n < L ? xr[n] : 0.f;
    s += v[j];
  }
  const double mean = block_sum<256>(s, sh) / SIM_FRAME;
  double q = 0.0;
#pragma unroll
  for (int j = 0; j < 4; ++j) q += (v[j] - mean) * (v[j] - mean);
  q = block_sum<256>(q, sh);
  if (threadIdx.x == 0) power[frame_off[r] + f] = q / SIM_FRAME;
}

// rms[r] = std of x_r over its non-silent samples (frames with power / mean power > 0.01, one flag per 512-sample shift, the last
// flag repeated to the end); rows shorter than a frame or of zero mean power count every sample.  mask (optional) = the flags.
__global__ void active_rms_kernel(const float* __restrict__ x, const int64_t* __restrict__ offs, const int64_t* __restrict__ frame_off,
                                  const double* __restrict__ power, double* __restrict__ rms, uint8_t* __restrict__ mask) {
  extern __shared__ uint8_t flags[];
  __shared__ double sh[RT];
  const int r = blockIdx.x;
  const float* xr = x + offs[r];
  const long long L = offs[r + 1] - offs[r], F = frame_off[r + 1] - frame_off[r];
  const double* pr = power + frame_off[r];
  double s = 0.0;
  for (long long f = threadIdx.x; f < F; f += RT) s += pr[f];
  const double mean = F > 0 ? block_sum<RT>(s, sh) / F : 0.0;
  const bool all = F == 0 || mean == 0.0;
  for (long long f = threadIdx.x; f < F; f += RT) flags[f] = all ? 1 : (pr[f] / mean > 0.01);
  __syncthreads();
  auto on = [&](long long n) -> bool { return all || flags[min(n / SIM_SHIFT, F - 1)]; };
  double c = 0.0;
  s = 0.0;
  for (long long n = threadIdx.x; n < L; n += RT)
    if (on(n)) { s += xr[n]; c += 1.0; }
  const double cnt = block_sum<RT>(c, sh), mu = block_sum<RT>(s, sh) / cnt;
  double q = 0.0;
  for (long long n = threadIdx.x; n < L; n += RT) {
    const bool k = on(n);
    if (k) q += (xr[n] - mu) * (xr[n] - mu);
    if (mask) mask[offs[r] + n] = k;
  }
  q = block_sum<RT>(q, sh);
  if (threadIdx.x == 0) rms[r] = sqrt(q / cnt);
}

// ------------------------------------------------------------------------------------------ 2. placement and mixing
// dst_r[n] = src_r[(n + shift[r]) mod len(src_r)] for n < len(dst_r): np.pad(mode="wrap") from an offset, or a cut at an offset.
__global__ void place_kernel(const float* __restrict__ src, const int64_t* __restrict__ src_offs, const int64_t* __restrict__ offs,
                             const int64_t* __restrict__ shift, float* __restrict__ dst) {
  const int r = blockIdx.y;
  const long long L = offs[r + 1] - offs[r], Ls = src_offs[r + 1] - src_offs[r];
  for (long long n = (long long)blockIdx.x * EW * EW_PER + threadIdx.x, e = min(L, n + EW * EW_PER); n < e; n += EW)
    dst[offs[r] + n] = Ls > 0 ? src[src_offs[r] + (n + shift[r]) % Ls] : 0.f;
}

// rows with on[r]: x = other * (10^(-snr/20) rms_x / (rms_o + 1e-10)) + x; diff (optional) = the added part (noisy - speech).
__global__ void mix_kernel(float* __restrict__ x, const float* __restrict__ other, const int64_t* __restrict__ offs,
                           const double* __restrict__ snr, const double* __restrict__ rms_x, const double* __restrict__ rms_o,
                           const int32_t* __restrict__ on, float* __restrict__ diff) {
  const int r = blockIdx.y;
  if (!on[r]) return;
  const long long L = offs[r + 1] - offs[r];
  const float scale = (float)(pow(10.0, -snr[r] / 20.0) * rms_x[r] / (rms_o[r] + 1e-10));
  for (long long n = (long long)blockIdx.x * EW * EW_PER + threadIdx.x, e = min(L, n + EW * EW_PER); n < e; n += EW) {
    const long long i = offs[r] + n;
    const float s = x[i], y = __fadd_rn(__fmul_rn(other[i], scale), s);
    x[i] = y;
    if (diff) diff[i] = __fsub_rn(y, s);
  }
}

// ------------------------------------------------------------------------------------------ 3. RIR normalisation, early window
// hn = h / (max|h| + 1e-5); p = first argmax |hn|; thr = 0.1 |hn[p]|; win = [first k <= p with |hn[k]| > thr, first k > p with
// |hn[k]| < thr, else p + 1).  status[r] = 1 when the peak is the last sample (get_rir_start_sample has no tail to search).
__global__ void rir_prep_kernel(const float* __restrict__ h, const int64_t* __restrict__ offs, const int32_t* __restrict__ on,
                                float* __restrict__ hn, int64_t* __restrict__ win, int32_t* __restrict__ status) {
  __shared__ float shf[RT];
  __shared__ long long shl[RT];
  const int r = blockIdx.x;
  if (!on[r]) {
    if (threadIdx.x == 0) status[r] = 0;
    return;
  }
  const float* hr = h + offs[r];
  float* out = hn + offs[r];
  const long long K = offs[r + 1] - offs[r];
  float m = 0.f;
  for (long long k = threadIdx.x; k < K; k += RT) m = fmaxf(m, fabsf(hr[k]));
  const float d = __fadd_rn(block_max<RT>(m, shf), 1e-5f);
  m = -1.f;
  for (long long k = threadIdx.x; k < K; k += RT) {
    const float v = __fdiv_rn(hr[k], d);
    out[k] = v;
    m = fmaxf(m, fabsf(v));
  }
  const float peak = block_max<RT>(m, shf);
  long long first = K;
  for (long long k = threadIdx.x; k < K; k += RT)
    if (fabsf(out[k]) == peak) { first = k; break; }
  const long long p = block_min_ll<RT>(first, shl);
  const float thr = __fmul_rn(0.1f, peak);
  long long s = K, e = K;
  for (long long k = threadIdx.x; k <= p; k += RT)
    if (fabsf(out[k]) > thr) { s = k; break; }
  for (long long k = p + 1 + threadIdx.x; k < K; k += RT)
    if (fabsf(out[k]) < thr) { e = k; break; }
  s = block_min_ll<RT>(s, shl);
  e = block_min_ll<RT>(e, shl);
  if (threadIdx.x == 0) {
    win[2 * r] = s == K ? 0 : s;     // np.argmax of an all-False array is 0
    win[2 * r + 1] = e == K ? p + 1 : e;
    status[r] = p == K - 1;
  }
}

// ------------------------------------------------------------------------------------------ 4. truncated full convolution
// y_r[n] = sum_{k0 <= k < k1} h_r[k] x_r[n - k] for n < len(x_r) (k1 - k0 = the whole RIR, or its early window); rows off: y = x.
// Block: 1024 outputs of one row; taps in tiles of 256 staged with the x segment they meet in shared memory; each tile's 256
// products sum in fp32, the tiles in fp64.
constexpr int CV_OUT = 1024, CV_TAPS = 256;
__global__ void __launch_bounds__(256) convolve_kernel(const float* __restrict__ x, const int64_t* __restrict__ offs,
                                                       const float* __restrict__ h, const int64_t* __restrict__ h_offs,
                                                       const int64_t* __restrict__ win, const int32_t* __restrict__ on,
                                                       float* __restrict__ y) {
  __shared__ float seg[CV_OUT + CV_TAPS];
  __shared__ float tap[CV_TAPS];
  const int r = blockIdx.y;
  const long long L = offs[r + 1] - offs[r], n0 = (long long)blockIdx.x * CV_OUT;
  if (n0 >= L) return;
  const float* xr = x + offs[r];
  float* yr = y + offs[r];
  if (!on[r]) {
    for (long long n = n0 + threadIdx.x; n < min(L, n0 + CV_OUT); n += 256) yr[n] = xr[n];
    return;
  }
  const float* hr = h + h_offs[r];
  const long long K = h_offs[r + 1] - h_offs[r];
  const long long k0 = win ? win[2 * r] : 0, k1 = win ? win[2 * r + 1] : K;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long kt = k0; kt < k1 && kt <= n0 + CV_OUT - 1; kt += CV_TAPS) {
    __syncthreads();
    const long long base = n0 - kt - (CV_TAPS - 1);
    for (int i = threadIdx.x; i < CV_OUT + CV_TAPS - 1; i += 256) {
      const long long n = base + i;
      seg[i] = (n >= 0 && n < L) ? xr[n] : 0.f;
    }
    tap[threadIdx.x] = kt + threadIdx.x < k1 ? hr[kt + threadIdx.x] : 0.f;
    __syncthreads();
    float a[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
    for (int t = 0; t < CV_TAPS; ++t) {
      const float w = tap[t];
#pragma unroll
      for (int j = 0; j < 4; ++j) a[j] = fmaf(w, seg[threadIdx.x + 256 * j + CV_TAPS - 1 - t], a[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] += a[j];
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long n = n0 + threadIdx.x + 256 * j;
    if (n < L) yr[n] = (float)acc[j];
  }
}

// ------------------------------------------------------------------------------------------ 5. bandwidth limitation
// torchaudio sinc_interp_hann (unified_audio_b200.ssl.resample_kernel taps): 16 kHz -> fs_new keeps y[m] = sum_i kd[i] xpad[o m + i]
// (xpad = `wd` zeros, x, zeros; m < ceil(L / o)), then fs_new -> 16 kHz gives z[o m + j] = sum_i ku[j][i] ypad[m + i], cut to L.
struct ResampleTaps {
  const float* down[2];   // [kd] for o = 4 (fs_new 4000) and o = 2 (8000)
  const float* up[2];     // [o, ku]
  int kd[2], wd[2], ku, wu;
};

__global__ void resample_down_kernel(const float* __restrict__ x, const int64_t* __restrict__ offs, const int32_t* __restrict__ fs_new,
                                     const int32_t* __restrict__ on, ResampleTaps t, float* __restrict__ tmp) {
  const int r = blockIdx.y;
  if (!on[r] || fs_new[r] == 16000) return;
  const bool four = fs_new[r] == 4000;
  const int o = four ? 4 : 2, K = four ? t.kd[0] : t.kd[1], W = four ? t.wd[0] : t.wd[1];
  const float* k = four ? t.down[0] : t.down[1];
  const long long L = offs[r + 1] - offs[r], Ld = (L + o - 1) / o;
  const float* xr = x + offs[r];
  for (long long m = (long long)blockIdx.x * EW * EW_PER + threadIdx.x, e = min(Ld, m + EW * EW_PER); m < e; m += EW) {
    float a = 0.f;
    for (int i = 0; i < K; ++i) {
      const long long n = o * m + i - W;
      if (n >= 0 && n < L) a = fmaf(k[i], xr[n], a);
    }
    tmp[offs[r] + m] = a;
  }
}

__global__ void resample_up_kernel(float* __restrict__ x, const int64_t* __restrict__ offs, const int32_t* __restrict__ fs_new,
                                   const int32_t* __restrict__ on, ResampleTaps t, const float* __restrict__ tmp) {
  const int r = blockIdx.y;
  if (!on[r] || fs_new[r] == 16000) return;
  const bool four = fs_new[r] == 4000;
  const int o = four ? 4 : 2;
  const float* k = four ? t.up[0] : t.up[1];
  const long long L = offs[r + 1] - offs[r], Ld = (L + o - 1) / o;
  const float* yr = tmp + offs[r];
  for (long long n = (long long)blockIdx.x * EW * EW_PER + threadIdx.x, e = min(L, n + EW * EW_PER); n < e; n += EW) {
    const long long m = n / o;
    const float* kj = k + (n % o) * t.ku;
    float a = 0.f;
    for (int i = 0; i < t.ku; ++i) {
      const long long q = m + i - t.wu;
      if (q >= 0 && q < Ld) a = fmaf(kj[i], yr[q], a);
    }
    x[offs[r] + n] = a;
  }
}

// ------------------------------------------------------------------------------------------ 6. clipping
// np.quantile(x, [q0, q1]) 'linear': order statistics of ranks floor(v), floor(v) + 1 (v = (L - 1) q; both L - 1 when v >= L - 1),
// selected exactly by a 4-pass 8-bit radix select over order-preserving uint32 keys; one block per (row, statistic).
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__device__ __forceinline__ void quantile_ranks(long long L, double q, long long& lo, long long& hi, double& gamma) {
  const double v = (double)(L - 1) * q;
  if (v >= (double)(L - 1)) {
    lo = hi = L - 1;
    gamma = v + 1.0;          // numpy: v - (-1); a == b makes it immaterial
  } else {
    lo = (long long)floor(v);
    hi = lo + 1;
    gamma = v - floor(v);
  }
}

__global__ void order_stat_kernel(const float* __restrict__ x, const int64_t* __restrict__ offs, const double* __restrict__ q,
                                  const int32_t* __restrict__ on, float* __restrict__ stats) {
  __shared__ unsigned int hist[256];
  __shared__ uint32_t s_prefix;
  __shared__ long long s_rank;
  const int r = blockIdx.y, s = blockIdx.x;   // s: 0/1 = the two ranks of q0, 2/3 = of q1
  if (!on[r]) return;
  const float* xr = x + offs[r];
  const long long L = offs[r + 1] - offs[r];
  long long lo, hi;
  double g;
  quantile_ranks(L, q[2 * r + (s >> 1)], lo, hi, g);
  if (threadIdx.x == 0) {
    s_prefix = 0;
    s_rank = (s & 1) ? hi : lo;
  }
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const uint32_t mask = pass == 0 ? 0u : (0xffffffffu << (32 - 8 * pass));
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (long long n = threadIdx.x; n < L; n += blockDim.x) {
      const uint32_t k = f2key(xr[n]);
      if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      long long rank = s_rank;
      int b = 0;
      while (rank >= (long long)hist[b]) rank -= hist[b++];
      s_rank = rank;
      s_prefix = prefix | ((uint32_t)b << shift);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) stats[4 * r + s] = key2f(s_prefix);
}

// numpy _lerp in fp64 from the float32 neighbours: d = b - a (fp32); t < 0.5 ? a + d t : b - d (1 - t)
__device__ __forceinline__ double np_lerp(float a, float b, double t) {
  const double d = (double)__fsub_rn(b, a);
  return t >= 0.5 ? (double)b - d * (1.0 - t) : (double)a + d * t;
}

__global__ void clip_kernel(float* __restrict__ x, const int64_t* __restrict__ offs, const double* __restrict__ q,
                            const int32_t* __restrict__ on, const float* __restrict__ stats) {
  const int r = blockIdx.y;
  if (!on[r]) return;
  const long long L = offs[r + 1] - offs[r];
  long long a, b;
  double g0, g1;
  quantile_ranks(L, q[2 * r], a, b, g0);
  quantile_ranks(L, q[2 * r + 1], a, b, g1);
  const double lo = np_lerp(stats[4 * r], stats[4 * r + 1], g0), hi = np_lerp(stats[4 * r + 2], stats[4 * r + 3], g1);
  for (long long n = (long long)blockIdx.x * EW * EW_PER + threadIdx.x, e = min(L, n + EW * EW_PER); n < e; n += EW) {
    const long long i = offs[r] + n;
    x[i] = (float)fmin(fmax((double)x[i], lo), hi);
  }
}

// ------------------------------------------------------------------------------------------ 7. packet loss
// one block per lost packet: x_r[p * len .. (p + 1) * len) = 0 (inside the row)
__global__ void packet_loss_kernel(float* __restrict__ x, const int64_t* __restrict__ offs, const int64_t* __restrict__ lost,
                                   const int32_t* __restrict__ lost_row, int packet) {
  const int r = lost_row[blockIdx.x];
  const long long L = offs[r + 1] - offs[r], s = lost[blockIdx.x] * packet;
  for (long long n = s + threadIdx.x; n < min(L, s + packet); n += blockDim.x) x[offs[r] + n] = 0.f;
}

// ------------------------------------------------------------------------------------------ 9. peak rule, cut, normalisation
// One block per row.  m = max(|noisy|, |speech|, |interf|) over the row; above 0.99 every signal becomes v / m * 0.99.  The cut
// (offset cut_off[r], or wrap padding when cut_off < 0) goes straight to the [rows, cut] outputs, normalised as normalize_src_tgt
// (no interferer) or normalize_mix_speech_inferf, with the host's uniform draw norm_r[r].  out_interf may be NULL ('se').
__global__ void finish_kernel(const float* __restrict__ noisy, const float* __restrict__ speech, const float* __restrict__ interf,
                              const int64_t* __restrict__ offs, const int32_t* __restrict__ has_interf, const int64_t* __restrict__ cut_off,
                              const double* __restrict__ norm_r, long long C, float* __restrict__ out_mix, float* __restrict__ out_speech,
                              float* __restrict__ out_interf) {
  __shared__ float sh[RT];
  const int r = blockIdx.x;
  const long long L = offs[r + 1] - offs[r], o = cut_off[r];
  const bool hi = has_interf[r];
  const float* sig[3] = {noisy + offs[r], speech + offs[r], hi ? interf + offs[r] : nullptr};
  float m = 0.f;
  for (long long n = threadIdx.x; n < L; n += RT) {
    m = fmaxf(m, fmaxf(fabsf(sig[0][n]), fabsf(sig[1][n])));
    if (hi) m = fmaxf(m, fabsf(sig[2][n]));
  }
  m = block_max<RT>(m, sh);
  const bool scale = m > 0.99f;
  auto val = [&](int c, long long n) -> float {
    const float v = sig[c][o < 0 ? n % L : o + n];
    return scale ? __fmul_rn(__fdiv_rn(v, m), 0.99f) : v;
  };
  float pk[3] = {0.f, 0.f, 0.f};
  for (long long n = threadIdx.x; n < C; n += RT)
    for (int c = 0; c < (hi ? 3 : 2); ++c) pk[c] = fmaxf(pk[c], fabsf(val(c, n)));
  const float a = block_max<RT>(pk[0], sh), b = block_max<RT>(pk[1], sh), c = hi ? block_max<RT>(pk[2], sh) : 0.f;
  float factor;
  if (!hi) {
    const float tgt = __fadd_rn(b, 1e-5f), src = __fadd_rn(a, 1e-5f);
    const float thr = __fdiv_rn(0.99f, fmaxf(tgt, src));
    // the reference's uniform(0.1, 0.99) level, rounded as Python rounds it: product, then sum.  A contracted fma moves the fp32
    // level by an ulp for some norm_r (tests/test_simulation_stages_gpu.py, FMA_NORM_R).
    const float level = (float)__dadd_rn(0.1, __dmul_rn(0.99 - 0.1, norm_r[r]));
    factor = fminf(__fdiv_rn(level, tgt), thr);
  } else {
    factor = __fdiv_rn(0.99f, __fadd_rn(fmaxf(fmaxf(a, b), c), 1e-5f));
    const float least = __fmul_rn(fminf(fminf(a, b), c), factor);
    if (least > 0.1f) {
      const float lo = __fdiv_rn(0.1f, least);
      factor = __fmul_rn(__fadd_rn(lo, __fmul_rn(__fsub_rn(1.f, lo), (float)norm_r[r])), factor);
    }
  }
  for (long long n = threadIdx.x; n < C; n += RT) {
    out_mix[r * C + n] = __fmul_rn(val(0, n), factor);
    out_speech[r * C + n] = __fmul_rn(val(1, n), factor);
    if (hi && out_interf) out_interf[r * C + n] = __fmul_rn(val(2, n), factor);
  }
}

// enrollment: cut at cut_off[r] (wrap padding when < 0) to C samples, then e / (max|e| + 1e-5) * 0.99
__global__ void enroll_kernel(const float* __restrict__ e, const int64_t* __restrict__ offs, const int64_t* __restrict__ cut_off,
                              long long C, float* __restrict__ out) {
  __shared__ float sh[RT];
  const int r = blockIdx.x;
  const long long L = offs[r + 1] - offs[r], o = cut_off[r];
  const float* er = e + offs[r];
  float m = 0.f;
  for (long long n = threadIdx.x; n < C; n += RT) m = fmaxf(m, fabsf(er[o < 0 ? n % L : o + n]));
  const float d = __fadd_rn(block_max<RT>(m, sh), 1e-5f);
  for (long long n = threadIdx.x; n < C; n += RT) out[r * C + n] = __fmul_rn(__fdiv_rn(er[o < 0 ? n % L : o + n], d), 0.99f);
}

static dim3 ew_grid(int64_t max_len, int64_t rows) { return dim3((unsigned)std::max<int64_t>(1, ceil_div(max_len, EW * EW_PER)), (unsigned)rows); }

}  // namespace qb

using namespace qb;

extern "C" int qb_sim_active_rms(const float* x, const int64_t* offs, const int64_t* frame_off, int64_t rows, int64_t max_len,
                                 int64_t max_frames, double* power, double* rms, uint8_t* mask, void* stream) {
  QB_REQUIRE(x && offs && frame_off && power && rms && rows >= 1 && rows <= 65535 && max_len >= 1, "sim_active_rms: bad args");
  QB_REQUIRE(max_frames <= 48 * 1024, "sim_active_rms: rows of more than %d frames", 48 * 1024);
  cudaStream_t st = (cudaStream_t)stream;
  int n = 0;
  if (max_frames > 0) {
    frame_power_kernel<<<dim3((unsigned)max_frames, (unsigned)rows), 256, 0, st>>>(x, offs, frame_off, power);
    ++n;
  }
  active_rms_kernel<<<(unsigned)rows, RT, (size_t)std::max<int64_t>(max_frames, 1), st>>>(x, offs, frame_off, power, rms, mask);
  QB_SIM_LAUNCHED(n + 1);
}

extern "C" int qb_sim_place(const float* src, const int64_t* src_offs, const int64_t* offs, const int64_t* shift, int64_t rows,
                            int64_t max_len, float* dst, void* stream) {
  QB_REQUIRE(src && src_offs && offs && shift && dst && rows >= 1 && rows <= 65535, "sim_place: bad args");
  place_kernel<<<ew_grid(max_len, rows), EW, 0, (cudaStream_t)stream>>>(src, src_offs, offs, shift, dst);
  QB_SIM_LAUNCHED(1);
}

extern "C" int qb_sim_mix(float* x, const float* other, const int64_t* offs, int64_t rows, int64_t max_len, const double* snr,
                          const double* rms_x, const double* rms_other, const int32_t* on, float* diff, void* stream) {
  QB_REQUIRE(x && other && offs && snr && rms_x && rms_other && on && rows >= 1 && rows <= 65535, "sim_mix: bad args");
  mix_kernel<<<ew_grid(max_len, rows), EW, 0, (cudaStream_t)stream>>>(x, other, offs, snr, rms_x, rms_other, on, diff);
  QB_SIM_LAUNCHED(1);
}

extern "C" int qb_sim_rir_prep(const float* h, const int64_t* offs, int64_t rows, const int32_t* on, float* hn, int64_t* win,
                               int32_t* status, void* stream) {
  QB_REQUIRE(h && offs && on && hn && win && status && rows >= 1, "sim_rir_prep: bad args");
  rir_prep_kernel<<<(unsigned)rows, RT, 0, (cudaStream_t)stream>>>(h, offs, on, hn, win, status);
  QB_SIM_LAUNCHED(1);
}

extern "C" int qb_sim_convolve(const float* x, const int64_t* offs, int64_t rows, int64_t max_len, const float* h, const int64_t* h_offs,
                               const int64_t* win, const int32_t* on, float* y, void* stream) {
  QB_REQUIRE(x && offs && h && h_offs && on && y && x != y && rows >= 1 && rows <= 65535 && max_len >= 1, "sim_convolve: bad args");
  convolve_kernel<<<dim3((unsigned)ceil_div(max_len, CV_OUT), (unsigned)rows), 256, 0, (cudaStream_t)stream>>>(x, offs, h, h_offs, win,
                                                                                                                on, y);
  QB_SIM_LAUNCHED(1);
}

extern "C" int qb_sim_bandwidth(float* x, const int64_t* offs, int64_t rows, int64_t max_len, const int32_t* fs_new, const int32_t* on,
                                const float* down4, const float* down2, int32_t kd4, int32_t wd4, int32_t kd2, int32_t wd2,
                                const float* up4, const float* up2, int32_t ku, int32_t wu, float* tmp, void* stream) {
  QB_REQUIRE(x && offs && fs_new && on && down4 && down2 && up4 && up2 && tmp && rows >= 1 && rows <= 65535, "sim_bandwidth: bad args");
  ResampleTaps t{{down4, down2}, {up4, up2}, {kd4, kd2}, {wd4, wd2}, ku, wu};
  cudaStream_t st = (cudaStream_t)stream;
  resample_down_kernel<<<ew_grid(ceil_div(max_len, 2), rows), EW, 0, st>>>(x, offs, fs_new, on, t, tmp);
  resample_up_kernel<<<ew_grid(max_len, rows), EW, 0, st>>>(x, offs, fs_new, on, t, tmp);
  QB_SIM_LAUNCHED(2);
}

extern "C" int qb_sim_clip(float* x, const int64_t* offs, int64_t rows, int64_t max_len, const double* q, const int32_t* on, float* stats,
                           void* stream) {
  QB_REQUIRE(x && offs && q && on && stats && rows >= 1 && rows <= 65535, "sim_clip: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  order_stat_kernel<<<dim3(4, (unsigned)rows), 1024, 0, st>>>(x, offs, q, on, stats);
  clip_kernel<<<ew_grid(max_len, rows), EW, 0, st>>>(x, offs, q, on, stats);
  QB_SIM_LAUNCHED(2);
}

extern "C" int qb_sim_packet_loss(float* x, const int64_t* offs, const int64_t* lost, const int32_t* lost_row, int64_t n_lost,
                                  int32_t packet, void* stream) {
  QB_REQUIRE(x && offs && lost && lost_row && n_lost >= 1 && n_lost < (1ll << 31) && packet >= 1, "sim_packet_loss: bad args");
  packet_loss_kernel<<<(unsigned)n_lost, 320, 0, (cudaStream_t)stream>>>(x, offs, lost, lost_row, packet);
  QB_SIM_LAUNCHED(1);
}

extern "C" int qb_sim_finish(const float* noisy, const float* speech, const float* interf, const int64_t* offs, int64_t rows,
                             const int32_t* has_interf, const int64_t* cut_off, const double* norm_r, int64_t cut, float* out_mix,
                             float* out_speech, float* out_interf, void* stream) {
  QB_REQUIRE(noisy && speech && offs && has_interf && cut_off && norm_r && out_mix && out_speech && rows >= 1 && cut >= 1,
             "sim_finish: bad args");
  finish_kernel<<<(unsigned)rows, RT, 0, (cudaStream_t)stream>>>(noisy, speech, interf, offs, has_interf, cut_off, norm_r, cut, out_mix,
                                                                 out_speech, out_interf);
  QB_SIM_LAUNCHED(1);
}

extern "C" int qb_sim_enroll(const float* e, const int64_t* offs, int64_t rows, const int64_t* cut_off, int64_t cut, float* out,
                             void* stream) {
  QB_REQUIRE(e && offs && cut_off && out && rows >= 1 && cut >= 1, "sim_enroll: bad args");
  enroll_kernel<<<(unsigned)rows, RT, 0, (cudaStream_t)stream>>>(e, offs, cut_off, cut, out);
  QB_SIM_LAUNCHED(1);
}
