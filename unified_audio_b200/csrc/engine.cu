// Handle-level engine of libquark_b200 (include/quark_b200.h "Handle-level contract", SURVEY.md 8b).
//
// qb_codec_*: H-Codec-2.0 `Codec.encode` / `Codec.decode` (QuarkAudio-HCodec/HCodec-2.0/vq/codec.py:75-99) as ONE C call each:
// the handle owns the repacked weights (fp16 planes, conv taps, interleaved SwiGLU rows, LSTM unit-major slices, DFT matrices
// built in fp64), the zero-padded channel-last workspace and the RoPE tables; the call enqueues ~340 kernels of this library on the
// caller's stream.  qb_rvq_*: the two residual quantisers row-level.
// Host code only orchestrates: every arithmetic op is one of the op-level kernels behind the same header.
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "quark_b200.h"

namespace qb {
extern std::atomic<long long> g_launches;

#define QB_TRY(expr)            \
  do {                          \
    if (int _e = (expr)) return _e; \
  } while (0)

struct PlanesD {
  __half* hi = nullptr;
  __half* lo = nullptr;
};

// device allocations owned by a handle (freed with it)
struct Arena {
  std::vector<void*> ptrs;
  int alloc(void** out, size_t bytes, bool zero) {
    void* p = nullptr;
    if (bytes == 0) bytes = 16;
    QB_CHECK_CUDA(cudaMalloc(&p, bytes));
    if (zero) QB_CHECK_CUDA(cudaMemset(p, 0, bytes));
    ptrs.push_back(p);
    *out = p;
    return 0;
  }
  ~Arena() {
    for (void* p : ptrs) cudaFree(p);
  }
};

// named, size-keyed workspace: allocated (zeroed) on first use - the first call of a shape is the warm-up, later calls and
// CUDA-graph captures only reuse.  The padded channel-last buffers (`padded`) hold clips of rows_per_batch rows whose zero pad
// rows no kernel writes: they are keyed by (B, rows_per_batch, ld, split) as well, so a buffer is only reused by calls that put
// their pad rows in the same places and the pads, zeroed at allocation, stay zero.  A size key alone would hand a buffer to a
// call of another (B, rows_per_batch) with the same product, whose pad rows hold the earlier call's activations.
struct Workspace {
  Arena arena;
  std::map<std::string, void*> bufs;
  int get(void** out, const std::string& name, size_t bytes) {
    const std::string key = name + ":" + std::to_string(bytes);
    auto it = bufs.find(key);
    if (it != bufs.end()) { *out = it->second; return 0; }
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    (void)cs;
    void* p = nullptr;
    QB_TRY(arena.alloc(&p, bytes, true));
    bufs[key] = p;
    *out = p;
    return 0;
  }
  int f32(float** out, const std::string& name, size_t n) { return get((void**)out, name, n * 4); }
  int planes(PlanesD* out, const std::string& name, size_t n, bool split) {
    QB_TRY(get((void**)&out->hi, name + ".hi", n * 2));
    out->lo = nullptr;
    if (split) QB_TRY(get((void**)&out->lo, name + ".lo", n * 2));
    return 0;
  }
  // planes [B, rows_per_batch, ld] with zero pad rows, keyed by their row layout
  int padded(PlanesD* out, const std::string& name, int64_t B, int64_t rpb, int64_t ld, bool split) {
    const std::string key = name + "[" + std::to_string(B) + "x" + std::to_string(rpb) + "x" + std::to_string(ld) + (split ? "s]" : "]");
    return planes(out, key, (size_t)(B * rpb * ld), split);
  }
};

static inline int64_t pad_to(int64_t n, int64_t m) { return (n + m - 1) / m * m; }

// ------------------------------------------------------------------ load-time repack kernels
// conv weight [Cout, Cin, k] fp32 -> [Cout, k, Cpad] planes (tap-major rows of the TMA-im2col GEMM; zero channel pad)
__global__ void repack_conv_kernel(const float* __restrict__ w, int Cout, int Cin, int k, int Cpad, __half* __restrict__ hi,
                                   __half* __restrict__ lo) {
  const long long total = (long long)Cout * k * Cpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int t = (int)((i / Cpad) % k);
    const int co = (int)(i / ((long long)Cpad * k));
    const float v = c < Cin ? w[((long long)co * Cin + c) * k + t] : 0.f;
    __half h, l;
    split_f16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}
// ConvTranspose1d weight [Cin, Cout, k], stride s -> phase GEMM weight [s * Cout, J * Cpad] planes (J = ceil(k / s) taps): row
// (r, co), tap t holds w[:, co, r + (J-1-t) * s] (zero beyond k and in the channel pad) - ops.convt_planes, same layout
__global__ void repack_convt_kernel(const float* __restrict__ w, int Cin, int Cout, int k, int s, int J, int Cpad,
                                    __half* __restrict__ hi, __half* __restrict__ lo) {
  const long long total = (long long)s * Cout * J * Cpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int t = (int)((i / Cpad) % J);
    const long long row = i / ((long long)Cpad * J);
    const int co = (int)(row % Cout), r = (int)(row / Cout);
    const int j = r + (J - 1 - t) * s;
    const float v = (c < Cin && j < k) ? w[((long long)c * Cout + co) * k + j] : 0.f;
    __half h, l;
    split_f16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}
// rows of a and b interleaved: out[2j] = a[j], out[2j+1] = b[j]  (SwiGLU gate/up pairs)
__global__ void interleave_rows_kernel(const float* __restrict__ a, const float* __restrict__ b, long long rows, int cols,
                                       float* __restrict__ out) {
  const long long total = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i % cols);
    out[(2 * r) * cols + c] = a[i];
    out[(2 * r + 1) * cols + c] = b[i];
  }
}
// W_hh [4H, H] gate-major (i|f|g|o) -> fp16 [H/U][4U][H]: row 4j+g of slice c = gate g of unit c*U+j (lstm_tc.cu)
__global__ void lstm_permute_kernel(const float* __restrict__ w, int H, int U, __half* __restrict__ out) {
  const long long total = 4LL * H * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % H);
    const long long row = i / H;                 // c*4U + 4j + g
    const int c = (int)(row / (4 * U)), r = (int)(row % (4 * U)), j = r >> 2, g = r & 3;
    out[i] = f2h_sat(w[((long long)g * H + c * U + j) * H + k]);
  }
}
__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}
// RVQ search constants in fp64: consts[q*K + j] = -|e_qj|^2 / 2, then K values of -2; e2 per code for the host max
__global__ void rvq_consts_kernel(const float* __restrict__ cb, int nq, int K, int D, float* __restrict__ consts, float* __restrict__ e2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq * K) {
    double s = 0.0;
    for (int d = 0; d < D; ++d) { const double v = cb[(long long)i * D + d]; s += v * v; }
    consts[i] = (float)(-0.5 * s);
    e2[i] = (float)s;
  }
  if (i < K) consts[(long long)nq * K + i] = -2.0f;
}
__global__ void gather_rows_kernel(const float* __restrict__ table, const int64_t* __restrict__ ids, long long rows, int cols,
                                   float* __restrict__ out) {
  const long long total = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    out[i] = table[ids[i / cols] * cols + i % cols];
}
// [B*N, nq] <-> [B, nq, N] int64 (the reference returns codes transposed, vq/codec.py:85-86)
__global__ void codes_rows_to_bqn_kernel(const int64_t* __restrict__ rows, int B, int N, int nq, int64_t* __restrict__ out) {
  const long long total = (long long)B * N * nq;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i % N), q = (int)((i / N) % nq), b = (int)(i / ((long long)N * nq));
    out[i] = rows[((long long)b * N + n) * nq + q];
  }
}
__global__ void codes_bqn_to_rows_kernel(const int64_t* __restrict__ bqn, int B, int N, int nq, int64_t* __restrict__ rows) {
  const long long total = (long long)B * N * nq;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % nq), n = (int)((i / nq) % N), b = (int)(i / ((long long)N * nq));
    rows[i] = bqn[((long long)b * nq + q) * N + n];
  }
}
// debug taps of plane buffers: out[b, r, c] = hi + lo of row (row_off + r) of a padded [B, rows_per_batch, ld] plane buffer
__global__ void planes_to_f32_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, long long B, long long rows, int C,
                                     long long ld, long long rpb, long long row_off, float* __restrict__ out) {
  const long long total = B * rows * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = (i / C) % rows, b = i / ((long long)C * rows);
    const long long o = (b * rpb + row_off + r) * ld + c;
    out[i] = __half2float(hi[o]) + (lo ? __half2float(lo[o]) : 0.f);
  }
}
static inline unsigned grid_for(long long total) {
  long long g = (total + 255) / 256;
  return (unsigned)(g < 1 ? 1 : (g > 132 * 32 ? 132 * 32 : g));
}

// ------------------------------------------------------------------ weights
struct WeightTable {
  std::unordered_map<std::string, const qb_tensor*> map;
  int init(const qb_tensor* t, int n) {
    for (int i = 0; i < n; ++i) {
      QB_REQUIRE(t[i].name && t[i].data, "load: tensor %d has a null name / pointer", i);
      map[t[i].name] = &t[i];
    }
    return 0;
  }
  const qb_tensor* find(const std::string& k) const {
    auto it = map.find(k);
    return it == map.end() ? nullptr : it->second;
  }
};
static long long numel(const qb_tensor* t) {
  long long n = 1;
  for (int i = 0; i < t->ndim; ++i) n *= t->shape[i];
  return n;
}

struct Loader {
  const WeightTable& wt;
  Arena& arena;
  Loader(const WeightTable& w, Arena& a) : wt(w), arena(a) {}
  int get(const qb_tensor** out, const std::string& key, int ndim) {
    const qb_tensor* t = wt.find(key);
    QB_REQUIRE(t != nullptr, "load: missing weight '%s'", key.c_str());
    QB_REQUIRE(t->ndim == ndim, "load: weight '%s' has %d dims, expected %d", key.c_str(), t->ndim, ndim);
    *out = t;
    return 0;
  }
  // fp32 vector copied into the arena (the caller may free its state-dict after load)
  int f32(const float** out, const std::string& key) {
    const qb_tensor* t = wt.find(key);
    QB_REQUIRE(t != nullptr, "load: missing weight '%s'", key.c_str());
    void* p;
    QB_TRY(arena.alloc(&p, (size_t)numel(t) * 4, false));
    QB_CHECK_CUDA(cudaMemcpy(p, t->data, (size_t)numel(t) * 4, cudaMemcpyDeviceToDevice));
    *out = (const float*)p;
    return 0;
  }
  int planes_from(PlanesD* out, const float* src, long long n, bool split) {
    QB_TRY(arena.alloc((void**)&out->hi, (size_t)n * 2, false));
    out->lo = nullptr;
    if (split) QB_TRY(arena.alloc((void**)&out->lo, (size_t)n * 2, false));
    return qb_split_f16(src, (qb_half*)out->hi, (qb_half*)out->lo, n, nullptr);
  }
  int lin(PlanesD* out, const std::string& key, bool split) {
    const qb_tensor* t;
    QB_TRY(get(&t, key, 2));
    return planes_from(out, t->data, numel(t), split);
  }
  int conv(PlanesD* out, const std::string& key, bool split, int* k_out = nullptr) {
    const qb_tensor* t;
    QB_TRY(get(&t, key, 3));
    const int Cout = (int)t->shape[0], Cin = (int)t->shape[1], k = (int)t->shape[2], Cpad = (int)pad_to(Cin, 64);
    const long long n = (long long)Cout * k * Cpad;
    QB_TRY(arena.alloc((void**)&out->hi, (size_t)n * 2, false));
    out->lo = nullptr;
    if (split) QB_TRY(arena.alloc((void**)&out->lo, (size_t)n * 2, false));
    repack_conv_kernel<<<grid_for(n), 256>>>(t->data, Cout, Cin, k, Cpad, out->hi, out->lo);
    QB_CHECK_CUDA(cudaGetLastError());
    if (k_out) *k_out = k;
    return 0;
  }
  // host fp64 matrix -> planes (DFT matrices: hi = rn16(w), lo = rn16(w - hi))
  int planes_from_f64(PlanesD* out, const std::vector<double>& w) {
    std::vector<__half> hi(w.size()), lo(w.size());
    for (size_t i = 0; i < w.size(); ++i) {
      double v = w[i];
      v = v > 65504.0 ? 65504.0 : (v < -65504.0 ? -65504.0 : v);
      hi[i] = __double2half(v);
      lo[i] = __double2half(v - (double)__half2float(hi[i]));
    }
    QB_TRY(arena.alloc((void**)&out->hi, w.size() * 2, false));
    QB_TRY(arena.alloc((void**)&out->lo, w.size() * 2, false));
    QB_CHECK_CUDA(cudaMemcpy(out->hi, hi.data(), w.size() * 2, cudaMemcpyHostToDevice));
    QB_CHECK_CUDA(cudaMemcpy(out->lo, lo.data(), w.size() * 2, cudaMemcpyHostToDevice));
    return 0;
  }
};

struct ConvNeXtW {
  const float *dw_w, *dw_b, *ln_w, *ln_b, *b1, *b2, *gamma;
  PlanesD w1, w2;
};
struct TfLayerW {
  const float *in_w, *post_w, *b_ih, *bqkv;
  PlanesD wih, wqkv, wo, w13, w2;
  __half* whh_perm;
};
struct ResnetW {
  const float *n1w, *n1b, *n2w, *n2b, *c1b, *c2b;
  PlanesD c1, c2;
};
struct SemBlockW {
  PlanesD u_c1[2], u_c2[2], conv;
  const float* conv_b;
  int stride, k;
};
struct SemDecBlockW {
  PlanesD conv, u_c1[2], u_c2[2];   // conv: k3 conv (stride 1) or the transposed conv's phase weight
  const float* b;                   // bias, repeated per phase for a transposed conv
  int stride, cout;
};
struct Policy {
  bool convnext, lstm_attn, mlp, mlp_dec, conv, head, dft;
};
static Policy policy_of(int p) {
  switch (p) {
    case QB_PRECISION_ACCURATE: return {true, true, true, true, true, true, true};
    case QB_PRECISION_FAST: return {false, false, false, false, false, false, true};
    case QB_PRECISION_MIXED_DEC16: return {false, false, true, false, true, true, true};
    default: return {false, false, true, true, true, true, true};
  }
}

}  // namespace qb
using namespace qb;

struct qb_handle {
  int device;
};

struct qb_rvq {
  qb_handle* h;
  Arena arena;
  Workspace ws;
  int nq, K, D;
  const float* cb;       // [nq, K, D]
  PlanesD planes;
  const float* consts;   // [nq*K + K]
  float e2max;
};

struct qb_codec {
  qb_handle* h;
  qb_codec_cfg cfg;
  Policy pol;
  Arena arena;
  Workspace ws;
  qb_tap_fn tap = nullptr;
  void* tap_user = nullptr;
  // geometry
  int nf, feat_ld, spec_ld, kin, lstm_u;
  PlanesD dft_inv;
  const float* istft_window;
  // two-stage STFT (n_fft = P*Q): stage matrices, twiddle table, analysis window
  int stft_P = 0, stft_Q = 0, stft_nB = 0, stft_ldX = 0;
  PlanesD stft_wA, stft_wB;
  const float *stft_tw = nullptr, *stft_window = nullptr;
  // encoder
  PlanesD e_embed, e_out;
  const float *e_embed_b, *e_norm_w, *e_norm_b, *e_fnorm_w, *e_fnorm_b, *e_out_b;
  std::vector<ConvNeXtW> e_cnx, d_cnx;
  std::vector<TfLayerW> e_tf, d_tf;
  // semantic encoder
  PlanesD s_conv, s_conv2;
  std::vector<SemBlockW> s_blocks;
  // decoder
  PlanesD d_embed, d_head;
  const float *d_embed_b, *d_gn_w, *d_gn_b, *d_norm_w, *d_norm_b, *d_fnorm_w, *d_fnorm_b, *d_head_b;
  ResnetW d_res[4];
  // semantic decoder (qb_codec_load_semantic_decoder; absent until loaded)
  bool has_sdec = false;
  int sd_code_dim = 0, sd_c0 = 0, sd_out = 0;
  PlanesD sd_conv1, sd_conv2;
  std::vector<SemDecBlockW> sd_blocks;
  // RoPE tables by sequence length
  std::map<int, std::pair<const float*, const float*>> rope;
  qb_rvq* q[2] = {nullptr, nullptr};
};

namespace qb {

static int load_convnext(Loader& L, const std::string& prefix, int n, bool split, std::vector<ConvNeXtW>* out) {
  out->resize(n);
  for (int i = 0; i < n; ++i) {
    const std::string p = prefix + std::to_string(i) + ".";
    ConvNeXtW& b = (*out)[i];
    QB_TRY(L.f32(&b.dw_w, p + "dwconv.conv.weight"));     // [C,1,7] contiguous == [C,7]
    QB_TRY(L.f32(&b.dw_b, p + "dwconv.conv.bias"));
    QB_TRY(L.f32(&b.ln_w, p + "norm.weight"));
    QB_TRY(L.f32(&b.ln_b, p + "norm.bias"));
    QB_TRY(L.lin(&b.w1, p + "pwconv1.linear.weight", split));
    QB_TRY(L.f32(&b.b1, p + "pwconv1.linear.bias"));
    QB_TRY(L.lin(&b.w2, p + "pwconv2.linear.weight", split));
    QB_TRY(L.f32(&b.b2, p + "pwconv2.linear.bias"));
    QB_TRY(L.f32(&b.gamma, p + "gamma"));
  }
  return 0;
}

static int load_transformer(Loader& L, const std::string& prefix, int n, int C, bool split_attn, bool split_mlp, int lstm_u,
                            std::vector<TfLayerW>* out) {
  out->resize(n);
  const int I = 4 * C < 4096 ? 4 * C : 4096;
  for (int i = 0; i < n; ++i) {
    const std::string p = prefix + "layers." + std::to_string(i) + ".", a = p + "self_attn.";
    TfLayerW& l = (*out)[i];
    QB_TRY(L.f32(&l.in_w, p + "input_layernorm.weight"));
    QB_TRY(L.f32(&l.post_w, p + "post_attention_layernorm.weight"));
    QB_TRY(L.lin(&l.wih, a + "rnn.weight_ih_l0", split_attn));
    const qb_tensor *bih, *bhh, *whh, *wq, *wk, *wv, *bq, *bk, *bv, *w1, *w3;
    QB_TRY(L.get(&bih, a + "rnn.bias_ih_l0", 1));
    QB_TRY(L.get(&bhh, a + "rnn.bias_hh_l0", 1));
    float* b;
    QB_TRY(L.arena.alloc((void**)&b, (size_t)4 * C * 4, false));
    add_vec_kernel<<<grid_for(4 * C), 256>>>(bih->data, bhh->data, 4 * C, b);
    l.b_ih = b;
    QB_TRY(L.get(&whh, a + "rnn.weight_hh_l0", 2));
    QB_REQUIRE(lstm_u > 0, "load: LSTM width %d unsupported by the wgmma recurrence (needs H %% 256 == 0)", C);
    QB_TRY(L.arena.alloc((void**)&l.whh_perm, (size_t)4 * C * C * 2, false));
    lstm_permute_kernel<<<grid_for(4LL * C * C), 256>>>(whh->data, C, lstm_u, l.whh_perm);
    // q|k|v rows concatenated
    QB_TRY(L.get(&wq, a + "q_proj.weight", 2)); QB_TRY(L.get(&wk, a + "k_proj.weight", 2)); QB_TRY(L.get(&wv, a + "v_proj.weight", 2));
    QB_TRY(L.get(&bq, a + "q_proj.bias", 1)); QB_TRY(L.get(&bk, a + "k_proj.bias", 1)); QB_TRY(L.get(&bv, a + "v_proj.bias", 1));
    float *tmp, *bqkv;
    QB_CHECK_CUDA(cudaMalloc(&tmp, (size_t)3 * C * C * 4));
    const qb_tensor* ws3[3] = {wq, wk, wv};
    const qb_tensor* bs3[3] = {bq, bk, bv};
    QB_TRY(L.arena.alloc((void**)&bqkv, (size_t)3 * C * 4, false));
    for (int j = 0; j < 3; ++j) {
      QB_CHECK_CUDA(cudaMemcpy(tmp + (size_t)j * C * C, ws3[j]->data, (size_t)C * C * 4, cudaMemcpyDeviceToDevice));
      QB_CHECK_CUDA(cudaMemcpy(bqkv + (size_t)j * C, bs3[j]->data, (size_t)C * 4, cudaMemcpyDeviceToDevice));
    }
    int e = L.planes_from(&l.wqkv, tmp, 3LL * C * C, split_attn);
    cudaDeviceSynchronize();
    cudaFree(tmp);
    QB_TRY(e);
    l.bqkv = bqkv;
    QB_TRY(L.lin(&l.wo, a + "o_proj.weight", split_attn));
    // SwiGLU: rows of w1 (gate) and w3 (up) interleaved
    QB_TRY(L.get(&w1, p + "mlp.w1.weight", 2)); QB_TRY(L.get(&w3, p + "mlp.w3.weight", 2));
    QB_CHECK_CUDA(cudaMalloc(&tmp, (size_t)2 * I * C * 4));
    interleave_rows_kernel<<<grid_for((long long)I * C), 256>>>(w1->data, w3->data, I, C, tmp);
    e = L.planes_from(&l.w13, tmp, 2LL * I * C, split_mlp);
    cudaDeviceSynchronize();
    cudaFree(tmp);
    QB_TRY(e);
    QB_TRY(L.lin(&l.w2, p + "mlp.w2.weight", split_mlp));
  }
  return 0;
}

static int tap(qb_codec* c, const char* name, const float* data, int64_t B, int64_t rows, int64_t C) {
  if (c->tap) c->tap(c->tap_user, name, data, B, rows, C);
  return 0;
}
static int tap_planes(qb_codec* c, const char* name, const PlanesD& p, int64_t B, int64_t rows, int64_t C, int64_t ld, int64_t rpb,
                      int64_t row_off, void* st) {
  if (!c->tap) return 0;
  float* tmp;
  QB_TRY(c->ws.f32(&tmp, std::string("tap_") + name, (size_t)B * rows * C));
  planes_to_f32_kernel<<<grid_for(B * rows * C), 256, 0, (cudaStream_t)st>>>(p.hi, p.lo, B, rows, (int)C, ld, rpb, row_off, tmp);
  QB_CHECK_CUDA(cudaGetLastError());
  c->tap(c->tap_user, name, tmp, B, rows, C);
  return 0;
}

static qb_rowmap rm(void* p, int64_t ld, int64_t rpb, int64_t off) {
  qb_rowmap r;
  r.ptr = p; r.ld = ld; r.rows_per_batch = rpb; r.row_off = off;
  return r;
}

// one dense contraction through the op-level ABI
struct G {
  qb_gemm_desc d;
  G(const PlanesD& a, int64_t a_batch, int64_t a_rpb, int64_t a_ld, int64_t m_per_batch, const PlanesD& w, int64_t n, int taps = 1,
    int stride = 1) {
    memset(&d, 0, sizeof(d));
    const bool split = a.lo != nullptr && w.lo != nullptr;
    d.a_hi = (const qb_half*)a.hi; d.a_lo = split ? (const qb_half*)a.lo : nullptr;
    d.a_batch = a_batch; d.a_rows_per_batch = a_rpb; d.a_ld = a_ld; d.taps = taps; d.stride = stride; d.m_per_batch = m_per_batch;
    d.w_hi = (const qb_half*)w.hi; d.w_lo = split ? (const qb_half*)w.lo : nullptr; d.n = n; d.dilation = 1;
  }
  G& bias(const float* b) { d.bias = b; return *this; }
  G& gamma(const float* g) { d.gamma = g; return *this; }
  G& act(int a) { d.act = a; return *this; }
  G& act2(int a) { d.act2 = a; return *this; }
  G& residual(float* p, int64_t ld, int64_t rpb, int64_t off) { d.residual = rm(p, ld, rpb, off); return *this; }
  G& out32(float* p, int64_t ld, int64_t rpb, int64_t off) { d.out_f32 = rm(p, ld, rpb, off); return *this; }
  G& outp(const PlanesD& p, int64_t ld, int64_t rpb, int64_t off) {
    d.out_hi = rm(p.hi, ld, rpb, off);
    d.out_lo = rm(p.lo, p.lo ? ld : 0, p.lo ? rpb : 0, p.lo ? off : 0);
    return *this;
  }
  int run(void* st) { return qb_gemm(&d, st); }
};
// nn.Linear over M rows
static G lin(const PlanesD& a, int64_t M, int64_t K, const PlanesD& w, int64_t n) { return G(a, 1, M, K, M, w, n); }

static int rope_tables(qb_codec* c, int T, int D, const float** cos_out, const float** sin_out) {
  auto it = c->rope.find(T * 1024 + D);
  if (it == c->rope.end()) {
    std::vector<float> cs((size_t)T * D), sn((size_t)T * D);
    for (int t = 0; t < T; ++t)
      for (int i = 0; i < D / 2; ++i) {
        const float inv = 1.0f / powf(10000.0f, (float)(2 * i) / (float)D);
        const float fr = (float)t * inv;
        cs[(size_t)t * D + i] = cs[(size_t)t * D + i + D / 2] = cosf(fr);
        sn[(size_t)t * D + i] = sn[(size_t)t * D + i + D / 2] = sinf(fr);
      }
    float *dc, *ds;
    QB_TRY(c->arena.alloc((void**)&dc, cs.size() * 4, false));
    QB_TRY(c->arena.alloc((void**)&ds, sn.size() * 4, false));
    QB_CHECK_CUDA(cudaMemcpy(dc, cs.data(), cs.size() * 4, cudaMemcpyHostToDevice));
    QB_CHECK_CUDA(cudaMemcpy(ds, sn.data(), sn.size() * 4, cudaMemcpyHostToDevice));
    it = c->rope.emplace(T * 1024 + D, std::make_pair((const float*)dc, (const float*)ds)).first;
  }
  *cos_out = it->second.first;
  *sin_out = it->second.second;
  return 0;
}

// vq/conv.py:200-213, n blocks; x [B*F, C] fp32 updated in place
static int run_convnext(qb_codec* c, const std::vector<ConvNeXtW>& blocks, float* x, int64_t B, int64_t F, int C, int I, void* st) {
  const int64_t M = B * F;
  PlanesD t1, hid;
  QB_TRY(c->ws.planes(&t1, "cnx_t1", (size_t)M * C, c->pol.convnext));
  QB_TRY(c->ws.planes(&hid, "cnx_hid", (size_t)M * I, c->pol.convnext));
  for (const ConvNeXtW& b : blocks) {
    QB_TRY(qb_dwconv7_ln(x, b.dw_w, b.dw_b, b.ln_w, b.ln_b, B, F, C, (qb_half*)t1.hi, (qb_half*)t1.lo, st));
    QB_TRY(lin(t1, M, C, b.w1, I).bias(b.b1).act(QB_ACT_GELU).outp(hid, I, M, 0).run(st));
    QB_TRY(lin(hid, M, I, b.w2, C).bias(b.b2).gamma(b.gamma).residual(x, C, M, 0).out32(x, C, M, 0).run(st));
  }
  return 0;
}

// encoder_modules/transformer.py:367-393 per layer; x [B*F, C] fp32 updated in place
static int run_transformer(qb_codec* c, const std::vector<TfLayerW>& layers, float* x, int64_t B, int64_t F, int C, bool split_mlp,
                           void* st) {
  const int heads = C / 64, hd = 64;
  const int64_t M = B * F;
  const int I = 4 * C < 4096 ? 4 * C : 4096;
  const bool pa = c->pol.lstm_attn;
  PlanesD t_a, t_b, t_m, hid;
  float *xp, *qkv;
  void *lstm_ws, *att_ws;
  QB_TRY(c->ws.planes(&t_a, "tf_a", (size_t)M * C, pa));
  QB_TRY(c->ws.planes(&t_b, "tf_b", (size_t)M * C, pa));
  QB_TRY(c->ws.planes(&t_m, "tf_m", (size_t)M * C, split_mlp));
  QB_TRY(c->ws.planes(&hid, split_mlp ? "tf_hid_s" : "tf_hid", (size_t)M * I, split_mlp));
  QB_TRY(c->ws.f32(&xp, "tf_xp", (size_t)M * 4 * C));
  QB_TRY(c->ws.f32(&qkv, "tf_qkv", (size_t)M * 3 * C));
  QB_TRY(c->ws.get(&lstm_ws, "lstm_ws", (size_t)qb_lstm_tc_workspace_bytes(B, C)));
  // wgmma attention (attention_umma.cu) in both precision policies
  QB_TRY(c->ws.get(&att_ws, "att5_ws", (size_t)qb_attention_umma_workspace_bytes(B, F, heads, hd, pa ? 1 : 0)));
  const float *rc, *rs;
  QB_TRY(rope_tables(c, (int)F, hd, &rc, &rs));
  for (const TfLayerW& L : layers) {
    QB_TRY(qb_rmsnorm(x, L.in_w, 1e-6f, M, C, nullptr, (qb_half*)t_a.hi, (qb_half*)t_a.lo, st));
    QB_TRY(lin(t_a, M, C, L.wih, 4 * C).bias(L.b_ih).out32(xp, 4 * C, M, 0).run(st));
    QB_TRY(qb_lstm_tc(xp, (const qb_half*)L.whh_perm, c->lstm_u, B, F, C, (qb_half*)t_b.hi, (qb_half*)t_b.lo, lstm_ws, st));
    QB_TRY(lin(t_b, M, C, L.wqkv, 3 * C).bias(L.bqkv).out32(qkv, 3 * C, M, 0).run(st));
    QB_TRY(qb_attention_umma(qkv, B, F, heads, hd, rc, rs, (qb_half*)t_a.hi, (qb_half*)t_a.lo, pa ? 1 : 0, 0, att_ws, st));
    QB_TRY(lin(t_a, M, C, L.wo, C).residual(x, C, M, 0).out32(x, C, M, 0).run(st));
    QB_TRY(qb_rmsnorm(x, L.post_w, 1e-6f, M, C, nullptr, (qb_half*)t_m.hi, (qb_half*)t_m.lo, st));
    QB_TRY(lin(t_m, M, C, L.w13, 2 * I).act(QB_ACT_SWIGLU).outp(hid, I, M, 0).run(st));
    QB_TRY(lin(hid, M, I, L.w2, C).residual(x, C, M, 0).out32(x, C, M, 0).run(st));
  }
  return 0;
}

// vq/conv.py:286-303
static int run_resnet(qb_codec* c, const ResnetW& R, float* x, int64_t B, int64_t F, int C, void* st) {
  const int64_t M = B * F;
  float *stats, *h;
  PlanesD pr;
  QB_TRY(c->ws.f32(&stats, "gn_stats", (size_t)B * 32 * 2));
  QB_TRY(c->ws.padded(&pr, "res_pr", B, F + 2, C, c->pol.conv));
  QB_TRY(c->ws.f32(&h, "res_h", (size_t)M * C));
  QB_TRY(qb_groupnorm_stats(x, B, F, C, 32, 1e-6f, stats, st));
  QB_TRY(qb_groupnorm_apply(x, stats, R.n1w, R.n1b, B, F, C, 32, 1, nullptr, (qb_half*)pr.hi, (qb_half*)pr.lo, C, F + 2, 1, st));
  QB_TRY(G(pr, B, F + 2, C, F, R.c1, C, 3).bias(R.c1b).out32(h, C, F, 0).run(st));
  QB_TRY(qb_groupnorm_stats(h, B, F, C, 32, 1e-6f, stats, st));
  QB_TRY(qb_groupnorm_apply(h, stats, R.n2w, R.n2b, B, F, C, 32, 1, nullptr, (qb_half*)pr.hi, (qb_half*)pr.lo, C, F + 2, 1, st));
  QB_TRY(G(pr, B, F + 2, C, F, R.c2, C, 3).bias(R.c2b).residual(x, C, F, 0).out32(x, C, F, 0).run(st));
  return 0;
}

// vq/codec_encoder.py:62-79 -> emb [B*N, dimension] fp32
static int encode_emb(qb_codec* c, const float* wav, int64_t B, int64_t T, float** emb_out, int64_t* N_out, void* st) {
  const qb_codec_cfg& g = c->cfg;
  const int hop = g.hop_length, nf = c->nf, stride = g.frame_stride, C = g.dim, I = g.intermediate_dim, Dq = g.dimension;
  QB_REQUIRE(T > 0 && T % ((int64_t)hop * stride) == 0, "codec_encode: waveform length %lld must be a multiple of %d (pad_wav, audio_tokenizer.py:63-66)",
             (long long)T, hop * stride);
  const int64_t F = T / hop, N = F / stride, M = B * F;
  PlanesD feat, fin, ga, Z;
  float *Y, *X, *x0, *x, *emb;
  QB_TRY(c->ws.padded(&feat, "enc_feat", B, F + 2, c->feat_ld, c->pol.conv));
  // two-stage DFT: gather -> P-point DFTs (GEMM, K = 64) -> twiddle -> Q-point DFTs (GEMM, K = 128) -> log-magnitude / phase
  const int P = c->stft_P, Q = c->stft_Q;
  QB_TRY(c->ws.planes(&ga, "enc_sg", (size_t)M * Q * 64, true));
  QB_TRY(qb_stft_gather(wav, B, T, hop, g.n_fft, P, Q, c->stft_window, (qb_half*)ga.hi, (qb_half*)ga.lo, st));
  QB_TRY(c->ws.f32(&Y, "enc_sy", (size_t)M * Q * 2 * P));
  QB_TRY(lin(ga, M * Q, 64, c->stft_wA, 2 * P).out32(Y, 2 * P, M * Q, 0).run(st));
  QB_TRY(c->ws.planes(&Z, "enc_sz", (size_t)M * P * 128, true));
  QB_TRY(qb_stft_twiddle(Y, 2 * P, M, P, Q, c->stft_tw, (qb_half*)Z.hi, (qb_half*)Z.lo, st));
  QB_TRY(c->ws.f32(&X, "enc_sx", (size_t)M * P * c->stft_ldX));
  QB_TRY(lin(Z, M * P, 128, c->stft_wB, c->stft_nB).out32(X, c->stft_ldX, M * P, 0).run(st));
  QB_TRY(qb_stft_post2(X, c->stft_ldX, B, F, nf, P, (qb_half*)feat.hi, (qb_half*)feat.lo, c->feat_ld, F + 2, 1, st));
  QB_TRY(tap_planes(c, "enc.feat", feat, B, F, 2 * nf, c->feat_ld, F + 2, 1, st));
  QB_TRY(c->ws.f32(&x0, "enc_x0", (size_t)M * C));
  QB_TRY(G(feat, B, F + 2, c->feat_ld, F, c->e_embed, C, 3).bias(c->e_embed_b).out32(x0, C, F, 0).run(st));
  QB_TRY(c->ws.f32(&x, "enc_x", (size_t)M * C));
  QB_TRY(qb_layernorm(x0, c->e_norm_w, c->e_norm_b, 1e-6f, B, F, C, x, nullptr, nullptr, 0, 0, 0, st));
  tap(c, "enc.embed_norm", x, B, F, C);
  QB_TRY(run_convnext(c, c->e_cnx, x, B, F, C, I, st));
  tap(c, "enc.prior", x, B, F, C);
  QB_TRY(run_transformer(c, c->e_tf, x, B, F, C, c->pol.mlp, st));
  tap(c, "enc.post", x, B, F, C);
  const int k = 2 * stride + 1, pad = k / 2;
  const int64_t rpb = pad_to(F + 2 * pad, stride);
  QB_TRY(c->ws.padded(&fin, "enc_fin", B, rpb, C, c->pol.conv));
  QB_TRY(qb_layernorm(x, c->e_fnorm_w, c->e_fnorm_b, 1e-6f, B, F, C, nullptr, (qb_half*)fin.hi, (qb_half*)fin.lo, C, rpb, pad, st));
  QB_TRY(c->ws.f32(&emb, "enc_emb", (size_t)B * N * Dq));
  QB_TRY(G(fin, B, rpb, C, N, c->e_out, Dq, k, stride).bias(c->e_out_b).out32(emb, Dq, N, 0).run(st));
  tap(c, "enc.out", emb, B, N, Dq);
  *emb_out = emb;
  *N_out = N;
  return 0;
}

// vq/semantic_module.py:196-201 -> [B*N, out_channels] fp32
static int encode_sem(qb_codec* c, const float* feat_in, int64_t B, int64_t F, float** out_p, int64_t* N_out, void* st) {
  const qb_codec_cfg& g = c->cfg;
  const int Cin = g.sem_input_channels, Cs = g.sem_encode_channels, Co = g.sem_out_channels;
  const bool pc = c->pol.conv;
  const int cin_pad = (int)pad_to(Cin, 64);
  PlanesD fin, pe, pu;
  float* sx;
  QB_TRY(c->ws.padded(&fin, "sem_in", B, F + 2, cin_pad, pc));
  QB_TRY(qb_bct_to_planes(feat_in, B, Cin, F, (qb_half*)fin.hi, (qb_half*)fin.lo, cin_pad, F + 2, 1, st));
  int64_t Tc = F;
  QB_TRY(c->ws.f32(&sx, "sem_x" + std::to_string(Tc), (size_t)B * Tc * Cs));
  QB_TRY(c->ws.padded(&pe, "sem_pe" + std::to_string(Tc), B, Tc + 2, Cs, pc));
  QB_TRY(G(fin, B, F + 2, cin_pad, F, c->s_conv, Cs, 3).out32(sx, Cs, Tc, 0).outp(pe, Cs, Tc + 2, 1).act2(QB_ACT_ELU).run(st));
  const int nb = (int)c->s_blocks.size();
  for (int bi = 0; bi < nb; ++bi) {
    const SemBlockW& blk = c->s_blocks[bi];
    QB_TRY(c->ws.planes(&pu, "sem_pu" + std::to_string(Tc), (size_t)B * Tc * Cs, pc));
    for (int u = 0; u < 2; ++u) {
      QB_TRY(G(pe, B, Tc + 2, Cs, Tc, blk.u_c1[u], Cs, 3).act(QB_ACT_ELU).outp(pu, Cs, Tc, 0).run(st));
      QB_TRY(G(pu, B, Tc, Cs, Tc, blk.u_c2[u], Cs).residual(sx, Cs, Tc, 0).out32(sx, Cs, Tc, 0).outp(pe, Cs, Tc + 2, 1)
                 .act2(u == 0 ? QB_ACT_ELU : QB_ACT_NONE).run(st));
    }
    const int s = blk.stride, k = blk.k, pad = (k - 1) / 2;
    QB_REQUIRE(pad == 1 && (Tc + 2) % s == 0, "codec_encode: semantic feature length %lld incompatible with stride %d", (long long)Tc, s);
    const int64_t Tn = (Tc + 2 * pad - k) / s + 1;
    float* sx2;
    PlanesD pe2;
    QB_TRY(c->ws.f32(&sx2, "sem_x" + std::to_string(Tn) + "_" + std::to_string(bi), (size_t)B * Tn * Cs));
    QB_TRY(c->ws.padded(&pe2, "sem_pe" + std::to_string(Tn) + "_" + std::to_string(bi), B, Tn + 2, Cs, pc));
    QB_TRY(G(pe, B, Tc + 2, Cs, Tn, blk.conv, Cs, k, s).bias(blk.conv_b).out32(sx2, Cs, Tn, 0).outp(pe2, Cs, Tn + 2, 1)
               .act2(bi + 1 < nb ? QB_ACT_ELU : QB_ACT_NONE).run(st));
    sx = sx2; pe = pe2; Tc = Tn;
    const std::string nm = "sem.block" + std::to_string(bi);
    tap(c, nm.c_str(), sx, B, Tc, Cs);
  }
  float* out;
  QB_TRY(c->ws.f32(&out, "sem_out", (size_t)B * Tc * Co));
  QB_TRY(G(pe, B, Tc + 2, Cs, Tc, c->s_conv2, Co, 3).out32(out, Co, Tc, 0).run(st));
  tap(c, "sem.out", out, B, Tc, Co);
  *out_p = out;
  *N_out = Tc;
  return 0;
}

// vq/semantic_module.py:294-299 (Decoder), :245-249 (DecoderBlock), :78-81 (ResidualUnit).  z [B*N, code_dim] fp32 -> pred_feat
// [B, output_channels, T] fp32.  Every conv input sits in a planes buffer padded by one zero frame on each side; a block's fp32
// trunk is updated in place by the 1x1 convs' residual epilogues, and each epilogue writes the planes its consumer reads.
static int semantic_decode_z(qb_codec* c, const float* z, int64_t B, int64_t N, float* pred, void* st) {
  const bool pc = c->pol.conv;
  const int cd = (int)pad_to(c->sd_code_dim, 64);
  PlanesD zp, xin;
  QB_TRY(c->ws.padded(&zp, "sd_z", B, N + 2, cd, pc));
  QB_TRY(qb_rows_to_planes(z, B, N, c->sd_code_dim, 1, QB_ACT_NONE, (qb_half*)zp.hi, (qb_half*)zp.lo, cd, N + 2, 1, st));
  int cp = (int)pad_to(c->sd_c0, 64);
  QB_TRY(c->ws.padded(&xin, "sd_in0", B, N + 2, cp, pc));
  QB_TRY(G(zp, B, N + 2, cd, N, c->sd_conv1, c->sd_c0, 3).outp(xin, cp, N + 2, 1).run(st));
  int64_t T = N;
  for (size_t bi = 0; bi < c->sd_blocks.size(); ++bi) {
    const SemDecBlockW& blk = c->sd_blocks[bi];
    const int co = blk.cout, cpo = (int)pad_to(co, 64), s = blk.stride;
    const std::string id = std::to_string(bi);
    float* trunk;
    int64_t tr_rpb, tr_off, Tn;
    PlanesD pe, pu, nxt;
    if (s == 1) {
      Tn = T; tr_rpb = T; tr_off = 0;
      QB_TRY(c->ws.f32(&trunk, "sd_x" + id, (size_t)B * T * co));
      QB_TRY(c->ws.padded(&pe, "sd_pe" + id, B, T + 2, cpo, pc));
      QB_TRY(G(xin, B, T + 2, cp, T, blk.conv, co, 3).bias(blk.b).out32(trunk, co, T, 0).outp(pe, cpo, T + 2, 1).act2(QB_ACT_ELU).run(st));
    } else {
      // ConvTranspose1d(2s, s, padding (s+1)/2, output_padding s%2) as a 2-tap GEMM over the one-frame-padded input: row q holds the
      // s phases of uncropped frames q*s.., and the output clip is frames [pad, pad + T*s) of the rows read as [(T+1)*s, co]
      const int pad = (s + 1) / 2;
      Tn = T * s; tr_rpb = (T + 1) * s; tr_off = pad;
      QB_TRY(c->ws.f32(&trunk, "sd_up" + id, (size_t)B * (T + 1) * s * co));
      QB_TRY(G(xin, B, T + 2, cp, T + 1, blk.conv, (int64_t)s * co, 2).bias(blk.b).out32(trunk, (int64_t)s * co, T + 1, 0).run(st));
      QB_TRY(c->ws.padded(&pe, "sd_pe" + id, B, Tn + 2, cpo, pc));
      QB_TRY(qb_elu_planes(trunk + (int64_t)pad * co, (T + 1) * s * co, B, Tn, co, (qb_half*)pe.hi, (qb_half*)pe.lo, cpo, Tn + 2, 1, st));
    }
    T = Tn;
    QB_TRY(c->ws.planes(&pu, "sd_pu" + id, (size_t)B * T * cpo, pc));
    QB_TRY(c->ws.padded(&nxt, "sd_in" + std::to_string(bi + 1), B, T + 2, cpo, pc));
    for (int u = 0; u < 2; ++u) {
      QB_TRY(G(pe, B, T + 2, cpo, T, blk.u_c1[u], co, 3).act(QB_ACT_ELU).outp(pu, cpo, T, 0).run(st));
      G g2(pu, B, T, cpo, T, blk.u_c2[u], co);
      g2.residual(trunk, co, tr_rpb, tr_off);
      if (u == 0) g2.out32(trunk, co, tr_rpb, tr_off).outp(pe, cpo, T + 2, 1).act2(QB_ACT_ELU);
      else g2.outp(nxt, cpo, T + 2, 1);
      QB_TRY(g2.run(st));
    }
    xin = nxt; cp = cpo;
  }
  float* rows;
  QB_TRY(c->ws.f32(&rows, "sd_out", (size_t)B * T * c->sd_out));
  QB_TRY(G(xin, B, T + 2, cp, T, c->sd_conv2, c->sd_out, 3).out32(rows, c->sd_out, T, 0).run(st));
  return qb_ssl_compress(rows, B, T, c->sd_out, 0.f, 1, pred, st);      // power 0: the plain [B, T, C] -> [B, C, T] copy
}

// vq/codec_decoder.py:62-72.  z [B*N, input_channels] fp32 -> wav [B, N*factor*hop]
static int decode_z(qb_codec* c, const float* z, int64_t B, int64_t N, float* wav, void* st) {
  const qb_codec_cfg& g = c->cfg;
  const int Cin = g.dec_input_channels, C = g.dim, I = g.intermediate_dim, f = g.frame_stride, hop = g.hop_length, nf = c->nf,
            n_fft = g.n_fft;
  const int64_t F = N * f, M = B * F;
  const int k = f + 1, pad = k / 2;
  PlanesD zin, t1, sp;
  float *x, *stats, *h, *head, *frames;
  QB_TRY(c->ws.padded(&zin, "dec_zin", B, F + 2 * pad, Cin, c->pol.conv));
  QB_TRY(qb_rows_to_planes(z, B, N, Cin, f, QB_ACT_NONE, (qb_half*)zin.hi, (qb_half*)zin.lo, Cin, F + 2 * pad, pad, st));
  QB_TRY(c->ws.f32(&x, "dec_x", (size_t)M * C));
  QB_TRY(G(zin, B, F + 2 * pad, Cin, F, c->d_embed, C, k).bias(c->d_embed_b).out32(x, C, F, 0).run(st));
  tap(c, "dec.embed", x, B, F, C);
  QB_TRY(run_resnet(c, c->d_res[0], x, B, F, C, st));
  tap(c, "dec.res0", x, B, F, C);
  QB_TRY(run_resnet(c, c->d_res[1], x, B, F, C, st));
  QB_TRY(run_transformer(c, c->d_tf, x, B, F, C, c->pol.mlp_dec, st));
  tap(c, "dec.tf", x, B, F, C);
  QB_TRY(run_resnet(c, c->d_res[2], x, B, F, C, st));
  QB_TRY(run_resnet(c, c->d_res[3], x, B, F, C, st));
  QB_TRY(c->ws.f32(&stats, "gn_stats", (size_t)B * 32 * 2));
  QB_TRY(c->ws.f32(&h, "res_h", (size_t)M * C));
  QB_TRY(qb_groupnorm_stats(x, B, F, C, 32, 1e-6f, stats, st));
  QB_TRY(qb_groupnorm_apply(x, stats, c->d_gn_w, c->d_gn_b, B, F, C, 32, 0, h, nullptr, nullptr, 0, 0, 0, st));
  tap(c, "dec.prior", h, B, F, C);
  QB_TRY(qb_layernorm(h, c->d_norm_w, c->d_norm_b, 1e-6f, B, F, C, x, nullptr, nullptr, 0, 0, 0, st));
  QB_TRY(run_convnext(c, c->d_cnx, x, B, F, C, I, st));
  tap(c, "dec.post", x, B, F, C);
  QB_TRY(c->ws.planes(&t1, "dec_fn", (size_t)M * C, c->pol.head));
  QB_TRY(qb_layernorm(x, c->d_fnorm_w, c->d_fnorm_b, 1e-6f, B, F, C, nullptr, (qb_half*)t1.hi, (qb_half*)t1.lo, C, F, 0, st));
  QB_TRY(tap_planes(c, "dec.final_norm", t1, B, F, C, C, F, 0, st));
  QB_TRY(c->ws.f32(&head, "dec_head", (size_t)M * c->spec_ld));
  QB_TRY(lin(t1, M, C, c->d_head, 2 * nf).bias(c->d_head_b).out32(head, c->spec_ld, M, 0).run(st));
  QB_TRY(c->ws.planes(&sp, "dec_sp", (size_t)M * c->kin, c->pol.dft));
  QB_TRY(qb_istft_pre(head, c->spec_ld, M, nf, (qb_half*)sp.hi, (qb_half*)sp.lo, c->kin, st));
  QB_TRY(c->ws.f32(&frames, "dec_frames", (size_t)M * n_fft));
  QB_TRY(lin(sp, M, c->kin, c->dft_inv, n_fft).out32(frames, n_fft, M, 0).run(st));
  QB_TRY(qb_istft_ola(frames, c->istft_window, B, F, n_fft, hop, wav, st));
  return 0;
}

static int rvq_build(qb_handle* h, const float* codebooks, int nq, int K, int D, bool copy, qb_rvq** out) {
  QB_REQUIRE(h && codebooks && out && nq >= 1 && K >= 1 && D % 64 == 0, "rvq_load: bad args (D must be a multiple of 64)");
  qb_rvq* q = new qb_rvq();
  q->h = h; q->nq = nq; q->K = K; q->D = D;
  const long long n = (long long)nq * K * D;
  float* cb;
  int e = q->arena.alloc((void**)&cb, (size_t)n * 4, false);
  if (!e && cudaMemcpy(cb, codebooks, (size_t)n * 4, cudaMemcpyDeviceToDevice) != cudaSuccess) { set_error("rvq_load: codebook copy failed"); e = -2; }
  (void)copy;
  float *consts = nullptr, *e2 = nullptr;
  if (!e) e = q->arena.alloc((void**)&q->planes.hi, (size_t)n * 2, false);
  if (!e) e = q->arena.alloc((void**)&q->planes.lo, (size_t)n * 2, false);
  if (!e) e = qb_split_f16(cb, (qb_half*)q->planes.hi, (qb_half*)q->planes.lo, n, nullptr);
  if (!e) e = q->arena.alloc((void**)&consts, (size_t)(nq * K + K) * 4, false);
  if (!e) e = q->arena.alloc((void**)&e2, (size_t)nq * K * 4, false);
  if (!e) {
    rvq_consts_kernel<<<(unsigned)ceil_div((long long)nq * K > K ? (long long)nq * K : K, 256), 256>>>(cb, nq, K, D, consts, e2);
    std::vector<float> he2((size_t)nq * K);
    if (cudaMemcpy(he2.data(), e2, he2.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { set_error("rvq_load: %s", cudaGetErrorString(cudaGetLastError())); e = -2; }
    float mx = 0.f;
    for (float v : he2) mx = v > mx ? v : mx;
    q->e2max = mx;
  }
  if (e) { delete q; return e; }
  q->cb = cb; q->consts = consts;
  *out = q;
  return 0;
}

}  // namespace qb

// ================================================================== C ABI
extern "C" int qb_init(int device, qb_handle** out) {
  QB_REQUIRE(out != nullptr, "qb_init: null out");
  int n = 0;
  QB_CHECK_CUDA(cudaGetDeviceCount(&n));
  QB_REQUIRE(device >= 0 && device < n, "qb_init: device %d out of range (%d visible)", device, n);
  QB_CHECK_CUDA(cudaSetDevice(device));
  int major = 0, minor = 0;
  QB_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  QB_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  QB_REQUIRE(major == 9 && minor == 0, "qb_init: libquark_b200 is built for sm_90a only (device %d is sm_%d%d)", device, major, minor);
  qb_handle* h = new qb_handle();
  h->device = device;
  *out = h;
  return 0;
}
extern "C" void qb_handle_free(qb_handle* h) { delete h; }
extern "C" int qb_memcpy_d2d(void* dst, const void* src, int64_t bytes, void* stream) {
  QB_REQUIRE(dst && src && bytes >= 0, "memcpy_d2d: bad args");
  QB_CHECK_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}
extern "C" const char* qb_handle_last_error(qb_handle*) { return qb_last_error(); }

extern "C" int qb_rvq_load(qb_handle* h, const float* codebooks, int32_t nq, int32_t K, int32_t D, qb_rvq** out) {
  return rvq_build(h, codebooks, nq, K, D, true, out);
}
extern "C" void qb_rvq_free(qb_rvq* q) { delete q; }
extern "C" int qb_rvq_encode_rows(qb_rvq* q, const float* x, int64_t M, int64_t* idx, float* quantized, void* stream) {
  QB_REQUIRE(q && x && idx && M >= 0, "rvq_encode_rows: bad args");
  if (M == 0) return 0;
  void* ws;
  QB_TRY(q->ws.get(&ws, "rvq_ws", (size_t)qb_rvq_workspace_bytes(M, q->D, q->K)));
  return qb_rvq_encode(x, q->cb, (const qb_half*)q->planes.hi, (const qb_half*)q->planes.lo, q->consts, q->e2max, M, q->D, q->K, q->nq,
                       idx, quantized, ws, stream);
}
extern "C" int qb_rvq_decode_rows(qb_rvq* q, const int64_t* idx, int64_t M, float* out, void* stream) {
  QB_REQUIRE(q && idx && out, "rvq_decode_rows: bad args");
  return qb_rvq_decode(idx, q->cb, M, q->D, q->K, q->nq, out, q->D, 0, stream);
}

extern "C" int qb_codec_load(qb_handle* h, const qb_codec_cfg* cfg, const qb_tensor* named, int32_t n, qb_codec** out) {
  QB_REQUIRE(h && cfg && named && out && n > 0, "codec_load: bad args");
  // n_fft <= 4096: the two-stage STFT needs n_fft = P*Q with P, Q <= 64
  QB_REQUIRE(cfg->n_fft == 2 * cfg->hop_length && cfg->hop_length % 64 == 0 && cfg->n_fft <= 4096,
             "codec_load: the STFT/ISTFT kernels assume n_fft == 2*hop, hop %% 64 == 0 and n_fft <= 4096 (n_fft = P*Q with P, Q <= 64); "
             "got n_fft %d, hop %d", cfg->n_fft, cfg->hop_length);
  QB_REQUIRE(cfg->dim % 256 == 0 && cfg->dimension % 64 == 0 && cfg->sem_n_blocks >= 0 && cfg->sem_n_blocks <= 8, "codec_load: unsupported widths");
  QB_CHECK_CUDA(cudaSetDevice(h->device));
  WeightTable wt;
  QB_TRY(wt.init(named, n));
  qb_codec* c = new qb_codec();
  struct Guard { qb_codec* c; ~Guard() { if (c) { delete c->q[0]; delete c->q[1]; delete c; } } } guard{c};
  c->h = h; c->cfg = *cfg; c->pol = policy_of(cfg->precision);
  Loader L(wt, c->arena);
  const int n_fft = cfg->n_fft, nf = n_fft / 2 + 1, C = cfg->dim;
  c->nf = nf; c->feat_ld = (int)pad_to(2 * nf, 64); c->spec_ld = (int)pad_to(2 * nf, 4); c->kin = (int)pad_to(2 * nf, 64);
  c->lstm_u = qb_lstm_tc_units(C);
  // ---- DFT matrices in fp64 with exact argument reduction (window folded in)
  {
    const qb_tensor *we, *wd;
    QB_TRY(L.get(&we, "encoder.stft.window", 1));
    QB_TRY(L.get(&wd, "decoder.head.istft.window", 1));
    std::vector<float> win_d(n_fft);
    QB_CHECK_CUDA(cudaMemcpy(win_d.data(), wd->data, (size_t)n_fft * 4, cudaMemcpyDeviceToHost));
    const double two_pi = 6.283185307179586476925286766559;
    std::vector<double> cs(n_fft), sn(n_fft);
    for (int r = 0; r < n_fft; ++r) { cs[r] = cos(two_pi * r / n_fft); sn[r] = sin(two_pi * r / n_fft); }
    // two-stage factorisation n_fft = P*Q with P = 64, Q = n_fft/64 <= 64 (checked above): chains of 4 / 8 MMAs instead of n_fft/16
    const int P = 64, Q = n_fft / 64, K2 = (nf - 1) / P + 1;
    c->stft_P = P; c->stft_Q = Q;
    c->stft_nB = 2 * K2; c->stft_ldX = (int)pad_to(2 * K2, 4);
    std::vector<double> wA((size_t)2 * P * 64, 0.0), wB((size_t)2 * K2 * 128, 0.0);
    for (int k1 = 0; k1 < P; ++k1)
      for (int a = 0; a < P; ++a) {
        const double ang = two_pi * ((k1 * a) % P) / P;
        wA[(size_t)(2 * k1) * 64 + a] = cos(ang);
        wA[(size_t)(2 * k1 + 1) * 64 + a] = -sin(ang);
      }
    for (int k2 = 0; k2 < K2; ++k2)
      for (int b = 0; b < Q; ++b) {
        const double ang = two_pi * ((k2 * b) % Q) / Q;
        wB[(size_t)(2 * k2) * 128 + b] = cos(ang);
        wB[(size_t)(2 * k2) * 128 + Q + b] = sin(ang);
        wB[(size_t)(2 * k2 + 1) * 128 + b] = -sin(ang);
        wB[(size_t)(2 * k2 + 1) * 128 + Q + b] = cos(ang);
      }
    QB_TRY(L.planes_from_f64(&c->stft_wA, wA));
    QB_TRY(L.planes_from_f64(&c->stft_wB, wB));
    std::vector<float> tw((size_t)Q * P * 2);
    for (int b = 0; b < Q; ++b)
      for (int k1 = 0; k1 < P; ++k1) {
        const double ang = two_pi * ((b * k1) % n_fft) / n_fft;
        tw[((size_t)b * P + k1) * 2] = (float)cos(ang);
        tw[((size_t)b * P + k1) * 2 + 1] = (float)(-sin(ang));
      }
    float* dtw;
    QB_TRY(c->arena.alloc((void**)&dtw, tw.size() * 4, false));
    QB_CHECK_CUDA(cudaMemcpy(dtw, tw.data(), tw.size() * 4, cudaMemcpyHostToDevice));
    c->stft_tw = dtw;
    QB_TRY(L.f32(&c->stft_window, "encoder.stft.window"));
    std::vector<double> inv((size_t)n_fft * c->kin, 0.0);    // [n_fft, kin]: 1/N, Hermitian weights, synthesis window folded in
    for (int s = 0; s < n_fft; ++s)
      for (int k = 0; k < nf; ++k) {
        const int r = (int)(((long long)k * s) % n_fft);
        const double ck = (k == 0 || k == nf - 1) ? 1.0 : 2.0;
        inv[(size_t)s * c->kin + k] = cs[r] * ck / n_fft * (double)win_d[s];
        inv[(size_t)s * c->kin + nf + k] = (k == 0 || k == nf - 1) ? 0.0 : -sn[r] * ck / n_fft * (double)win_d[s];   // irfft ignores imag of DC / Nyquist
      }
    QB_TRY(L.planes_from_f64(&c->dft_inv, inv));
    QB_TRY(L.f32(&c->istft_window, "decoder.head.istft.window"));
  }
  const Policy& P = c->pol;
  // ---- encoder
  QB_TRY(L.conv(&c->e_embed, "encoder.embed.conv.weight", P.conv));
  QB_TRY(L.f32(&c->e_embed_b, "encoder.embed.conv.bias"));
  QB_TRY(L.f32(&c->e_norm_w, "encoder.norm.weight")); QB_TRY(L.f32(&c->e_norm_b, "encoder.norm.bias"));
  QB_TRY(load_convnext(L, "encoder.prior_net.", cfg->enc_convnext_layers, P.convnext, &c->e_cnx));
  QB_TRY(load_transformer(L, "encoder.post_net.1.", cfg->enc_transformer_layers, C, P.lstm_attn, P.mlp, c->lstm_u, &c->e_tf));
  QB_TRY(L.f32(&c->e_fnorm_w, "encoder.final_layer_norm.weight")); QB_TRY(L.f32(&c->e_fnorm_b, "encoder.final_layer_norm.bias"));
  QB_TRY(L.conv(&c->e_out, "encoder.out.conv.weight", P.conv));
  QB_TRY(L.f32(&c->e_out_b, "encoder.out.conv.bias"));
  // ---- semantic encoder
  QB_TRY(L.conv(&c->s_conv, "semantic_encoder.conv.conv.weight", P.conv));
  c->s_blocks.resize(cfg->sem_n_blocks);
  for (int i = 0; i < cfg->sem_n_blocks; ++i) {
    const std::string p = "semantic_encoder.conv_blocks." + std::to_string(i) + ".";
    SemBlockW& b = c->s_blocks[i];
    for (int u = 0; u < 2; ++u) {
      QB_TRY(L.conv(&b.u_c1[u], p + "res_units." + std::to_string(u) + ".conv1.conv.weight", P.conv));
      QB_TRY(L.conv(&b.u_c2[u], p + "res_units." + std::to_string(u) + ".conv2.weight", P.conv));
    }
    QB_TRY(L.conv(&b.conv, p + "conv.conv.weight", P.conv, &b.k));
    QB_TRY(L.f32(&b.conv_b, p + "conv.conv.bias"));
    b.stride = cfg->sem_strides[i];
    QB_REQUIRE(b.k == (b.stride == 1 ? 3 : 2 * b.stride), "codec_load: semantic block %d kernel %d does not match stride %d", i, b.k, b.stride);
  }
  QB_TRY(L.conv(&c->s_conv2, "semantic_encoder.conv2.conv.weight", P.conv));
  // ---- decoder
  QB_TRY(L.conv(&c->d_embed, "decoder.embed.conv.weight", P.conv));
  QB_TRY(L.f32(&c->d_embed_b, "decoder.embed.conv.bias"));
  const int res_ids[4] = {0, 1, 5, 6};
  for (int i = 0; i < 4; ++i) {
    const std::string p = "decoder.prior_net." + std::to_string(res_ids[i]) + ".";
    ResnetW& r = c->d_res[i];
    QB_TRY(L.f32(&r.n1w, p + "norm1.weight")); QB_TRY(L.f32(&r.n1b, p + "norm1.bias"));
    QB_TRY(L.f32(&r.n2w, p + "norm2.weight")); QB_TRY(L.f32(&r.n2b, p + "norm2.bias"));
    QB_TRY(L.conv(&r.c1, p + "conv1.conv.weight", P.conv)); QB_TRY(L.f32(&r.c1b, p + "conv1.conv.bias"));
    QB_TRY(L.conv(&r.c2, p + "conv2.conv.weight", P.conv)); QB_TRY(L.f32(&r.c2b, p + "conv2.conv.bias"));
  }
  QB_TRY(load_transformer(L, "decoder.prior_net.3.", cfg->dec_transformer_layers, C, P.lstm_attn, P.mlp_dec, c->lstm_u, &c->d_tf));
  QB_TRY(L.f32(&c->d_gn_w, "decoder.prior_net.7.weight")); QB_TRY(L.f32(&c->d_gn_b, "decoder.prior_net.7.bias"));
  QB_TRY(L.f32(&c->d_norm_w, "decoder.norm.weight")); QB_TRY(L.f32(&c->d_norm_b, "decoder.norm.bias"));
  QB_TRY(load_convnext(L, "decoder.post_net.", cfg->dec_convnext_layers, P.convnext, &c->d_cnx));
  QB_TRY(L.f32(&c->d_fnorm_w, "decoder.final_layer_norm.weight")); QB_TRY(L.f32(&c->d_fnorm_b, "decoder.final_layer_norm.bias"));
  QB_TRY(L.lin(&c->d_head, "decoder.head.out.weight", P.head));
  QB_TRY(L.f32(&c->d_head_b, "decoder.head.out.bias"));
  // ---- quantisers: codebooks quantizer.layers.{i}._codebook.embed [1, K, D]
  const char* qn[2] = {"quantizer", "semantic_quantizer"};
  for (int w = 0; w < 2; ++w) {
    const int nq = cfg->num_quantizers, K = cfg->codebook_size, D = cfg->dimension;
    float* tmp;
    QB_CHECK_CUDA(cudaMalloc(&tmp, (size_t)nq * K * D * 4));
    int e = 0;
    for (int i = 0; i < nq && !e; ++i) {
      const qb_tensor* t = wt.find(std::string(qn[w]) + ".layers." + std::to_string(i) + "._codebook.embed");
      if (!t || numel(t) != (long long)K * D) { set_error("codec_load: missing / mis-shaped codebook %s layer %d", qn[w], i); e = -1; break; }
      if (cudaMemcpy(tmp + (size_t)i * K * D, t->data, (size_t)K * D * 4, cudaMemcpyDeviceToDevice) != cudaSuccess) { set_error("codec_load: codebook copy failed"); e = -2; }
    }
    if (!e) e = rvq_build(h, tmp, nq, K, D, true, &c->q[w]);
    cudaFree(tmp);
    QB_TRY(e);
  }
  QB_CHECK_CUDA(cudaDeviceSynchronize());
  QB_CHECK_CUDA(cudaGetLastError());
  guard.c = nullptr;
  *out = c;
  return 0;
}

extern "C" void qb_codec_free(qb_codec* c) {
  if (!c) return;
  delete c->q[0];
  delete c->q[1];
  delete c;
}
extern "C" int qb_codec_set_tap(qb_codec* c, qb_tap_fn cb, void* user) {
  QB_REQUIRE(c != nullptr, "codec_set_tap: null codec");
  c->tap = cb; c->tap_user = user;
  return 0;
}
extern "C" qb_rvq* qb_codec_rvq(qb_codec* c, int32_t which) { return c && which >= 0 && which < 2 ? c->q[which] : nullptr; }

extern "C" int qb_codec_encode(qb_codec* c, const float* wav, int64_t B, int64_t T, const float* feat, int64_t* ac_codes,
                               int64_t* sem_codes, void* stream) {
  QB_REQUIRE(c && wav && feat && ac_codes && sem_codes && B >= 1, "codec_encode: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  float *emb, *sem;
  int64_t N, Ns;
  QB_TRY(encode_emb(c, wav, B, T, &emb, &N, stream));
  QB_TRY(encode_sem(c, feat, B, T / c->cfg.hop_length, &sem, &Ns, stream));
  QB_REQUIRE(Ns == N, "codec_encode: semantic stream has %lld frames but the acoustic stream has %lld", (long long)Ns, (long long)N);
  const int nq = c->cfg.num_quantizers;
  int64_t* rows;
  QB_TRY(c->ws.get((void**)&rows, "codes_rows", (size_t)B * N * nq * 8));
  const long long total = (long long)B * N * nq;
  QB_TRY(qb_rvq_encode_rows(c->q[0], emb, B * N, rows, nullptr, stream));
  codes_rows_to_bqn_kernel<<<grid_for(total), 256, 0, st>>>(rows, (int)B, (int)N, nq, ac_codes);
  g_launches++;
  QB_TRY(qb_rvq_encode_rows(c->q[1], sem, B * N, rows, nullptr, stream));
  codes_rows_to_bqn_kernel<<<grid_for(total), 256, 0, st>>>(rows, (int)B, (int)N, nq, sem_codes);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qb_codec_decode(qb_codec* c, const int64_t* ac_codes, const int64_t* sem_codes, int64_t B, int64_t N, float* wav,
                               void* stream) {
  QB_REQUIRE(c && ac_codes && sem_codes && wav && B >= 1 && N >= 1, "codec_decode: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int nq = c->cfg.num_quantizers, Dq = c->cfg.dimension;
  QB_REQUIRE(c->cfg.dec_input_channels == 2 * Dq, "codec_decode: decoder input_channels must be 2 x the quantiser dim");
  int64_t* rows;
  float* z;
  QB_TRY(c->ws.get((void**)&rows, "codes_rows", (size_t)B * N * nq * 8));
  QB_TRY(c->ws.f32(&z, "dec_z", (size_t)B * N * 2 * Dq));
  const long long total = (long long)B * N * nq;
  codes_bqn_to_rows_kernel<<<grid_for(total), 256, 0, st>>>(ac_codes, (int)B, (int)N, nq, rows);
  g_launches++;
  QB_TRY(qb_rvq_decode(rows, c->q[0]->cb, B * N, Dq, c->cfg.codebook_size, nq, z, 2 * Dq, 0, stream));
  codes_bqn_to_rows_kernel<<<grid_for(total), 256, 0, st>>>(sem_codes, (int)B, (int)N, nq, rows);
  g_launches++;
  QB_TRY(qb_rvq_decode(rows, c->q[1]->cb, B * N, Dq, c->cfg.codebook_size, nq, z, 2 * Dq, Dq, stream));
  return decode_z(c, z, B, N, wav, stream);
}

extern "C" int qb_codec_load_semantic_decoder(qb_codec* c, const qb_semantic_decoder_cfg* cfg, const qb_tensor* named, int32_t n) {
  QB_REQUIRE(c && cfg && named && n > 0, "codec_load_semantic_decoder: bad args");
  QB_REQUIRE(!c->has_sdec, "codec_load_semantic_decoder: this codec already holds a semantic decoder");
  QB_REQUIRE(cfg->n_blocks >= 0 && cfg->n_blocks <= 8 && cfg->code_dim > 0 && cfg->output_channels > 0,
             "codec_load_semantic_decoder: n_blocks must be in [0, 8]");
  QB_CHECK_CUDA(cudaSetDevice(c->h->device));
  WeightTable wt;
  QB_TRY(wt.init(named, n));
  Loader L(wt, c->arena);
  const bool pc = c->pol.conv;
  const std::string p = "semantic_decoder.";
  const qb_tensor* t;
  QB_TRY(L.get(&t, p + "conv1.conv.weight", 3));
  QB_REQUIRE(t->shape[1] == cfg->code_dim && t->shape[2] == 3, "codec_load_semantic_decoder: conv1 must be [C, code_dim %d, 3]", cfg->code_dim);
  c->sd_code_dim = cfg->code_dim;
  c->sd_c0 = (int)t->shape[0];
  QB_TRY(L.conv(&c->sd_conv1, p + "conv1.conv.weight", pc));
  std::vector<SemDecBlockW> blocks(cfg->n_blocks);
  int cin = c->sd_c0;
  for (int i = 0; i < cfg->n_blocks; ++i) {
    const std::string b = p + "conv_blocks." + std::to_string(i) + ".";
    SemDecBlockW& w = blocks[i];
    w.stride = cfg->strides[i];
    QB_REQUIRE(w.stride >= 1, "codec_load_semantic_decoder: block %d stride %d", i, w.stride);
    if (w.stride == 1) {
      QB_TRY(L.get(&t, b + "conv.conv.weight", 3));
      QB_REQUIRE(t->shape[1] == cin && t->shape[2] == 3, "codec_load_semantic_decoder: block %d conv must be [Cout, %d, 3]", i, cin);
      w.cout = (int)t->shape[0];
      QB_TRY(L.conv(&w.conv, b + "conv.conv.weight", pc));
      QB_TRY(L.f32(&w.b, b + "conv.conv.bias"));
    } else {
      const int s = w.stride;
      QB_TRY(L.get(&t, b + "conv.deconv.weight", 3));
      QB_REQUIRE(t->shape[0] == cin && t->shape[2] == 2 * s, "codec_load_semantic_decoder: block %d deconv must be [%d, Cout, %d]", i, cin, 2 * s);
      w.cout = (int)t->shape[1];
      const int Cpad = (int)pad_to(cin, 64), J = 2;
      const long long nel = (long long)s * w.cout * J * Cpad;
      QB_TRY(c->arena.alloc((void**)&w.conv.hi, (size_t)nel * 2, false));
      w.conv.lo = nullptr;
      if (pc) QB_TRY(c->arena.alloc((void**)&w.conv.lo, (size_t)nel * 2, false));
      repack_convt_kernel<<<grid_for(nel), 256>>>(t->data, cin, w.cout, 2 * s, s, J, Cpad, w.conv.hi, w.conv.lo);
      QB_CHECK_CUDA(cudaGetLastError());
      const qb_tensor* bt;
      QB_TRY(L.get(&bt, b + "conv.deconv.bias", 1));
      QB_REQUIRE(bt->shape[0] == w.cout, "codec_load_semantic_decoder: block %d deconv bias must have %d entries", i, w.cout);
      std::vector<float> hb(w.cout), rep((size_t)s * w.cout);
      QB_CHECK_CUDA(cudaMemcpy(hb.data(), bt->data, (size_t)w.cout * 4, cudaMemcpyDeviceToHost));
      for (int r = 0; r < s; ++r) std::copy(hb.begin(), hb.end(), rep.begin() + (size_t)r * w.cout);
      float* db;
      QB_TRY(c->arena.alloc((void**)&db, rep.size() * 4, false));
      QB_CHECK_CUDA(cudaMemcpy(db, rep.data(), rep.size() * 4, cudaMemcpyHostToDevice));
      w.b = db;
    }
    for (int u = 0; u < 2; ++u) {
      const std::string r = b + "res_units." + std::to_string(u) + ".";
      QB_TRY(L.get(&t, r + "conv1.conv.weight", 3));
      QB_REQUIRE(t->shape[0] == w.cout && t->shape[1] == w.cout && t->shape[2] == 3, "codec_load_semantic_decoder: %sconv1 shape", r.c_str());
      QB_TRY(L.conv(&w.u_c1[u], r + "conv1.conv.weight", pc));
      QB_TRY(L.get(&t, r + "conv2.weight", 3));
      QB_REQUIRE(t->shape[0] == w.cout && t->shape[1] == w.cout && t->shape[2] == 1, "codec_load_semantic_decoder: %sconv2 shape", r.c_str());
      QB_TRY(L.conv(&w.u_c2[u], r + "conv2.weight", pc));
    }
    cin = w.cout;
  }
  QB_TRY(L.get(&t, p + "conv2.conv.weight", 3));
  QB_REQUIRE(t->shape[0] == cfg->output_channels && t->shape[1] == cin && t->shape[2] == 3,
             "codec_load_semantic_decoder: conv2 must be [%d, %d, 3]", cfg->output_channels, cin);
  QB_TRY(L.conv(&c->sd_conv2, p + "conv2.conv.weight", pc));
  c->sd_out = cfg->output_channels;
  c->sd_blocks = blocks;
  QB_CHECK_CUDA(cudaDeviceSynchronize());
  c->has_sdec = true;
  return 0;
}

extern "C" int qb_codec_semantic_decode(qb_codec* c, const int64_t* sem_codes, int64_t B, int64_t N, float* pred_feat, void* stream) {
  QB_REQUIRE(c && sem_codes && pred_feat && B >= 1 && N >= 1, "codec_semantic_decode: bad args");
  QB_REQUIRE(c->has_sdec, "codec_semantic_decode: no semantic decoder loaded (qb_codec_load_semantic_decoder)");
  QB_REQUIRE(c->sd_code_dim == c->cfg.dimension, "codec_semantic_decode: decoder code_dim %d != quantiser dim %d", c->sd_code_dim,
             c->cfg.dimension);
  cudaStream_t st = (cudaStream_t)stream;
  const int nq = c->cfg.num_quantizers, Dq = c->cfg.dimension;
  int64_t* rows;
  float* z;
  QB_TRY(c->ws.get((void**)&rows, "codes_rows", (size_t)B * N * nq * 8));
  QB_TRY(c->ws.f32(&z, "sd_zrows", (size_t)B * N * Dq));
  codes_bqn_to_rows_kernel<<<grid_for((long long)B * N * nq), 256, 0, st>>>(sem_codes, (int)B, (int)N, nq, rows);
  g_launches++;
  QB_CHECK_CUDA(cudaGetLastError());
  QB_TRY(qb_rvq_decode(rows, c->q[1]->cb, B * N, Dq, c->cfg.codebook_size, nq, z, Dq, 0, stream));
  return semantic_decode_z(c, z, B, N, pred_feat, stream);
}
