// T5 encoder: Hugging Face T5EncoderModel (transformers models/t5/modeling_t5.py), the module the reference's
// T5Conditioner wraps (reference models/conditioners.py T5Conditioner), on this library's kernels.
//
// Tokens are packed.  The B prompts of one call lie back to back as M = sum of their lengths rows: item b holds rows
// [off[b], off[b + 1]), off computed on the host from the lengths.  No row is computed for padding.  In the reference
// the padded positions are masked keys (their scores get the dtype's minimum) and the conditioner multiplies their
// output rows by zero, so nothing a valid position computes depends on them: the packed encoder is exact there.
//
// Residual stream fp32 [M, d_model]; GEMM operands 16-bit (fp16 or bf16), fp32 accumulation.  One encode:
//   embedding gather                                   t5_embed_kernel
//   per block:  RMSNorm -> 16-bit                      t5_rmsnorm_kernel
//               QKV  [M, 3 inner]                      GEMM, EpiStore16 (q | k | v rows of one fused weight)
//               attention core [M, inner]              t5_attn_kernel<d_kv>
//               h += o-projection                      GEMM, EpiResidual
//               RMSNorm -> 16-bit                      t5_rmsnorm_kernel
//               FF-in [M, d_ff]                        GEMM, EpiRelu16 (relu) / EpiGeglu16 (gated-gelu)
//               h += FF-out                            GEMM, EpiResidual
//   final RMSNorm (-> fp32, or -> 16-bit and proj_out: GEMM, EpiStore32 with bias), scatter to [B, L, out] with
//   zero rows at the padding                           t5_scatter_kernel
// 3 + 7 num_layers launches without proj_out, 4 + 7 num_layers with it (88 for t5-base with proj_out), all with
// programmatic dependent launch.  The relative-position bias table [H, 2 kT5MaxLen - 1] is built once, at finalize,
// from block 0's relative_attention_bias and the bucket of every relative position, which the caller computes with
// T5Attention._relative_position_bucket itself (satb_t5_set_buckets): no float log inside a kernel can move a bucket
// boundary.
//
// Deliberate deviations from the reference, whose whole model is cast to fp16: the residual stream is fp32 (the
// reference's fp16 stream relies on HF's clamp of fp16 infinities, modeling_t5.py:451-456), and the 16-bit stores of
// the RMSNorm and FF-in activations saturate at +-65504 in fp16 instead of overflowing (gemm.cuh pack16_satfinite).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/satb200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.h"
#include "linear.cuh"
#include "mma_tile.cuh"
#include "ptx.cuh"

namespace satb {
namespace {

constexpr int kT5MaxLen = 512;                   // longest prompt (max_length) an encode accepts
constexpr int kT5BiasSpan = 2 * kT5MaxLen - 1;   // relative positions -(kT5MaxLen - 1) .. kT5MaxLen - 1
constexpr int kT5MaxDim = 4096;                  // d_model
constexpr int kNormThreads = 128;
constexpr int kNormVec = kT5MaxDim / 4 / kNormThreads;   // float4 per thread at the widest row

// Item of packed row m: the b with off[b] <= m < off[b + 1] (off nondecreasing, off[0] = 0).
__device__ __forceinline__ int item_of_row(const int* off, int B, int m) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= m) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// h[m, :] = emb[id, :] for packed row m (item b, position t = m - off[b]), id = ids[b L + t] clamped to the table:
// the host refuses ids outside [0, vocab), and no input makes this kernel read outside the table.
__global__ void __launch_bounds__(kNormThreads) t5_embed_kernel(const long long* ids, const int* off, int B, int L,
                                                                 const float* emb, int vocab, int D, float* h) {
  pdl_launch_dependents();
  pdl_wait();
  const int m = blockIdx.x;
  const int b = item_of_row(off, B, m);
  long long id = ids[static_cast<size_t>(b) * L + (m - off[b])];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const float4* src = reinterpret_cast<const float4*>(emb + static_cast<size_t>(id) * D);
  float4* dst = reinterpret_cast<float4*>(h + static_cast<size_t>(m) * D);
  for (int c = threadIdx.x; c < D / 4; c += kNormThreads) dst[c] = __ldg(src + c);
}

// T5LayerNorm (modeling_t5.py:46-68): y = w * (x * rsqrt(mean(x^2) + eps)), fp32 statistics over the row held in
// registers.  OUT 0: fp16 (saturating), 1: bf16, 2: fp32.  One CTA per row; D a multiple of 4, at most kT5MaxDim.
template <int OUT>
__global__ void __launch_bounds__(kNormThreads) t5_rmsnorm_kernel(const float* x, const float* w, void* out, int D,
                                                                   float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[kNormThreads / 32];
  const int row = blockIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
  float4 v[kNormVec];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kNormVec; ++i) {
    const int c = threadIdx.x + i * kNormThreads;
    v[i] = c < D / 4 ? xr[c] : make_float4(0.f, 0.f, 0.f, 0.f);
    ss = fmaf(v[i].x, v[i].x, ss);
    ss = fmaf(v[i].y, v[i].y, ss);
    ss = fmaf(v[i].z, v[i].z, ss);
    ss = fmaf(v[i].w, v[i].w, ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < kNormThreads / 32; ++i) tot += red[i];
  const float r = rsqrtf(tot / static_cast<float>(D) + eps);
  const float4* wr = reinterpret_cast<const float4*>(w);
#pragma unroll
  for (int i = 0; i < kNormVec; ++i) {
    const int c = threadIdx.x + i * kNormThreads;
    if (c >= D / 4) break;
    const float4 g = __ldg(wr + c);
    const float4 y = make_float4(g.x * (v[i].x * r), g.y * (v[i].y * r), g.z * (v[i].z * r), g.w * (v[i].w * r));
    if constexpr (OUT == 2) {
      reinterpret_cast<float4*>(static_cast<float*>(out) + static_cast<size_t>(row) * D)[c] = y;
    } else {
      reinterpret_cast<uint2*>(static_cast<uint16_t*>(out) + static_cast<size_t>(row) * D)[c] =
          make_uint2(pack16_satfinite<OUT == 1>(y.x, y.y), pack16_satfinite<OUT == 1>(y.z, y.w));
    }
  }
}

// tab[h, d] = rel[bucket[d], h]: the bias of relative position d - (kT5MaxLen - 1) for head h (T5Attention.compute_bias,
// modeling_t5.py:236-251; rel is relative_attention_bias.weight [num_buckets, H]).  Buckets are clamped to the table.
__global__ void t5_bias_table_kernel(const float* rel, const int* bucket, int nb, int H, float* tab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * kT5BiasSpan) return;
  const int h = i / kT5BiasSpan, d = i - h * kT5BiasSpan;
  int bk = bucket[d];
  bk = bk < 0 ? 0 : (bk >= nb ? nb - 1 : bk);
  tab[i] = rel[static_cast<size_t>(bk) * H + h];
}

// out[b, t, :] = t < len_b ? src[off[b] + t, :] : 0 for every (b, t) of the padded [B, L, n] output.  src may be null
// (every item empty).  n a multiple of 4.
__global__ void __launch_bounds__(kNormThreads) t5_scatter_kernel(const float* src, const int* off, int L, int n,
                                                                   float* out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x / L, t = blockIdx.x - b * L;
  const int start = off[b], len = off[b + 1] - start;
  float4* dst = reinterpret_cast<float4*>(out + static_cast<size_t>(blockIdx.x) * n);
  if (t < len) {
    const float4* s = reinterpret_cast<const float4*>(src + static_cast<size_t>(start + t) * n);
    for (int c = threadIdx.x; c < n / 4; c += kNormThreads) dst[c] = s[c];
  } else {
    for (int c = threadIdx.x; c < n / 4; c += kNormThreads) dst[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// ---- attention core: O = softmax(Q K^T + bias[h, j - i]) V per (item, head), T5Attention.forward
// (modeling_t5.py:253-340) on packed rows, with no 1 / sqrt(d) scale (T5 folds it into the q weights' initialisation).
// One CTA of four warps per (64-query tile, head, item) runs mma_tile.cuh's mma.sync core (mma_attention) over the
// keys of the item only, with the bias row of the head (kT5BiasSpan fp32) staged in shared memory.  mma.sync rather
// than wgmma: a prompt holds at most 512 keys and usually 10 - 40, so the CTA tile is 64 queries (a wgmma consumer
// warpgroup would want 128 and leave most rows empty), and there is no key stream long enough for a producer /
// consumer ring to hide anything.  Rows past the item's length are computed on zero queries and never stored.

// (s + bias of relative position key - query) in log2 units, from the head's bias row in shared memory.  Query rows
// past the item use the last row's entries: in range, and never stored.
struct T5BiasScore {
  const float* sbias;   // [kT5BiasSpan]
  int last;             // the item's last row
  __device__ __forceinline__ float operator()(float s, int query, int key) const {
    return (s + sbias[key - min(query, last) + kT5MaxLen - 1]) * 1.4426950408889634f;
  }
};

// qkv [M, 3 inner]: q of head h at column h D, k at inner + h D, v at 2 inner + h D; o [M, inner]; off [B + 1];
// bias [H, kT5BiasSpan]
template <int D, bool BF16>
__global__ void __launch_bounds__(kMmaAttnThreads) t5_attn_kernel(const uint16_t* qkv, uint16_t* o, const int* off,
                                                                   const float* bias, int inner) {
  extern __shared__ __align__(128) uint16_t smem_t5[];
  __shared__ float sbias[kT5BiasSpan];
  pdl_launch_dependents();
  pdl_wait();   // qkv is written by the previous kernel
  const int q0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z;
  const int start = off[b], n = off[b + 1] - start;
  if (q0 >= n) return;
  {   // bias entries of relative positions j - i, i in [q0, min(q0 + 63, n - 1)], j in [0, n), by cp.async: they join
      // mma_attention's first copy group, so their fetch overlaps that of the first Q / K / V tiles
    const float* brow = bias + static_cast<size_t>(h) * kT5BiasSpan;
    const int lo = kT5MaxLen - 1 - min(q0 + 63, n - 1), hi = kT5MaxLen - 1 + n - 1;
    for (int i = lo + threadIdx.x; i <= hi; i += kMmaAttnThreads) cp_async4(smem_u32(sbias + i), brow + i);
  }
  const int64_t ld = 3LL * inner;
  const uint16_t* base = qkv + start * ld;
  mma_attention<D, BF16>(smem_t5, base, ld, h * D, base, ld, inner + h * D, base, ld, 2 * inner + h * D,
                         o + static_cast<int64_t>(start) * inner, inner, h * D, q0, n, n, T5BiasScore{sbias, n - 1});
}

}  // namespace

// ---- launchers (also the probes' path)
static int launch_t5_rmsnorm(const float* x, const float* w, void* out, int rows, int D, float eps, int out_kind,
                             cudaStream_t st) {
  SATB_REQUIRE(D >= 4 && D % 4 == 0 && D <= kT5MaxDim, "T5 RMSNorm: D must be a multiple of 4, at most 4096");
  SATB_REQUIRE(out_kind >= 0 && out_kind <= 2, "T5 RMSNorm: out_kind must be 0 (fp16), 1 (bf16) or 2 (fp32)");
  if (rows <= 0) return 0;
  if (out_kind == 0) SATB_CHECK_CUDA(launch_pdl(t5_rmsnorm_kernel<0>, dim3(rows), dim3(kNormThreads), 0, st, x, w, out, D, eps));
  else if (out_kind == 1) SATB_CHECK_CUDA(launch_pdl(t5_rmsnorm_kernel<1>, dim3(rows), dim3(kNormThreads), 0, st, x, w, out, D, eps));
  else SATB_CHECK_CUDA(launch_pdl(t5_rmsnorm_kernel<2>, dim3(rows), dim3(kNormThreads), 0, st, x, w, out, D, eps));
  count_launch();
  return 0;
}

// qkv [M, 3 H dk], o [M, H dk] (M = off[B]), bias [H, kT5BiasSpan]; max_len >= every item's length
static int launch_t5_attention(const void* qkv, const float* bias, const int* off_dev, int B, int max_len, int H,
                               int dk, bool bf16, void* o, cudaStream_t st) {
  SATB_REQUIRE(dk == 64 || dk == 128, "T5 attention: d_kv must be 64 or 128");
  if (B <= 0 || max_len <= 0) return 0;
  const dim3 grid(ceil_div(max_len, 64), H, B);
  SATB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "T5 attention grid too large");
  const uint16_t* q = static_cast<const uint16_t*>(qkv);
  uint16_t* out = static_cast<uint16_t*>(o);
  const int inner = H * dk;
  if (dk == 64)
    SATB_PROPAGATE((bf16 ? launch_mma_attention<t5_attn_kernel<64, true>, 64>(grid, st, q, out, off_dev, bias, inner)
                         : launch_mma_attention<t5_attn_kernel<64, false>, 64>(grid, st, q, out, off_dev, bias, inner)));
  else
    SATB_PROPAGATE((bf16 ? launch_mma_attention<t5_attn_kernel<128, true>, 128>(grid, st, q, out, off_dev, bias, inner)
                         : launch_mma_attention<t5_attn_kernel<128, false>, 128>(grid, st, q, out, off_dev, bias, inner)));
  count_launch();
  return 0;
}

// C[M, N] = A[M, K] W[N, K]^T through Epi; A's tensor map spans a_rows >= M rows (the workspace's capacity, so that one
// map serves every M), the tiles cover M.
template <class Epi, bool BF16>
static int t5_linear(TmapCache& tc, const void* A, int a_rows, int M, int K, const void* W, int N,
                     const typename Epi::Params& ep, cudaStream_t st, int bn = 0) {
  if (M <= 0) return 0;
  if (bn == 0) bn = auto_bn(ceil_div(M, kBlockM), N);
  const CUtensorMap *ta, *tb;
  SATB_PROPAGATE(tc.get_a(A, K, a_rows, 1, K, static_cast<int64_t>(a_rows) * K, &ta));
  SATB_PROPAGATE(tc.get_b(W, K, N, K, bn, &tb));
  GemmShape s;
  s.L = M; s.batches = 1; s.N = N; s.K = K; s.n_taps = 1; s.tap_base = 0; s.tap_step = 0; s.b_tap_rows = N; s.stride = 1;
  s.b_static = 1;
  if (bn == 128) return launch_gemm<Epi, 128, BF16>(*ta, *tb, s, ep, st);
  return launch_gemm<Epi, 256, BF16>(*ta, *tb, s, ep, st);
}

struct T5Layer {
  float *ln0 = nullptr, *ln1 = nullptr;
  uint16_t *w_qkv = nullptr, *w_o = nullptr, *w_fi = nullptr, *w_fo = nullptr;
};

}  // namespace satb

using namespace satb;

struct SatbT5 {
  SatbT5Config cfg;
  int D, H, dk, inner, dff, depth;
  bool gated, bf16;
  float* emb = nullptr;
  float* rel = nullptr;       // block 0's relative_attention_bias.weight [num_buckets, H]
  float* ln_f = nullptr;
  std::vector<T5Layer> layers;
  uint16_t* w_proj = nullptr;
  float* b_proj = nullptr;
  int out_dim = 0;            // 0: no proj_out
  int* bucket = nullptr;      // [kT5BiasSpan] (satb_t5_set_buckets)
  float* bias_tab = nullptr;  // [H, kT5BiasSpan] (finalize)
  std::map<std::string, int> loaded;
  bool finalized = false;
  std::vector<void*> owned;
  TmapCache tmaps;
  DevBuf ws_h, ws_a16, ws_qkv, ws_attn, ws_ff, ws_y, ws_off;
  int cap = 0;                // rows the workspaces hold
  std::vector<int> off;       // host copy of the last encode's offsets

  template <class T>
  int alloc(T** p, size_t n) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, n * sizeof(T) < 256 ? 256 : n * sizeof(T));
    if (e != cudaSuccess) {
      set_last_error(std::string("cudaMalloc failed: ") + cudaGetErrorString(e));
      return -2;
    }
    owned.push_back(q);
    *p = static_cast<T*>(q);
    return 0;
  }
};

static int t5_reserve(SatbT5* t, int rows) {
  if (rows <= t->cap) return 0;
  const int cap = std::max(rows, 2 * t->cap);
  const size_t r = static_cast<size_t>(cap);
  const int ffw = t->dff;
  SATB_PROPAGATE(t->ws_h.ensure(r * t->D * 4));
  SATB_PROPAGATE(t->ws_a16.ensure(r * t->D * 2));
  SATB_PROPAGATE(t->ws_qkv.ensure(r * 3 * t->inner * 2));
  SATB_PROPAGATE(t->ws_attn.ensure(r * t->inner * 2));
  SATB_PROPAGATE(t->ws_ff.ensure(r * ffw * 2));
  SATB_PROPAGATE(t->ws_y.ensure(r * std::max(t->D, t->out_dim) * 4));
  t->tmaps.maps.clear();   // the maps span the old buffers
  t->cap = cap;
  return 0;
}

template <bool BF16>
static int t5_encode_impl(SatbT5* t, const long long* ids, int B, int L, int M, int max_len, float* out, cudaStream_t st) {
  const int D = t->D, inner = t->inner, dff = t->dff, cap = t->cap;
  const int* off = t->ws_off.as<int>();
  float* h = t->ws_h.as<float>();
  uint16_t* a16 = t->ws_a16.as<uint16_t>();
  uint16_t* qkv = t->ws_qkv.as<uint16_t>();
  uint16_t* att = t->ws_attn.as<uint16_t>();
  uint16_t* ff = t->ws_ff.as<uint16_t>();
  float* y = t->ws_y.as<float>();
  const float eps = t->cfg.layer_norm_epsilon;
  const int o16 = BF16 ? 1 : 0;
  SATB_CHECK_CUDA(launch_pdl(t5_embed_kernel, dim3(M), dim3(kNormThreads), 0, st, ids, off, B, L,
                             static_cast<const float*>(t->emb), t->cfg.vocab_size, D, h));
  count_launch();
  for (int li = 0; li < t->depth; ++li) {
    const T5Layer& W = t->layers[li];
    SATB_PROPAGATE(launch_t5_rmsnorm(h, W.ln0, a16, M, D, eps, o16, st));
    SATB_PROPAGATE((t5_linear<EpiStore16<BF16>, BF16>(t->tmaps, a16, cap, M, D, W.w_qkv, 3 * inner,
                                                      typename EpiStore16<BF16>::Params{qkv, 3 * inner, nullptr, 0}, st)));
    SATB_PROPAGATE(launch_t5_attention(qkv, t->bias_tab, off, B, max_len, t->H, t->dk, BF16, att, st));
    const EpiResidual::Params res{h, D, nullptr, nullptr, 1, 0, 1};
    SATB_PROPAGATE((t5_linear<EpiResidual, BF16>(t->tmaps, att, cap, M, inner, W.w_o, D, res, st)));
    SATB_PROPAGATE(launch_t5_rmsnorm(h, W.ln1, a16, M, D, eps, o16, st));
    if (t->gated)
      SATB_PROPAGATE((t5_linear<EpiGeglu16<BF16>, BF16>(t->tmaps, a16, cap, M, D, W.w_fi, 2 * dff,
                                                        typename EpiGeglu16<BF16>::Params{ff, dff}, st)));
    else
      SATB_PROPAGATE((t5_linear<EpiRelu16<BF16>, BF16>(t->tmaps, a16, cap, M, D, W.w_fi, dff,
                                                       typename EpiRelu16<BF16>::Params{ff, dff}, st)));
    SATB_PROPAGATE((t5_linear<EpiResidual, BF16>(t->tmaps, ff, cap, M, dff, W.w_fo, D, res, st)));
  }
  int n_out = D;
  if (t->out_dim > 0) {
    SATB_PROPAGATE(launch_t5_rmsnorm(h, t->ln_f, a16, M, D, eps, o16, st));
    SATB_PROPAGATE((t5_linear<EpiStore32, BF16>(t->tmaps, a16, cap, M, D, t->w_proj, t->out_dim,
                                                EpiStore32::Params{y, t->out_dim, t->b_proj}, st)));
    n_out = t->out_dim;
  } else {
    SATB_PROPAGATE(launch_t5_rmsnorm(h, t->ln_f, y, M, D, eps, 2, st));
  }
  SATB_CHECK_CUDA(launch_pdl(t5_scatter_kernel, dim3(B * L), dim3(kNormThreads), 0, st, static_cast<const float*>(y),
                             off, L, n_out, out));
  count_launch();
  return 0;
}

// Offsets of the packed rows from the host lengths; checks every length against L.
static int t5_offsets(const int* lengths, int B, int L, std::vector<int>* off, int* max_len) {
  off->assign(B + 1, 0);
  *max_len = 0;
  for (int b = 0; b < B; ++b) {
    SATB_REQUIRE(lengths[b] >= 0 && lengths[b] <= L, "T5: every length must lie in [0, L]");
    (*off)[b + 1] = (*off)[b] + lengths[b];
    *max_len = std::max(*max_len, lengths[b]);
  }
  return 0;
}

extern "C" {

int satb_t5_create(const SatbT5Config* cfg, SatbT5** out) {
  SATB_REQUIRE(cfg && out, "null argument");
  const SatbT5Config& c = *cfg;
  SATB_REQUIRE(c.d_kv == 64 || c.d_kv == 128, "T5: d_kv must be 64 or 128");
  SATB_REQUIRE(c.feed_forward_proj == SATB_T5_FF_RELU || c.feed_forward_proj == SATB_T5_FF_GATED_GELU,
               "T5: feed_forward_proj must be relu (0) or gated-gelu (1)");
  SATB_REQUIRE(c.d_model >= 128 && c.d_model % 128 == 0 && c.d_model <= kT5MaxDim,
               "T5: d_model must be a multiple of 128, at most 4096");
  SATB_REQUIRE(c.num_heads >= 1 && c.num_heads <= 1024, "T5: num_heads must be >= 1");
  SATB_REQUIRE(c.d_ff >= 32 && c.d_ff % 32 == 0, "T5: d_ff must be a positive multiple of 32");
  SATB_REQUIRE(c.num_layers >= 1 && c.vocab_size >= 1, "T5: need num_layers >= 1 and vocab_size >= 1");
  SATB_REQUIRE(c.relative_attention_num_buckets >= 2, "T5: need relative_attention_num_buckets >= 2");
  SATB_REQUIRE(c.layer_norm_epsilon >= 0.f, "T5: layer_norm_epsilon must not be negative");
  SATB_REQUIRE(c.operand_dtype == 0 || c.operand_dtype == 1, "T5: operand_dtype must be 0 (fp16) or 1 (bf16)");
  SatbT5* t = new SatbT5();
  t->cfg = c;
  t->D = c.d_model;
  t->H = c.num_heads;
  t->dk = c.d_kv;
  t->inner = c.num_heads * c.d_kv;
  t->dff = c.d_ff;
  t->depth = c.num_layers;
  t->gated = c.feed_forward_proj == SATB_T5_FF_GATED_GELU;
  t->bf16 = c.operand_dtype == 1;
  t->layers.resize(c.num_layers);
  *out = t;
  return 0;
}

void satb_t5_destroy(SatbT5* t) {
  if (!t) return;
  cudaDeviceSynchronize();
  for (void* p : t->owned) cudaFree(p);
  for (DevBuf* b : {&t->ws_h, &t->ws_a16, &t->ws_qkv, &t->ws_attn, &t->ws_ff, &t->ws_y, &t->ws_off}) b->release();
  delete t;
}

// One T5EncoderModel state-dict entry by its HF key; src: device fp32, contiguous.  Matrices are cast to the 16-bit
// operand type here; q, k, v go to the row ranges of the fused QKV weight, wi_1 / wi_0 to the value / gate rows of
// EpiGeglu16's interleave (every 64 rows: 32 of wi_1, the same 32 of wi_0).
int satb_t5_load_weight(SatbT5* t, const char* name_c, const float* src, long long numel, void* stream_v) {
  SATB_REQUIRE(t && name_c && src, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  const std::string name(name_c);
  const int D = t->D, inner = t->inner, dff = t->dff;
  auto copy_f32 = [&](float** dst, long long expect) -> int {
    SATB_REQUIRE(numel == expect, ("bad size for " + name).c_str());
    if (!*dst) SATB_PROPAGATE(t->alloc(dst, expect));
    SATB_CHECK_CUDA(cudaMemcpyAsync(*dst, src, expect * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
  };
  // rows x cols of src into the stored matrix *dst (total_rows x cols) at row `row0`, every `group` rows of src
  // `stride` rows apart (group 0: contiguous)
  auto cast16 = [&](uint16_t** dst, long long total_rows, int rows, int cols, long long row0, int group, int stride) -> int {
    SATB_REQUIRE(numel == static_cast<long long>(rows) * cols, ("bad size for " + name).c_str());
    if (!*dst) SATB_PROPAGATE(t->alloc(dst, static_cast<size_t>(total_rows) * cols));
    uint16_t* d = *dst + static_cast<size_t>(row0) * cols;
    if (group == 0) return launch_cast_rows(src, d, nullptr, rows, cols, cols, cols, t->bf16, st);
    return launch_cast_rows(src, d, nullptr, rows / group, group * cols, static_cast<int64_t>(group) * cols,
                            static_cast<int64_t>(stride) * cols, t->bf16, st);
  };
  t->finalized = false;
  t->loaded[name] = 1;
  if (name == "shared.weight" || name == "encoder.embed_tokens.weight")
    return copy_f32(&t->emb, static_cast<long long>(t->cfg.vocab_size) * D);
  if (name == "encoder.final_layer_norm.weight") return copy_f32(&t->ln_f, D);
  if (name == "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight")
    return copy_f32(&t->rel, static_cast<long long>(t->cfg.relative_attention_num_buckets) * t->H);
  const std::string lp = "encoder.block.";
  if (name.compare(0, lp.size(), lp) == 0) {
    const size_t dot = name.find('.', lp.size());
    SATB_REQUIRE(dot != std::string::npos, ("bad key " + name).c_str());
    const int li = atoi(name.substr(lp.size(), dot - lp.size()).c_str());
    SATB_REQUIRE(li >= 0 && li < t->depth, ("layer index out of range in " + name).c_str());
    T5Layer& L = t->layers[li];
    const std::string k = name.substr(dot + 1);
    if (k == "layer.0.layer_norm.weight") return copy_f32(&L.ln0, D);
    if (k == "layer.1.layer_norm.weight") return copy_f32(&L.ln1, D);
    if (k == "layer.0.SelfAttention.q.weight") return cast16(&L.w_qkv, 3LL * inner, inner, D, 0, 0, 0);
    if (k == "layer.0.SelfAttention.k.weight") return cast16(&L.w_qkv, 3LL * inner, inner, D, inner, 0, 0);
    if (k == "layer.0.SelfAttention.v.weight") return cast16(&L.w_qkv, 3LL * inner, inner, D, 2LL * inner, 0, 0);
    if (k == "layer.0.SelfAttention.o.weight") return cast16(&L.w_o, D, D, inner, 0, 0, 0);
    if (!t->gated && k == "layer.1.DenseReluDense.wi.weight") return cast16(&L.w_fi, dff, dff, D, 0, 0, 0);
    if (t->gated && k == "layer.1.DenseReluDense.wi_1.weight") return cast16(&L.w_fi, 2LL * dff, dff, D, 0, 32, 64);
    if (t->gated && k == "layer.1.DenseReluDense.wi_0.weight") return cast16(&L.w_fi, 2LL * dff, dff, D, 32, 32, 64);
    if (k == "layer.1.DenseReluDense.wo.weight") return cast16(&L.w_fo, D, D, dff, 0, 0, 0);
  }
  t->loaded.erase(name);
  set_last_error("unknown T5 weight key: " + name);
  return -4;
}

int satb_t5_set_buckets(SatbT5* t, const int* buckets, int n) {
  SATB_REQUIRE(t && buckets, "null argument");
  SATB_REQUIRE(n == kT5BiasSpan, "T5: the bucket table holds 1023 entries (relative positions -511 .. 511)");
  const int nb = t->cfg.relative_attention_num_buckets;
  for (int i = 0; i < n; ++i) SATB_REQUIRE(buckets[i] >= 0 && buckets[i] < nb, "T5: bucket outside [0, num_buckets)");
  if (!t->bucket) SATB_PROPAGATE(t->alloc(&t->bucket, kT5BiasSpan));
  SATB_CHECK_CUDA(cudaMemcpy(t->bucket, buckets, n * sizeof(int), cudaMemcpyHostToDevice));
  t->finalized = false;
  t->loaded["<buckets>"] = 1;
  return 0;
}

int satb_t5_set_proj_out(SatbT5* t, const float* W, const float* b, int out_dim, void* stream_v) {
  SATB_REQUIRE(t && W && b, "null argument");
  SATB_REQUIRE(out_dim >= 8 && out_dim % 8 == 0, "T5: proj_out's output width must be a positive multiple of 8");
  SATB_REQUIRE(t->out_dim == 0 || t->out_dim == out_dim, "T5: proj_out is already set with another width");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  if (!t->w_proj) SATB_PROPAGATE(t->alloc(&t->w_proj, static_cast<size_t>(out_dim) * t->D));
  if (!t->b_proj) SATB_PROPAGATE(t->alloc(&t->b_proj, out_dim));
  SATB_PROPAGATE(launch_cast_rows(W, t->w_proj, nullptr, out_dim, t->D, t->D, t->D, t->bf16, st));
  SATB_CHECK_CUDA(cudaMemcpyAsync(t->b_proj, b, out_dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
  t->out_dim = out_dim;
  t->cap = 0;   // the output workspace may need to grow
  return 0;
}

int satb_t5_finalize(SatbT5* t, void* stream_v) {
  SATB_REQUIRE(t, "null handle");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  std::string missing;
  auto need = [&](const std::string& k) {
    if (!t->loaded.count(k)) missing += (missing.empty() ? "" : ", ") + k;
  };
  if (!t->emb) missing = "shared.weight";   // or its alias encoder.embed_tokens.weight
  need("encoder.final_layer_norm.weight");
  need("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight");
  need("<buckets>");
  for (int i = 0; i < t->depth; ++i) {
    const std::string p = "encoder.block." + std::to_string(i) + ".";
    for (const char* k : {"layer.0.layer_norm.weight", "layer.1.layer_norm.weight", "layer.0.SelfAttention.q.weight",
                          "layer.0.SelfAttention.k.weight", "layer.0.SelfAttention.v.weight",
                          "layer.0.SelfAttention.o.weight", "layer.1.DenseReluDense.wo.weight"})
      need(p + k);
    if (t->gated) {
      need(p + "layer.1.DenseReluDense.wi_0.weight");
      need(p + "layer.1.DenseReluDense.wi_1.weight");
    } else {
      need(p + "layer.1.DenseReluDense.wi.weight");
    }
  }
  SATB_REQUIRE(missing.empty(), ("T5 finalize: missing weights: " + missing).c_str());
  if (!t->bias_tab) SATB_PROPAGATE(t->alloc(&t->bias_tab, static_cast<size_t>(t->H) * kT5BiasSpan));
  const int n = t->H * kT5BiasSpan;
  t5_bias_table_kernel<<<ceil_div(n, 256), 256, 0, st>>>(t->rel, t->bucket, t->cfg.relative_attention_num_buckets, t->H,
                                                       t->bias_tab);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  SATB_CHECK_CUDA(cudaStreamSynchronize(st));
  t->finalized = true;
  return 0;
}

int satb_t5_encode(SatbT5* t, const long long* ids, const int* lengths, int B, int L, float* out, void* stream_v) {
  SATB_REQUIRE(t && ids && lengths && out, "null argument");
  SATB_REQUIRE(t->finalized, "T5: call satb_t5_finalize after loading the weights");
  SATB_REQUIRE(B >= 1 && L >= 1 && L <= kT5MaxLen, "T5: need B >= 1 and 1 <= L <= 512");
  SATB_REQUIRE(static_cast<long long>(B) * L <= 0x7fffffffLL, "T5: B * L too large");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  int max_len = 0;
  SATB_PROPAGATE(t5_offsets(lengths, B, L, &t->off, &max_len));
  const int M = t->off[B];
  SATB_PROPAGATE(dev_int_upload(t->ws_off, t->off, st));
  if (M == 0) {   // every item empty: zeros
    SATB_CHECK_CUDA(launch_pdl(t5_scatter_kernel, dim3(B * L), dim3(kNormThreads), 0, st, static_cast<const float*>(nullptr),
                               static_cast<const int*>(t->ws_off.as<int>()), L, t->out_dim > 0 ? t->out_dim : t->D, out));
    count_launch();
    return 0;
  }
  SATB_PROPAGATE(t5_reserve(t, M));
  return t->bf16 ? t5_encode_impl<true>(t, ids, B, L, M, max_len, out, st)
                 : t5_encode_impl<false>(t, ids, B, L, M, max_len, out, st);
}

// ---- test entry points
int satb_t5_rmsnorm_probe(const float* x, const float* w, void* out, int rows, int D, float eps, int out_kind,
                          void* stream) {
  SATB_REQUIRE(x && w && out, "null argument");
  SATB_REQUIRE(rows >= 1, "T5 RMSNorm probe: need rows >= 1");
  return launch_t5_rmsnorm(x, w, out, rows, D, eps, out_kind, static_cast<cudaStream_t>(stream));
}

int satb_t5_attention_probe(const void* qkv16, const float* bias_tab, const int* lengths, int B, int H, int d_kv,
                            int bf16, void* o16, void* stream) {
  SATB_REQUIRE(qkv16 && bias_tab && lengths && o16, "null argument");
  SATB_REQUIRE(B >= 1 && H >= 1, "T5 attention probe: need B, H >= 1");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(qkv16) & 15) == 0 && (reinterpret_cast<uintptr_t>(o16) & 15) == 0,
               "T5 attention probe: qkv and o must be 16-byte aligned");
  std::vector<int> off;
  int max_len = 0;
  SATB_PROPAGATE(t5_offsets(lengths, B, kT5MaxLen, &off, &max_len));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DevBuf d_off;
  int rc = dev_int_upload(d_off, off, st);
  if (rc == 0) rc = launch_t5_attention(qkv16, bias_tab, d_off.as<int>(), B, max_len, H, d_kv, bf16 != 0, o16, st);
  const cudaError_t e = cudaStreamSynchronize(st);
  d_off.release();
  SATB_PROPAGATE(rc);
  SATB_CHECK_CUDA(e);
  return 0;
}

int satb_t5_gemm_probe(const void* a16, const void* w16, int M, int N, int K, const SatbGemmProbe* p, void* stream) {
  SATB_REQUIRE(a16 && w16 && p && p->out, "null argument");
  SATB_REQUIRE(M >= 1 && K >= 8 && K % 8 == 0, "T5 gemm probe: need M >= 1 and K % 8 == 0");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(a16) & 15) == 0 && (reinterpret_cast<uintptr_t>(w16) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(p->out) & 15) == 0,
               "T5 gemm probe: operands and out must be 16-byte aligned");
  SATB_REQUIRE(p->bn == 128 || p->bn == 256, "T5 gemm probe: bn must be 128 or 256");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  TmapCache tc;
  if (p->epi == SATB_EPI_RELU16) {
    SATB_REQUIRE(N >= 32 && N % 32 == 0 && p->ld >= N && p->ld % 8 == 0, "T5 gemm probe relu16: N % 32 == 0, ld >= N");
    if (p->bf16) return t5_linear<EpiRelu16<true>, true>(tc, a16, M, M, K, w16, N, {p->out, p->ld}, st, p->bn);
    return t5_linear<EpiRelu16<false>, false>(tc, a16, M, M, K, w16, N, {p->out, p->ld}, st, p->bn);
  }
  if (p->epi == SATB_EPI_GEGLU16) {
    SATB_REQUIRE(N >= 64 && N % 64 == 0 && p->ld >= N / 2 && p->ld % 8 == 0,
                 "T5 gemm probe geglu16: N % 64 == 0, ld >= N / 2");
    if (p->bf16) return t5_linear<EpiGeglu16<true>, true>(tc, a16, M, M, K, w16, N, {p->out, p->ld}, st, p->bn);
    return t5_linear<EpiGeglu16<false>, false>(tc, a16, M, M, K, w16, N, {p->out, p->ld}, st, p->bn);
  }
  set_last_error("T5 gemm probe: no such instance (epi " + std::to_string(p->epi) +
                 "); the T5 encoder's own epilogues are relu16 (10) and geglu16 (11), BN 128 / 256");
  return -1;
}

}  // extern "C"

// Every GEMM of an encode through t5_linear, with the parameters t5_encode_impl passes.
template <bool BF16>
static int t5_linear_probe(const void* a16, int a_rows, const void* w16, int M, int N, int K, const SatbGemmProbe& p,
                           cudaStream_t st) {
  TmapCache tc;
  const int bn = p.bn;
  auto out_ok = [&](int cols, int elem) {
    return p.out && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0 && p.ld >= cols && (p.ld * elem) % 16 == 0;
  };
  switch (p.epi) {
    case SATB_EPI_STORE16:   // QKV
      SATB_REQUIRE(N % 32 == 0 && out_ok(N, 2), "T5 linear probe store16: N % 32 == 0, out 16-byte aligned, ld >= N");
      return t5_linear<EpiStore16<BF16>, BF16>(tc, a16, a_rows, M, K, w16, N,
                                              typename EpiStore16<BF16>::Params{p.out, p.ld, nullptr, 0}, st, bn);
    case SATB_EPI_RESIDUAL:  // o-projection, FF-out
      SATB_REQUIRE(N % 8 == 0 && p.h && (reinterpret_cast<uintptr_t>(p.h) & 15) == 0 && p.ld >= N && p.ld % 4 == 0,
                   "T5 linear probe residual: N % 8 == 0, h 16-byte aligned, ld >= N, ld % 4 == 0");
      return t5_linear<EpiResidual, BF16>(tc, a16, a_rows, M, K, w16, N,
                                          EpiResidual::Params{p.h, p.ld, nullptr, nullptr, 1, 0, 1}, st, bn);
    case SATB_EPI_STORE32:   // proj_out
      SATB_REQUIRE(N % 8 == 0 && out_ok(N, 4) && p.bias && (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0,
                   "T5 linear probe store32: N % 8 == 0, out and bias 16-byte aligned, ld >= N");
      return t5_linear<EpiStore32, BF16>(tc, a16, a_rows, M, K, w16, N,
                                         EpiStore32::Params{static_cast<float*>(p.out), p.ld, p.bias}, st, bn);
    case SATB_EPI_RELU16:    // FF-in, relu
      SATB_REQUIRE(N % 32 == 0 && out_ok(N, 2), "T5 linear probe relu16: N % 32 == 0, out 16-byte aligned, ld >= N");
      return t5_linear<EpiRelu16<BF16>, BF16>(tc, a16, a_rows, M, K, w16, N,
                                             typename EpiRelu16<BF16>::Params{p.out, p.ld}, st, bn);
    case SATB_EPI_GEGLU16:   // FF-in, gated-gelu
      SATB_REQUIRE(N % 64 == 0 && out_ok(N / 2, 2),
                   "T5 linear probe geglu16: N % 64 == 0, out 16-byte aligned, ld >= N / 2");
      return t5_linear<EpiGeglu16<BF16>, BF16>(tc, a16, a_rows, M, K, w16, N,
                                              typename EpiGeglu16<BF16>::Params{p.out, p.ld}, st, bn);
    default:
      break;
  }
  set_last_error("T5 linear probe: no such instance (epi " + std::to_string(p.epi) +
                 "); an encode runs store16 (1), residual (5), store32 (0), relu16 (10) and geglu16 (11)");
  return -1;
}

extern "C" {

int satb_t5_linear_probe(const void* a16, int a_rows, const void* w16, int M, int N, int K, const SatbGemmProbe* p,
                         void* stream) {
  SATB_REQUIRE(a16 && w16 && p, "null argument");
  SATB_REQUIRE(M >= 1 && a_rows >= M && N >= 8 && K >= 8 && K % 8 == 0,
               "T5 linear probe: need 1 <= M <= a_rows, N >= 8 and K % 8 == 0");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(a16) & 15) == 0 && (reinterpret_cast<uintptr_t>(w16) & 15) == 0,
               "T5 linear probe: operands must be 16-byte aligned");
  SATB_REQUIRE(p->bn == 0 || p->bn == 128 || p->bn == 256, "T5 linear probe: bn must be 0 (auto_bn), 128 or 256");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return p->bf16 ? t5_linear_probe<true>(a16, a_rows, w16, M, N, K, *p, st)
                 : t5_linear_probe<false>(a16, a_rows, w16, M, N, K, *p, st);
}

int satb_t5_bias_table(SatbT5* t, float* dst, void* stream) {
  SATB_REQUIRE(t && dst, "null argument");
  SATB_REQUIRE(t->finalized, "T5: call satb_t5_finalize first (it builds the bias table)");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  SATB_CHECK_CUDA(cudaMemcpyAsync(dst, t->bias_tab, static_cast<size_t>(t->H) * kT5BiasSpan * sizeof(float),
                                  cudaMemcpyDeviceToDevice, st));
  SATB_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
