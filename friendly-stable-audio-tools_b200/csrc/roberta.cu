// RoBERTa encoder: Hugging Face RobertaModel (transformers models/roberta/modeling_roberta.py), the text branch of
// laion_clap's CLAP_Module (tmodel "roberta") that the reference's CLAPTextConditioner reads hidden states from
// (reference models/conditioners.py CLAPTextConditioner.get_clap_features), on this library's kernels.
//
// Rows are not packed: the conditioner returns the features of every one of the L positions, padded ones included
// (it does not multiply them by the mask), so all B L rows are computed.  Keys are limited to each item's valid
// prefix, which is what HF's additive key mask does for right-padded masks.
//
// Residual stream fp32 [B L, d]; GEMM operands 16-bit (fp16 or bf16), fp32 accumulation.  One encode of n layers:
//   embeddings: word + token_type[0] + position, LayerNorm -> fp32 stream and 16-bit rows   rb_embed_ln_kernel
//   per layer:  QKV [M, 3 d] + bias                     GEMM, EpiStore16 (q | k | v rows of one fused weight)
//               attention core [M, d]                   rb_attn_kernel (scale 1/8, keys of the valid prefix)
//               h += out-proj + bias                    GEMM, EpiResidual
//               LayerNorm (post-LN: the normalised value is the new stream) -> fp32 and 16-bit   rb_layernorm_kernel
//               FF-in [M, d_ff] = gelu(x W + b)         GEMM, EpiBiasGelu16 (erf GELU)
//               h += FF-out + bias                      GEMM, EpiResidual
//               LayerNorm -> fp32 and 16-bit            rb_layernorm_kernel
//   optional proj_out [M, out] = x W + b                GEMM, EpiStore32
// The last LayerNorm (or the embedding kernel when n = 0) writes its fp32 rows straight to the output when there is no
// proj_out.  1 + 7 n launches without proj_out, 2 + 7 n with it (78 for Stable Audio 2.0's 11 layers, whose proj_out is
// an identity), all with programmatic dependent launch.  n is the number of layers whose output the caller wants: hidden_states[n]
// of RobertaModel(output_hidden_states=True), index 0 being the embedding output.
//
// Position ids follow RobertaEmbeddings.create_position_ids_from_input_ids: pos = cumsum(id != pad) * (id != pad) +
// pad over the item's ids (not its mask), counted in integers inside the embedding kernel.
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

constexpr int kRbMaxLen = 512;     // longest prompt an encode accepts
constexpr int kRbMaxDim = 1024;    // hidden size (roberta-large)
constexpr int kRbHeadDim = 64;
constexpr int kRbThreads = 128;
constexpr int kRbVec = kRbMaxDim / 4 / kRbThreads;   // float4 per thread at the widest row

template <class T>
__device__ __forceinline__ T rb_block_sum(T v, T* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();   // red may still be read by an earlier call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T tot = 0;
#pragma unroll
  for (int i = 0; i < kRbThreads / 32; ++i) tot += red[i];
  return tot;
}

// nn.LayerNorm of one row held in registers (v: float4 c = threadIdx.x + i kRbThreads of the row, zeros past D):
// y = (x - mean) rsqrt(var + eps) g + b with fp32 statistics, the variance from the centred values.  Writes the fp32
// row to y32 and its 16-bit copy (fp16 saturating at +-65504, or bf16) to y16.
template <bool BF16>
__device__ __forceinline__ void rb_ln_store(float4 (&v)[kRbVec], const float* g, const float* b, int D, float eps,
                                            float* y32, uint16_t* y16, float* red) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kRbVec; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = rb_block_sum(s, red) / static_cast<float>(D);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kRbVec; ++i) {
    const int c = threadIdx.x + i * kRbThreads;
    if (c < D / 4) {
      const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
      ss = fmaf(dx, dx, ss);
      ss = fmaf(dy, dy, ss);
      ss = fmaf(dz, dz, ss);
      ss = fmaf(dw, dw, ss);
    }
  }
  const float r = rsqrtf(rb_block_sum(ss, red) / static_cast<float>(D) + eps);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(b);
#pragma unroll
  for (int i = 0; i < kRbVec; ++i) {
    const int c = threadIdx.x + i * kRbThreads;
    if (c >= D / 4) break;
    const float4 gg = __ldg(g4 + c), bb = __ldg(b4 + c);
    const float4 y = make_float4(fmaf((v[i].x - mean) * r, gg.x, bb.x), fmaf((v[i].y - mean) * r, gg.y, bb.y),
                                 fmaf((v[i].z - mean) * r, gg.z, bb.z), fmaf((v[i].w - mean) * r, gg.w, bb.w));
    reinterpret_cast<float4*>(y32)[c] = y;
    reinterpret_cast<uint2*>(y16)[c] = make_uint2(pack16_satfinite<BF16>(y.x, y.y), pack16_satfinite<BF16>(y.z, y.w));
  }
}

struct RbEmbedArgs {
  const long long* ids;   // [B, L]
  int L;
  const float* word;      // [vocab, D]
  int vocab;
  const float* pos;       // [max_pos, D]
  int max_pos;
  const float* tok;       // token_type_embeddings row 0 [D]
  const float* g;
  const float* b;
  int D;
  int pad;
  float eps;
  float* y32;             // [B L, D]
  uint16_t* y16;
};

// Row m = b L + t: RobertaEmbeddings.forward (modeling_roberta.py: inputs_embeds + token_type_embeddings, then +
// position_embeddings, then LayerNorm).  Ids and positions are clamped to their tables: the host refuses ids outside
// [0, vocab) and prompts whose positions would pass max_pos, and no input makes this kernel read outside a table.
template <bool BF16>
__global__ void __launch_bounds__(kRbThreads) rb_embed_ln_kernel(const RbEmbedArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float redf[kRbThreads / 32];
  __shared__ int redi[kRbThreads / 32];
  const int m = blockIdx.x;
  const int t = m % a.L;
  const long long* idr = a.ids + static_cast<size_t>(m - t);
  int cnt = 0;
  for (int j = threadIdx.x; j <= t; j += kRbThreads) cnt += idr[j] != a.pad;
  cnt = rb_block_sum(cnt, redi);
  long long id = idr[t];
  int p = id != a.pad ? cnt + a.pad : a.pad;
  p = p < 0 ? 0 : (p >= a.max_pos ? a.max_pos - 1 : p);
  id = id < 0 ? 0 : (id >= a.vocab ? a.vocab - 1 : id);
  const float4* w4 = reinterpret_cast<const float4*>(a.word + static_cast<size_t>(id) * a.D);
  const float4* p4 = reinterpret_cast<const float4*>(a.pos + static_cast<size_t>(p) * a.D);
  const float4* t4 = reinterpret_cast<const float4*>(a.tok);
  float4 v[kRbVec];
#pragma unroll
  for (int i = 0; i < kRbVec; ++i) {
    const int c = threadIdx.x + i * kRbThreads;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < a.D / 4) {
      const float4 w = __ldg(w4 + c), pp = __ldg(p4 + c), tt = __ldg(t4 + c);
      v[i] = make_float4((w.x + tt.x) + pp.x, (w.y + tt.y) + pp.y, (w.z + tt.z) + pp.z, (w.w + tt.w) + pp.w);
    }
  }
  rb_ln_store<BF16>(v, a.g, a.b, a.D, a.eps, a.y32 + static_cast<size_t>(m) * a.D, a.y16 + static_cast<size_t>(m) * a.D,
                    redf);
}

// Post-LN of a RobertaSelfOutput / RobertaOutput: y = LayerNorm(x), where x already holds hidden + dense + bias (the
// residual GEMM added them into the stream).  y32 may alias x.
template <bool BF16>
__global__ void __launch_bounds__(kRbThreads) rb_layernorm_kernel(const float* x, const float* g, const float* b, int D,
                                                                   float eps, float* y32, uint16_t* y16) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[kRbThreads / 32];
  const int row = blockIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
  float4 v[kRbVec];
#pragma unroll
  for (int i = 0; i < kRbVec; ++i) {
    const int c = threadIdx.x + i * kRbThreads;
    v[i] = c < D / 4 ? xr[c] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  rb_ln_store<BF16>(v, g, b, D, eps, y32 + static_cast<size_t>(row) * D, y16 + static_cast<size_t>(row) * D, red);
}

// ---- attention core: O = softmax(Q K^T / 8 + key mask) V per (item, head), RobertaSelfAttention at head dim 64.
// One CTA of four warps per (64-query tile, head, item) runs mma_tile.cuh's mma.sync core (mma_attention), scale 1/8
// in log2 units.  Every one of the item's L query rows is computed and stored; only keys [0, len) take part.  len >= 1
// (the host refuses empty prompts), so every row has a key.
// qkv [B L, 3 H 64]: q of head h at column 64 h, k at 64 (H + h), v at 64 (2 H + h); o [B L, H 64]; lens [B]
template <bool BF16>
__global__ void __launch_bounds__(kMmaAttnThreads) rb_attn_kernel(const uint16_t* qkv, uint16_t* o, const int* lens,
                                                                   int L, int H) {
  constexpr int D = kRbHeadDim;
  extern __shared__ __align__(128) uint16_t smem_rb[];
  pdl_launch_dependents();
  pdl_wait();   // qkv is written by the previous kernel
  const int h = blockIdx.y, b = blockIdx.z;
  const int n = lens[b];
  const int inner = H * D;
  const int64_t ld = 3LL * inner;
  const uint16_t* base = qkv + static_cast<int64_t>(b) * L * ld;
  mma_attention<D, BF16>(smem_rb, base, ld, h * D, base, ld, inner + h * D, base, ld, 2 * inner + h * D,
                         o + static_cast<int64_t>(b) * L * inner, inner, h * D, blockIdx.x * 64, L, n,
                         ScaleScore{0.125f * 1.4426950408889634f});
}

}  // namespace

// ---- launchers (also the probes' path)
static int launch_rb_embed(const RbEmbedArgs& a, int rows, bool bf16, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (bf16) SATB_CHECK_CUDA(launch_pdl(rb_embed_ln_kernel<true>, dim3(rows), dim3(kRbThreads), 0, st, a));
  else SATB_CHECK_CUDA(launch_pdl(rb_embed_ln_kernel<false>, dim3(rows), dim3(kRbThreads), 0, st, a));
  count_launch();
  return 0;
}

static int launch_rb_layernorm(const float* x, const float* g, const float* b, int rows, int D, float eps, float* y32,
                               void* y16, bool bf16, cudaStream_t st) {
  if (rows <= 0) return 0;
  uint16_t* o16 = static_cast<uint16_t*>(y16);
  if (bf16)
    SATB_CHECK_CUDA(launch_pdl(rb_layernorm_kernel<true>, dim3(rows), dim3(kRbThreads), 0, st, x, g, b, D, eps, y32, o16));
  else
    SATB_CHECK_CUDA(launch_pdl(rb_layernorm_kernel<false>, dim3(rows), dim3(kRbThreads), 0, st, x, g, b, D, eps, y32, o16));
  count_launch();
  return 0;
}

// qkv [B L, 3 H 64], o [B L, H 64]; lens_dev [B], each in [1, L]
static int launch_rb_attention(const void* qkv, const int* lens_dev, int B, int L, int H, bool bf16, void* o,
                               cudaStream_t st) {
  if (B <= 0 || L <= 0) return 0;
  const dim3 grid(ceil_div(L, 64), H, B);
  SATB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "RoBERTa attention grid too large");
  const uint16_t* q = static_cast<const uint16_t*>(qkv);
  uint16_t* out = static_cast<uint16_t*>(o);
  SATB_PROPAGATE((bf16 ? launch_mma_attention<rb_attn_kernel<true>, kRbHeadDim>(grid, st, q, out, lens_dev, L, H)
                       : launch_mma_attention<rb_attn_kernel<false>, kRbHeadDim>(grid, st, q, out, lens_dev, L, H)));
  count_launch();
  return 0;
}

static int rb_dims_ok(int D) {
  SATB_REQUIRE(D >= 128 && D % 128 == 0 && D <= kRbMaxDim, "RoBERTa: hidden_size must be a multiple of 128, at most 1024");
  return 0;
}

struct RbLayer {
  uint16_t *w_qkv = nullptr, *w_o = nullptr, *w_fi = nullptr, *w_fo = nullptr;
  float *b_qkv = nullptr, *b_o = nullptr, *b_fi = nullptr, *b_fo = nullptr;
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
};

}  // namespace satb

using namespace satb;

struct SatbRoberta {
  SatbRobertaConfig cfg;
  int D, H, F, depth;
  bool bf16;
  float *word = nullptr, *pos = nullptr, *tok = nullptr, *emb_g = nullptr, *emb_b = nullptr;
  std::vector<RbLayer> layers;
  uint16_t* w_proj = nullptr;
  float* b_proj = nullptr;
  int out_dim = 0;            // 0: no proj_out
  std::map<std::string, int> loaded;
  bool finalized = false;
  std::vector<void*> owned;
  TmapCache tmaps;
  DevBuf ws_h, ws_a16, ws_qkv, ws_attn, ws_ff, ws_len;
  int cap = 0;                // rows the workspaces hold

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

static int rb_reserve(SatbRoberta* t, int rows) {
  if (rows <= t->cap) return 0;
  const int cap = std::max(rows, 2 * t->cap);
  const size_t r = static_cast<size_t>(cap);
  SATB_PROPAGATE(t->ws_h.ensure(r * t->D * 4));
  SATB_PROPAGATE(t->ws_a16.ensure(r * t->D * 2));
  SATB_PROPAGATE(t->ws_qkv.ensure(r * 3 * t->D * 2));
  SATB_PROPAGATE(t->ws_attn.ensure(r * t->D * 2));
  SATB_PROPAGATE(t->ws_ff.ensure(r * t->F * 2));
  t->tmaps.maps.clear();   // the maps span the old buffers
  t->cap = cap;
  return 0;
}

// The encoder's GEMM: C[M, N] = A[M, K] W[N, K]^T through Epi, with linear.cuh's N-tile choice.
template <class Epi, bool BF16>
static int rb_linear(TmapCache& tc, const void* A, int M, int K, const void* W, int N, const typename Epi::Params& ep,
                     cudaStream_t st) {
  if (M <= 0) return 0;
  return linear_auto<Epi, BF16>(tc, A, K, M, K, W, N, ep, st);
}

template <bool BF16>
static int rb_encode_impl(SatbRoberta* t, const long long* ids, int B, int L, float* out, cudaStream_t st) {
  const int D = t->D, F = t->F, M = B * L;
  const int* lens = t->ws_len.as<int>();
  float* h = t->ws_h.as<float>();
  uint16_t* a16 = t->ws_a16.as<uint16_t>();
  uint16_t* qkv = t->ws_qkv.as<uint16_t>();
  uint16_t* att = t->ws_attn.as<uint16_t>();
  uint16_t* ff = t->ws_ff.as<uint16_t>();
  const float eps = t->cfg.layer_norm_eps;
  // the fp32 rows of the last stage go straight to the output when nothing follows them
  auto dst32 = [&](bool last) { return last && t->out_dim == 0 ? out : h; };
  RbEmbedArgs e;
  e.ids = ids; e.L = L; e.word = t->word; e.vocab = t->cfg.vocab_size; e.pos = t->pos;
  e.max_pos = t->cfg.max_position_embeddings; e.tok = t->tok; e.g = t->emb_g; e.b = t->emb_b; e.D = D;
  e.pad = t->cfg.pad_token_id; e.eps = eps; e.y32 = dst32(t->depth == 0); e.y16 = a16;
  SATB_PROPAGATE(launch_rb_embed(e, M, BF16, st));
  for (int li = 0; li < t->depth; ++li) {
    const RbLayer& W = t->layers[li];
    const bool last = li + 1 == t->depth;
    SATB_PROPAGATE((rb_linear<EpiStore16<BF16>, BF16>(t->tmaps, a16, M, D, W.w_qkv, 3 * D,
                                                      typename EpiStore16<BF16>::Params{qkv, 3 * D, W.b_qkv, 0}, st)));
    SATB_PROPAGATE(launch_rb_attention(qkv, lens, B, L, t->H, BF16, att, st));
    SATB_PROPAGATE((rb_linear<EpiResidual, BF16>(t->tmaps, att, M, D, W.w_o, D,
                                                 EpiResidual::Params{h, D, W.b_o, nullptr, 1, 0, 1}, st)));
    SATB_PROPAGATE(launch_rb_layernorm(h, W.ln1_g, W.ln1_b, M, D, eps, h, a16, BF16, st));
    SATB_PROPAGATE((rb_linear<EpiBiasGelu16<BF16>, BF16>(t->tmaps, a16, M, D, W.w_fi, F,
                                                         typename EpiBiasGelu16<BF16>::Params{ff, F, W.b_fi}, st)));
    SATB_PROPAGATE((rb_linear<EpiResidual, BF16>(t->tmaps, ff, M, F, W.w_fo, D,
                                                 EpiResidual::Params{h, D, W.b_fo, nullptr, 1, 0, 1}, st)));
    SATB_PROPAGATE(launch_rb_layernorm(h, W.ln2_g, W.ln2_b, M, D, eps, dst32(last), a16, BF16, st));
  }
  if (t->out_dim > 0)
    SATB_PROPAGATE((rb_linear<EpiStore32, BF16>(t->tmaps, a16, M, D, t->w_proj, t->out_dim,
                                                EpiStore32::Params{out, t->out_dim, t->b_proj}, st)));
  return 0;
}

static int rb_lengths(const int* lengths, int B, int L, std::vector<int>* v) {
  v->assign(lengths, lengths + B);
  for (int b = 0; b < B; ++b)
    SATB_REQUIRE(lengths[b] >= 1 && lengths[b] <= L, "RoBERTa: every length must lie in [1, L]");
  return 0;
}

extern "C" {

int satb_roberta_create(const SatbRobertaConfig* cfg, SatbRoberta** out) {
  SATB_REQUIRE(cfg && out, "null argument");
  const SatbRobertaConfig& c = *cfg;
  SATB_PROPAGATE(rb_dims_ok(c.hidden_size));
  SATB_REQUIRE(c.num_heads >= 1 && c.num_heads * kRbHeadDim == c.hidden_size,
               "RoBERTa: the attention head dim (hidden_size / num_heads) must be 64");
  SATB_REQUIRE(c.intermediate_size >= 32 && c.intermediate_size % 32 == 0,
               "RoBERTa: intermediate_size must be a positive multiple of 32");
  SATB_REQUIRE(c.num_layers >= 0, "RoBERTa: num_layers (the layers an encode runs) must be >= 0");
  SATB_REQUIRE(c.vocab_size >= 1 && c.type_vocab_size >= 1, "RoBERTa: need vocab_size >= 1 and type_vocab_size >= 1");
  SATB_REQUIRE(c.pad_token_id >= 0 && c.max_position_embeddings > c.pad_token_id + 1,
               "RoBERTa: need 0 <= pad_token_id < max_position_embeddings - 1");
  SATB_REQUIRE(c.layer_norm_eps >= 0.f, "RoBERTa: layer_norm_eps must not be negative");
  SATB_REQUIRE(c.operand_dtype == 0 || c.operand_dtype == 1, "RoBERTa: operand_dtype must be 0 (fp16) or 1 (bf16)");
  SatbRoberta* t = new SatbRoberta();
  t->cfg = c;
  t->D = c.hidden_size;
  t->H = c.num_heads;
  t->F = c.intermediate_size;
  t->depth = c.num_layers;
  t->bf16 = c.operand_dtype == 1;
  t->layers.resize(c.num_layers);
  *out = t;
  return 0;
}

void satb_roberta_destroy(SatbRoberta* t) {
  if (!t) return;
  cudaDeviceSynchronize();
  for (void* p : t->owned) cudaFree(p);
  for (DevBuf* b : {&t->ws_h, &t->ws_a16, &t->ws_qkv, &t->ws_attn, &t->ws_ff, &t->ws_len}) b->release();
  delete t;
}

// One RobertaModel state-dict entry by its HF key; src: device fp32, contiguous.  Matrices are cast to the 16-bit
// operand type; query / key / value weights and biases go to the row ranges of the fused QKV weight and bias.
int satb_roberta_load_weight(SatbRoberta* t, const char* name_c, const float* src, long long numel, void* stream_v) {
  SATB_REQUIRE(t && name_c && src, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  const std::string name(name_c);
  const int D = t->D, F = t->F;
  // src into the fp32 vector *dst (total elements) at element off0
  auto copy_f32 = [&](float** dst, long long total, long long expect, long long off0) -> int {
    SATB_REQUIRE(numel == expect, ("bad size for " + name).c_str());
    if (!*dst) SATB_PROPAGATE(t->alloc(dst, total));
    SATB_CHECK_CUDA(cudaMemcpyAsync(*dst + off0, src, expect * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
  };
  auto cast16 = [&](uint16_t** dst, long long total_rows, int rows, int cols, long long row0) -> int {
    SATB_REQUIRE(numel == static_cast<long long>(rows) * cols, ("bad size for " + name).c_str());
    if (!*dst) SATB_PROPAGATE(t->alloc(dst, static_cast<size_t>(total_rows) * cols));
    return launch_cast_rows(src, *dst + static_cast<size_t>(row0) * cols, nullptr, rows, cols, cols, cols, t->bf16, st);
  };
  t->finalized = false;
  t->loaded[name] = 1;
  const long long d = D;
  if (name == "embeddings.word_embeddings.weight") return copy_f32(&t->word, t->cfg.vocab_size * d, t->cfg.vocab_size * d, 0);
  if (name == "embeddings.position_embeddings.weight")
    return copy_f32(&t->pos, t->cfg.max_position_embeddings * d, t->cfg.max_position_embeddings * d, 0);
  if (name == "embeddings.token_type_embeddings.weight")
    return copy_f32(&t->tok, t->cfg.type_vocab_size * d, t->cfg.type_vocab_size * d, 0);
  if (name == "embeddings.LayerNorm.weight") return copy_f32(&t->emb_g, d, d, 0);
  if (name == "embeddings.LayerNorm.bias") return copy_f32(&t->emb_b, d, d, 0);
  const std::string lp = "encoder.layer.";
  if (name.compare(0, lp.size(), lp) == 0) {
    const size_t dot = name.find('.', lp.size());
    SATB_REQUIRE(dot != std::string::npos, ("bad key " + name).c_str());
    const int li = atoi(name.substr(lp.size(), dot - lp.size()).c_str());
    SATB_REQUIRE(li >= 0 && li < t->depth, ("layer index out of range in " + name).c_str());
    RbLayer& L = t->layers[li];
    const std::string k = name.substr(dot + 1);
    const char* qkv_names[3] = {"attention.self.query.", "attention.self.key.", "attention.self.value."};
    for (int j = 0; j < 3; ++j) {
      if (k == std::string(qkv_names[j]) + "weight") return cast16(&L.w_qkv, 3 * d, D, D, j * d);
      if (k == std::string(qkv_names[j]) + "bias") return copy_f32(&L.b_qkv, 3 * d, d, j * d);
    }
    if (k == "attention.output.dense.weight") return cast16(&L.w_o, D, D, D, 0);
    if (k == "attention.output.dense.bias") return copy_f32(&L.b_o, d, d, 0);
    if (k == "attention.output.LayerNorm.weight") return copy_f32(&L.ln1_g, d, d, 0);
    if (k == "attention.output.LayerNorm.bias") return copy_f32(&L.ln1_b, d, d, 0);
    if (k == "intermediate.dense.weight") return cast16(&L.w_fi, F, F, D, 0);
    if (k == "intermediate.dense.bias") return copy_f32(&L.b_fi, F, F, 0);
    if (k == "output.dense.weight") return cast16(&L.w_fo, D, D, F, 0);
    if (k == "output.dense.bias") return copy_f32(&L.b_fo, d, d, 0);
    if (k == "output.LayerNorm.weight") return copy_f32(&L.ln2_g, d, d, 0);
    if (k == "output.LayerNorm.bias") return copy_f32(&L.ln2_b, d, d, 0);
  }
  t->loaded.erase(name);
  set_last_error("unknown RoBERTa weight key: " + name);
  return -4;
}

int satb_roberta_set_proj_out(SatbRoberta* t, const float* W, const float* b, int out_dim, void* stream_v) {
  SATB_REQUIRE(t && W && b, "null argument");
  SATB_REQUIRE(out_dim >= 8 && out_dim % 8 == 0, "RoBERTa: proj_out's output width must be a positive multiple of 8");
  SATB_REQUIRE(t->out_dim == 0 || t->out_dim == out_dim, "RoBERTa: proj_out is already set with another width");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  if (!t->w_proj) SATB_PROPAGATE(t->alloc(&t->w_proj, static_cast<size_t>(out_dim) * t->D));
  if (!t->b_proj) SATB_PROPAGATE(t->alloc(&t->b_proj, out_dim));
  SATB_PROPAGATE(launch_cast_rows(W, t->w_proj, nullptr, out_dim, t->D, t->D, t->D, t->bf16, st));
  SATB_CHECK_CUDA(cudaMemcpyAsync(t->b_proj, b, out_dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
  t->out_dim = out_dim;
  return 0;
}

int satb_roberta_finalize(SatbRoberta* t, void* stream_v) {
  SATB_REQUIRE(t, "null handle");
  std::string missing;
  auto need = [&](const std::string& k) {
    if (!t->loaded.count(k)) missing += (missing.empty() ? "" : ", ") + k;
  };
  for (const char* k : {"embeddings.word_embeddings.weight", "embeddings.position_embeddings.weight",
                        "embeddings.token_type_embeddings.weight", "embeddings.LayerNorm.weight",
                        "embeddings.LayerNorm.bias"})
    need(k);
  for (int i = 0; i < t->depth; ++i) {
    const std::string p = "encoder.layer." + std::to_string(i) + ".";
    for (const char* k : {"attention.self.query.weight", "attention.self.query.bias", "attention.self.key.weight",
                          "attention.self.key.bias", "attention.self.value.weight", "attention.self.value.bias",
                          "attention.output.dense.weight", "attention.output.dense.bias",
                          "attention.output.LayerNorm.weight", "attention.output.LayerNorm.bias",
                          "intermediate.dense.weight", "intermediate.dense.bias", "output.dense.weight",
                          "output.dense.bias", "output.LayerNorm.weight", "output.LayerNorm.bias"})
      need(p + k);
  }
  SATB_REQUIRE(missing.empty(), ("RoBERTa finalize: missing weights: " + missing).c_str());
  SATB_CHECK_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream_v)));
  t->finalized = true;
  return 0;
}

int satb_roberta_encode(SatbRoberta* t, const long long* ids, const int* lengths, int B, int L, float* out,
                        void* stream_v) {
  SATB_REQUIRE(t && ids && lengths && out, "null argument");
  SATB_REQUIRE(t->finalized, "RoBERTa: call satb_roberta_finalize after loading the weights");
  SATB_REQUIRE(B >= 1 && L >= 1 && L <= kRbMaxLen, "RoBERTa: need B >= 1 and 1 <= L <= 512");
  SATB_REQUIRE(L + t->cfg.pad_token_id < t->cfg.max_position_embeddings,
               "RoBERTa: L + pad_token_id must be below max_position_embeddings (the largest position id)");
  SATB_REQUIRE(static_cast<long long>(B) * L <= 0x7fffffffLL / 4, "RoBERTa: B * L too large");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  std::vector<int> lens;
  SATB_PROPAGATE(rb_lengths(lengths, B, L, &lens));
  SATB_PROPAGATE(dev_int_upload(t->ws_len, lens, st));
  SATB_PROPAGATE(rb_reserve(t, B * L));
  return t->bf16 ? rb_encode_impl<true>(t, ids, B, L, out, st) : rb_encode_impl<false>(t, ids, B, L, out, st);
}

// ---- test entry points
int satb_roberta_embed_probe(const long long* ids, int B, int L, const float* word, int vocab, const float* pos,
                             int max_pos, const float* tok, const float* gamma, const float* beta, int D, int pad,
                             float eps, float* y32, void* y16, int bf16, void* stream) {
  SATB_REQUIRE(ids && word && pos && tok && gamma && beta && y32 && y16, "null argument");
  SATB_PROPAGATE(rb_dims_ok(D));
  SATB_REQUIRE(B >= 1 && L >= 1 && L <= kRbMaxLen && vocab >= 1 && pad >= 0 && max_pos > L + pad,
               "RoBERTa embed probe: need B >= 1, 1 <= L <= 512, vocab >= 1 and max_pos > L + pad");
  RbEmbedArgs a;
  a.ids = ids; a.L = L; a.word = word; a.vocab = vocab; a.pos = pos; a.max_pos = max_pos; a.tok = tok; a.g = gamma;
  a.b = beta; a.D = D; a.pad = pad; a.eps = eps; a.y32 = y32; a.y16 = static_cast<uint16_t*>(y16);
  return launch_rb_embed(a, B * L, bf16 != 0, static_cast<cudaStream_t>(stream));
}

int satb_roberta_layernorm_probe(const float* x, const float* gamma, const float* beta, int rows, int D, float eps,
                                 float* y32, void* y16, int bf16, void* stream) {
  SATB_REQUIRE(x && gamma && beta && y32 && y16, "null argument");
  SATB_PROPAGATE(rb_dims_ok(D));
  SATB_REQUIRE(rows >= 1, "RoBERTa LayerNorm probe: need rows >= 1");
  return launch_rb_layernorm(x, gamma, beta, rows, D, eps, y32, y16, bf16 != 0, static_cast<cudaStream_t>(stream));
}

int satb_roberta_attention_probe(const void* qkv16, const int* lengths, int B, int L, int H, int bf16, void* o16,
                                 void* stream) {
  SATB_REQUIRE(qkv16 && lengths && o16, "null argument");
  SATB_REQUIRE(B >= 1 && H >= 1 && L >= 1 && L <= kRbMaxLen, "RoBERTa attention probe: need B, H >= 1, 1 <= L <= 512");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(qkv16) & 15) == 0 && (reinterpret_cast<uintptr_t>(o16) & 15) == 0,
               "RoBERTa attention probe: qkv and o must be 16-byte aligned");
  std::vector<int> lens;
  SATB_PROPAGATE(rb_lengths(lengths, B, L, &lens));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DevBuf d_len;
  int rc = dev_int_upload(d_len, lens, st);
  if (rc == 0) rc = launch_rb_attention(qkv16, d_len.as<int>(), B, L, H, bf16 != 0, o16, st);
  const cudaError_t e = cudaStreamSynchronize(st);
  d_len.release();
  SATB_PROPAGATE(rc);
  SATB_CHECK_CUDA(e);
  return 0;
}

}  // extern "C"

// Every GEMM of an encode through rb_linear, with the parameters rb_encode_impl passes.
template <bool BF16>
static int rb_linear_probe(const void* a16, const void* w16, int M, int N, int K, const SatbGemmProbe& p,
                           cudaStream_t st) {
  TmapCache tc;
  auto out_ok = [&](int cols, int elem) {
    return p.out && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0 && p.ld >= cols && (p.ld * elem) % 16 == 0;
  };
  const bool bias_ok = p.bias && (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0;
  switch (p.epi) {
    case SATB_EPI_STORE16:   // QKV
      SATB_REQUIRE(N % 32 == 0 && out_ok(N, 2) && bias_ok,
                   "RoBERTa linear probe store16: N % 32 == 0, out and bias 16-byte aligned, ld >= N");
      return rb_linear<EpiStore16<BF16>, BF16>(tc, a16, M, K, w16, N,
                                              typename EpiStore16<BF16>::Params{p.out, p.ld, p.bias, 0}, st);
    case SATB_EPI_RESIDUAL:  // out-proj, FF-out
      SATB_REQUIRE(N % 8 == 0 && p.h && (reinterpret_cast<uintptr_t>(p.h) & 15) == 0 && p.ld == N && bias_ok,
                   "RoBERTa linear probe residual: N % 8 == 0, h and bias 16-byte aligned, ld == N");
      return rb_linear<EpiResidual, BF16>(tc, a16, M, K, w16, N, EpiResidual::Params{p.h, p.ld, p.bias, nullptr, 1, 0, 1},
                                          st);
    case SATB_EPI_STORE32:   // proj_out
      SATB_REQUIRE(N % 8 == 0 && out_ok(N, 4) && p.ld == N && bias_ok,
                   "RoBERTa linear probe store32: N % 8 == 0, out and bias 16-byte aligned, ld == N");
      return rb_linear<EpiStore32, BF16>(tc, a16, M, K, w16, N,
                                         EpiStore32::Params{static_cast<float*>(p.out), p.ld, p.bias}, st);
    case SATB_EPI_BIAS_GELU16:   // FF-in
      SATB_REQUIRE(N % 32 == 0 && out_ok(N, 2) && p.ld == N && bias_ok,
                   "RoBERTa linear probe bias_gelu16: N % 32 == 0, out and bias 16-byte aligned, ld == N");
      return rb_linear<EpiBiasGelu16<BF16>, BF16>(tc, a16, M, K, w16, N,
                                                  typename EpiBiasGelu16<BF16>::Params{p.out, p.ld, p.bias}, st);
    default:
      break;
  }
  set_last_error("RoBERTa linear probe: no such instance (epi " + std::to_string(p.epi) +
                 "); an encode runs store16 (1), residual (5), store32 (0) and bias_gelu16 (12)");
  return -1;
}

extern "C" {

int satb_roberta_linear_probe(const void* a16, const void* w16, int M, int N, int K, const SatbGemmProbe* p,
                              void* stream) {
  SATB_REQUIRE(a16 && w16 && p, "null argument");
  SATB_REQUIRE(M >= 1 && N >= 8 && K >= 8 && K % 8 == 0, "RoBERTa linear probe: need M >= 1, N >= 8 and K % 8 == 0");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(a16) & 15) == 0 && (reinterpret_cast<uintptr_t>(w16) & 15) == 0,
               "RoBERTa linear probe: operands must be 16-byte aligned");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return p->bf16 ? rb_linear_probe<true>(a16, w16, M, N, K, *p, st) : rb_linear_probe<false>(a16, w16, M, N, K, *p, st);
}

}  // extern "C"
