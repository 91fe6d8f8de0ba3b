// Host orchestration of the DiffusionTransformer forward (reference models/dit.py:135-364,
// models/transformer.py:656-809) on the kernels of this library.  One handle per
// (device, model); all work is enqueued on the caller's stream; no allocation and no
// synchronisation inside satb_dit_forward once the workspace has been reserved, so a
// whole denoise step can be captured in a CUDA graph.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/satb200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.h"
#include "linear.cuh"

namespace satb {

// Convolution over the tokens of every item (FeedForward use_conv, models/transformer.py:262-271, padding k / 2):
//   C[r * n_seq + l, n] = sum_t sum_c A[r, l + t - k / 2, c] * W[t * N + n, c]
// on the Linears' GEMM instances (n_taps = k, batches = R).  Rows outside an item's n_seq read as zeros (TMA zero fill),
// so each item, every CFG row included, is zero-padded at its own ends.  A: 16-bit [R, item_stride rows, K]; W: the
// tap-major weight [k * N, K]; C rows are dense ([R * n_seq] in the epilogue's row space).  The tiles are per item
// (ceil(n_seq / 128) m-tiles each).  bn: 0 picks the N tile as linear_auto does, over those m-tiles; else 128 or 256.
template <class Epi, bool BF16>
static int token_conv(TmapCache& tc, const void* A, int64_t item_stride, int R, int n_seq, int K, const void* W, int N,
                      int k, const typename Epi::Params& ep, cudaStream_t stream, int bn = 0) {
  if (bn == 0) bn = auto_bn(R * ceil_div(n_seq, kBlockM), N);
  const CUtensorMap *ta, *tb;
  SATB_PROPAGATE(tc.get_a(A, K, n_seq, R, K, item_stride * K, &ta));
  GemmShape s;
  s.L = n_seq; s.batches = R; s.N = N; s.K = K; s.n_taps = k; s.tap_base = -(k / 2); s.tap_step = 1; s.b_tap_rows = N;
  s.stride = 1; s.b_static = 1;
  SATB_PROPAGATE(tc.get_b(W, K, k * N, K, bn, &tb));
  if (bn == 128) return launch_gemm<Epi, 128, BF16>(*ta, *tb, s, ep, stream);
  return launch_gemm<Epi, 256, BF16>(*ta, *tb, s, ep, stream);
}

struct LayerW {
  float *pre_g = nullptr, *pre_b = nullptr, *ca_g = nullptr, *ca_b = nullptr, *ff_g = nullptr, *ff_b = nullptr;
  uint16_t *w_qkv = nullptr, *w_o = nullptr, *w_q = nullptr, *w_kv = nullptr, *w_co = nullptr, *w_ff1 = nullptr,
           *w_ff2 = nullptr;
  float *b_ff1 = nullptr, *b_ff2 = nullptr;
  // FP8 mode: e4m3 copies of to_qkv, cross_attn.to_q and ff.0 (in place of their 16-bit ones) and their row scales
  uint8_t *w8_qkv = nullptr, *w8_q = nullptr, *w8_ff1 = nullptr;
  float *s_qkv = nullptr, *s_q = nullptr, *s_ff1 = nullptr;
  // FP8 FF-out option (satb_dit_set_ff_out_fp8): the e4m3 copy of ff.2 (in place of w_ff2) and its row scales
  uint8_t* w8_ff2 = nullptr;
  float* s_ff2 = nullptr;
  // conformer branch (satb_dit_set_conformer): in_norm, glu.proj folded with pointwise_conv (16-bit, SwiGLU row
  // interleave, bias interleaved alike), depthwise_conv [D][17] fp32, mid_norm, pointwise_conv_2 (16-bit)
  float *cf_in_g = nullptr, *cf_in_b = nullptr, *cf_b1 = nullptr, *cf_dw = nullptr, *cf_mid_g = nullptr,
        *cf_mid_b = nullptr;
  uint16_t *cf_w1 = nullptr, *cf_w2 = nullptr;
  // fp32 copies of pointwise_conv [D, D] and glu.proj [2D, D] until both are loaded and folded into cf_w1 (then freed)
  float *cf_pw_src = nullptr, *cf_glu_src = nullptr;
};

}  // namespace satb

using namespace satb;

struct SatbDit {
  SatbDitConfig cfg;
  int D, H, dh, C, Cin, ct, ce, gd, ge, ffi, depth, F, nf;   // C = output channels, Cin = C + input_concat_dim
  // row pitches of project_in's input (Cin up to a multiple of 8: 16-byte TMA rows) and of project_out's output y (C up
  // to a multiple of 32: EpiStore32's column chunk).  The folded weights carry zero columns / rows in the padding, so
  // the padded products are exact; an aligned width pads nothing.
  int Cin_p, C_p;
  int pdim = 0;               // prepend_cond_dim
  float *pe0_w = nullptr, *pe2_w = nullptr;   // to_prepend_embed (fp32, bias-free)
  int Pp = 0;                 // prepend-conditioning tokens of the current conditioning
  DevBuf ws_prep;             // their embeddings [B, Pp, D] + scratch
  bool bf16, fp8, adaln, qk_norm = false;   // fp8: e4m3 operands for the QKV, cross q and FF-in GEMMs (fp16 elsewhere)
  bool conformer = false;     // every block runs the conformer branch (satb_dit_set_conformer)
  bool attn_fp8 = false;      // self-attention with e4m3 q, k, v and P (satb_dit_set_attention_fp8)
  bool ff_out_fp8 = false;    // FF-out on e4m3 operands, 1 x 128 block scales for the activations (satb_dit_set_ff_out_fp8)
  int* cf_perm = nullptr;     // SwiGLU row interleave of the folded [2D, D] conformer GLU weight
  // feed-forward (satb_dit_set_feedforward; default: SwiGLU Linear, inner 4D, biased).  ffi above is ff_inner padded up
  // to a multiple of 64.  ff_k: kernel size of the token convolutions, 0 = Linear (with ff_glu, FF-out only).  ff_bias:
  // FF-out (and a plain FF-in) carry a bias; the SwiGLU projection always does.
  int ff_inner = 0, ff_k = 0;
  bool ff_set = false, ff_glu = true, ff_bias = true;
  bool ff_conv_in() const { return !ff_glu && ff_k > 0; }
  // positions (satb_dit_set_positions; default: rotary, no embedding).  pos_type 1: ScaledSinusoidalEmbedding (pos_scale
  // [1], pos_inv [D / 2]); 2: AbsolutePositionalEmbedding (pos_emb [abs_max_len, D]).  ws_pos: the [pos_len, D] fp32
  // table project_in adds, built by satb_dit_reserve (pos_len 0: stale).
  bool rotary = true;
  int pos_type = 0, abs_max_len = 0, pos_len = 0;
  float *pos_scale = nullptr, *pos_inv = nullptr, *pos_emb = nullptr;
  DevBuf ws_pos;
  int P;  // prepended tokens: 1 (the global-conditioning token; 0 in adaLN mode) + Pp
  std::vector<LayerW> layers;
  std::vector<void*> owned;   // every cudaMalloc of weight storage
  // globals
  float *ts_w = nullptr, *te0_w = nullptr, *te0_b = nullptr, *te2_w = nullptr, *te2_b = nullptr;
  uint16_t *ce0_w = nullptr, *ce2_w = nullptr;
  float *ge0_w = nullptr, *ge2_w = nullptr;
  float *pre_w = nullptr, *post_w = nullptr, *pin_w = nullptr, *pout_w = nullptr, *inv_freq = nullptr;
  uint16_t *w_in16 = nullptr, *w_out16 = nullptr;
  float* w_ssg = nullptr;   // [depth*6D, D] fp32 (adaLN)
  int* ff_perm = nullptr;   // SwiGLU row interleave
  int* qkv_perm = nullptr;  // rotary pair layout of the q / k rows of to_qkv (null: identity, head dims 32 and 64)
  std::map<std::string, int> loaded;
  bool finalized = false;
  // conditioning state
  int B = 0, Mctx = 0, Rc = 0;  // Rc = rows that run cross-attention
  bool cfg_on = false, has_cross = false, has_global = false;
  // workspace
  TmapCache tmaps;
  DevBuf ws_h, ws_a16, ws_qkv, ws_attn, ws_q16, ws_ff, ws_ain, ws_y, ws_small, ws_cond, ws_kv, ws_rope;
  DevBuf ws_a8, ws_ascale;   // FP8 mode: e4m3 LayerNorm rows [M, D] and their scales [M]
  DevBuf ws_attn8;            // FP8 self-attention operands (attn_fp8_bufs), with their tensor maps for res_R rows
  AttnFp8Maps attn8_maps;
  int attn8_R = 0;            // the rows ws_attn8 is carved for and attn8_maps were made for (the last reserve_rows)
  int rope_len = 0;
  int res_R = 0, res_L = 0, res_P = -1;
  // bumped whenever weights, conditioning or workspaces may have moved or changed (satb_dit_finalize,
  // satb_dit_set_prepend_cond, satb_dit_prepare_cond, reserve_rows): a group's captured graph compares it at launch
  unsigned long long gen = 0;
  // optional per-category CUDA-event timing (bench.py roofline)
  bool prof_on = false;
  struct ProfRec { int cat; cudaEvent_t a, b; };
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> prof_pool;
  cudaEvent_t prof_event() {
    if (!prof_pool.empty()) { cudaEvent_t e = prof_pool.back(); prof_pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
  }

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

static bool ends_with(const std::string& s, const std::string& suf) {
  return s.size() >= suf.size() && s.compare(s.size() - suf.size(), suf.size(), suf) == 0;
}

// Source row of every stored row of to_qkv [3D, D] (the layout EpiQkvRope rotates, gemm.cuh): inside each q and k head,
// stored position 32 ci + i (i < 16) holds dim 16 ci + i and 32 ci + 16 + i holds its rotary partner 16 ci + i + nf,
// for the first clamp(nf - 16 ci, 0, 16) pairs of 32-column chunk ci; the dims from 2 nf up fill the remaining
// positions in order.  v rows are untouched.  Head dim 128 (nf 32): chunk 0 = [0..15 | 32..47], chunk 1 = [16..31 |
// 48..63], chunks 2-3 = 64..127.  Head dim 96 (nf 24): [0..15 | 24..39], [16..23, 48..55 | 40..47, 56..63], 64..95.
// Head dims 32 and 64 give the identity.
static std::vector<int> qkv_head_perm(int D, int dh, int nf) {
  std::vector<int> within(dh);
  int next_pass = 2 * nf;
  for (int s = 0; s < dh; ++s) {
    const int ci = s / 32, w = s % 32, i = w % 16;
    const int n_rot = std::min(std::max(nf - 16 * ci, 0), 16);
    within[s] = i < n_rot ? 16 * ci + i + (w >= 16 ? nf : 0) : next_pass++;
  }
  std::vector<int> perm(3 * D);
  for (int n = 0; n < 3 * D; ++n) perm[n] = n < 2 * D ? (n / dh) * dh + within[n % dh] : n;
  return perm;
}

// Row interleave of a [2 n, K] GLU projection for EpiSwiglu: every 64-row group = 32 value rows, then their 32 gate rows.
static std::vector<int> swiglu_perm(int n) {
  std::vector<int> perm(2 * n);
  for (int r = 0; r < 2 * n; ++r) {
    const int g = r / 64, w = r % 64;
    perm[r] = w < 32 ? g * 32 + w : n + g * 32 + (w - 32);
  }
  return perm;
}

// Conformer: W = W_glu W_pw ([2D, D], transformer.py:579-581: pointwise_conv then glu.proj, no nonlinearity between)
// with fp64 accumulation, rounded to fp32 and then to the 16-bit operand type in the SwiGLU row interleave; the fp32
// sources are freed.  Runs once both are loaded.
static int fold_conformer_glu(SatbDit* d, LayerW& L, cudaStream_t st) {
  const int D = d->D;
  float* fused = nullptr;
  SATB_CHECK_CUDA(cudaMalloc(&fused, static_cast<size_t>(2) * D * D * sizeof(float)));
  if (!L.cf_w1) {
    const int rc = d->alloc(&L.cf_w1, static_cast<size_t>(2) * D * D);
    if (rc) { cudaFree(fused); return rc; }
  }
  int rc = launch_matmul_f64(L.cf_glu_src, L.cf_pw_src, fused, 2 * D, D, D, st);
  if (rc == 0) rc = launch_cast_rows(fused, L.cf_w1, d->cf_perm, 2 * D, D, D, D, d->bf16, st);
  const cudaError_t e = cudaStreamSynchronize(st);
  cudaFree(fused);
  cudaFree(L.cf_pw_src);
  cudaFree(L.cf_glu_src);
  L.cf_pw_src = L.cf_glu_src = nullptr;
  SATB_PROPAGATE(rc);
  SATB_CHECK_CUDA(e);
  return 0;
}

// Stored fp32 layout of a feed-forward matrix of a satb_dit_set_feedforward variant, built on the host:
//   W [G * out, in, taps] (a Linear: taps = 1) -> [taps * G * out_p, in_p],  row (t G + g) out_p + n = W[g out + n, :, t]
// with zero rows and columns in the padding.  G = 2 for the GLU projection: its value and gate halves are padded
// separately, so the SwiGLU row interleave then applies at out_p.  A Conv1d weight comes out tap-major and K-major.
static std::vector<float> ff_stored_layout(const std::vector<float>& w, int G, int out, int in, int taps, int out_p,
                                           int in_p) {
  std::vector<float> s(static_cast<size_t>(taps) * G * out_p * in_p, 0.f);
  for (int t = 0; t < taps; ++t)
    for (int g = 0; g < G; ++g)
      for (int n = 0; n < out; ++n) {
        float* dst = s.data() + (static_cast<size_t>(t * G + g) * out_p + n) * in_p;
        const float* row = w.data() + static_cast<size_t>(g * out + n) * in * taps;
        for (int c = 0; c < in; ++c) dst[c] = row[static_cast<size_t>(c) * taps + t];
      }
  return s;
}

// One "ff.*" state-dict entry of a variant set by satb_dit_set_feedforward (the default keeps its own path in
// satb_dit_load_weight).  Keys, per transformer.py:258-284: ff.ff.0.proj.{weight, bias} (GLU, always biased) or
// ff.ff.0.1.weight [inner, D(, k)] (+ .bias); ff.ff.2.weight [D, inner(, k)] (+ .bias).  Returns 1 for a key the
// variant does not have.  Synchronous (load time only).
static int load_ff_weight(SatbDit* d, LayerW& L, const std::string& name, const std::string& k, const float* src,
                          long long numel, cudaStream_t st) {
  const int D = d->D, inner = d->ff_inner, ip = d->ffi, taps = d->ff_k > 0 ? d->ff_k : 1;
  enum { W_IN, B_IN, W_OUT, B_OUT } what;
  int G = 1, out, in = 1, tp = 1, out_p;
  if (d->ff_glu && k == "ff.ff.0.proj.weight") { what = W_IN; G = 2; out = inner; in = D; out_p = ip; }
  else if (d->ff_glu && k == "ff.ff.0.proj.bias") { what = B_IN; G = 2; out = inner; out_p = ip; }
  else if (!d->ff_glu && k == "ff.ff.0.1.weight") { what = W_IN; out = inner; in = D; tp = d->ff_conv_in() ? taps : 1; out_p = ip; }
  else if (!d->ff_glu && d->ff_bias && k == "ff.ff.0.1.bias") { what = B_IN; out = inner; out_p = ip; }
  else if (k == "ff.ff.2.weight") { what = W_OUT; out = D; in = inner; tp = taps; out_p = D; }
  else if (d->ff_bias && k == "ff.ff.2.bias") { what = B_OUT; out = D; out_p = D; }
  else return 1;
  SATB_REQUIRE(numel == static_cast<long long>(G) * out * in * tp, ("bad size for " + name).c_str());
  const int in_p = what == W_OUT ? ip : in;
  const int rows = tp * G * out_p;
  if (G == 2 && !d->ff_perm) {
    const std::vector<int> perm = swiglu_perm(ip);
    SATB_PROPAGATE(d->alloc(&d->ff_perm, perm.size()));
    SATB_CHECK_CUDA(cudaMemcpy(d->ff_perm, perm.data(), perm.size() * sizeof(int), cudaMemcpyHostToDevice));
  }
  std::vector<float> w(numel);
  SATB_CHECK_CUDA(cudaMemcpyAsync(w.data(), src, numel * sizeof(float), cudaMemcpyDeviceToHost, st));
  SATB_CHECK_CUDA(cudaStreamSynchronize(st));
  const std::vector<float> s = ff_stored_layout(w, G, out, in, tp, out_p, in_p);
  float* tmp = nullptr;
  SATB_CHECK_CUDA(cudaMalloc(&tmp, s.size() * sizeof(float)));
  int rc = 0;
  if (cudaMemcpy(tmp, s.data(), s.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
    set_last_error("cudaMemcpy of a feed-forward weight failed");
    rc = -2;
  }
  float** bias = what == B_IN ? &L.b_ff1 : &L.b_ff2;
  uint16_t** w16 = what == W_IN ? &L.w_ff1 : &L.w_ff2;
  if (rc == 0 && (what == B_IN || what == B_OUT)) {
    if (!*bias) rc = d->alloc(bias, rows);
    if (rc == 0 && G == 2) rc = launch_gather_f32(tmp, *bias, d->ff_perm, rows, st);
    else if (rc == 0 && cudaMemcpyAsync(*bias, tmp, rows * sizeof(float), cudaMemcpyDeviceToDevice, st) != cudaSuccess) rc = -2;
  } else if (rc == 0 && what == W_IN && d->fp8 && !d->ff_conv_in()) {   // e4m3 rows; the zero rows take scale 1
    if (!L.w8_ff1) rc = d->alloc(&L.w8_ff1, static_cast<size_t>(rows) * in_p);
    if (rc == 0 && !L.s_ff1) rc = d->alloc(&L.s_ff1, rows);
    if (rc == 0) rc = launch_quant_rows_fp8(tmp, L.w8_ff1, L.s_ff1, G == 2 ? d->ff_perm : nullptr, rows, in_p, st);
  } else if (rc == 0 && what == W_OUT && d->ff_out_fp8) {   // e4m3 rows; the zero pad columns leave the scales alone
    if (!L.w8_ff2) rc = d->alloc(&L.w8_ff2, static_cast<size_t>(rows) * in_p);
    if (rc == 0 && !L.s_ff2) rc = d->alloc(&L.s_ff2, rows);
    if (rc == 0) rc = launch_quant_rows_fp8(tmp, L.w8_ff2, L.s_ff2, nullptr, rows, in_p, st);
  } else if (rc == 0) {
    if (!*w16) rc = d->alloc(w16, static_cast<size_t>(rows) * in_p);
    if (rc == 0) rc = launch_cast_rows(tmp, *w16, G == 2 ? d->ff_perm : nullptr, rows, in_p, in_p, in_p, d->bf16, st);
  }
  const cudaError_t e = cudaStreamSynchronize(st);
  cudaFree(tmp);
  SATB_PROPAGATE(rc);
  SATB_CHECK_CUDA(e);
  return 0;
}

extern "C" {

const char* satb_last_error(void) { return get_last_error(); }
unsigned long long satb_launch_count(void) { return g_launch_count; }
void satb_reset_launch_count(void) { g_launch_count = 0; }
void satb_add_launch_count(unsigned long long n) { g_launch_count += n; }
int satb_abi_version(void) { return SATB_ABI_VERSION; }

int satb_dit_create(const SatbDitConfig* cfg, SatbDit** out) {
  SATB_REQUIRE(cfg && out, "null argument");
  SATB_REQUIRE(cfg->embed_dim % 128 == 0, "embed_dim must be a multiple of 128");
  // the LayerNorm holds a row in registers (<= 2048 wide); the conditioning MLPs stage K % 4 == 0, K <= 6400 inputs
  SATB_REQUIRE(cfg->embed_dim >= 128 && cfg->embed_dim <= 2048, "embed_dim must be between 128 and 2048");
  SATB_REQUIRE(cfg->global_cond_dim >= 0 && cfg->global_cond_dim % 4 == 0 && cfg->global_cond_dim <= 6400,
               "global_cond_dim must be a multiple of 4, at most 6400");
  SATB_REQUIRE(cfg->num_heads > 0 && cfg->embed_dim % cfg->num_heads == 0, "embed_dim must be a multiple of num_heads");
  const int dh = cfg->num_heads > 0 ? cfg->embed_dim / cfg->num_heads : 0;
  SATB_REQUIRE(dh == 32 || dh == 64 || dh == 96 || dh == 128, "head dim (embed_dim / num_heads) must be 32, 64, 96 or 128");
  SATB_REQUIRE(!(cfg->qk_norm && dh != 64), "qk_norm is supported with head dim 64 only");
  SATB_REQUIRE(cfg->io_channels >= 1, "io_channels must be >= 1");
  SATB_REQUIRE(cfg->patch_size == 1, "patch_size 1 only");
  SATB_REQUIRE(cfg->input_concat_dim >= 0, "input_concat_dim must be >= 0");
  SATB_REQUIRE(static_cast<long long>(cfg->io_channels) + cfg->input_concat_dim <= 32768,
               "io_channels + input_concat_dim must be at most 32768");
  SATB_REQUIRE(cfg->prepend_cond_dim >= 0 && cfg->prepend_cond_dim % 4 == 0 && cfg->prepend_cond_dim <= 6400,
               "prepend_cond_dim must be a multiple of 4, at most 6400");
  SATB_REQUIRE(!(cfg->prepend_cond_dim > 0 && cfg->global_cond_type == 1),
               "prepend conditioning is supported with global_cond_type \"prepend\" only");
  SATB_REQUIRE(cfg->operand_dtype >= 0 && cfg->operand_dtype <= 2, "operand_dtype must be 0 (fp16), 1 (bf16) or 2 (fp8)");
  SatbDit* d = new SatbDit();
  d->cfg = *cfg;
  d->D = cfg->embed_dim;
  d->H = cfg->num_heads;
  d->dh = d->D / d->H;
  d->C = cfg->io_channels;
  d->Cin = cfg->io_channels + (cfg->input_concat_dim > 0 ? cfg->input_concat_dim : 0);
  d->Cin_p = (d->Cin + 7) / 8 * 8;
  d->C_p = (d->C + 31) / 32 * 32;
  d->pdim = cfg->prepend_cond_dim > 0 ? cfg->prepend_cond_dim : 0;
  d->ct = cfg->cond_token_dim;
  d->ce = cfg->project_cond_tokens ? d->D : d->ct;
  d->gd = cfg->global_cond_dim;
  d->ge = cfg->project_global_cond ? d->D : d->gd;
  d->ffi = 4 * d->D;
  d->ff_inner = d->ffi;
  d->depth = cfg->depth;
  d->F = 128;  // timestep_features_dim 256 = cos | sin of 128 frequencies (models/dit.py:41-43)
  const int rot = d->dh / 2 > 32 ? d->dh / 2 : 32;  // models/transformer.py:737
  d->nf = rot / 2;
  d->bf16 = cfg->operand_dtype == 1;
  d->fp8 = cfg->operand_dtype == 2;
  d->adaln = cfg->global_cond_type == 1;
  d->qk_norm = cfg->qk_norm != 0;
  d->P = d->adaln ? 0 : 1;
  if (d->ct > 0) {
    // cross-attention kv heads = cond embed dim / head dim (models/transformer.py:306-312)
    if (d->ce % d->dh != 0 || d->H % (d->ce / d->dh) != 0) {
      delete d;
      set_last_error("cond embed dim must be a multiple of the head dim (" + std::to_string(d->dh) +
                     ") with kv heads dividing num_heads");
      return -1;
    }
  }
  if (d->gd > 0 && d->ge != d->D) {
    delete d;
    set_last_error("global embed dim must equal embed_dim");
    return -1;
  }
  d->layers.resize(d->depth);
  *out = d;
  return 0;
}

// Conformer blocks (transformer.py:557-591,645): call before the first satb_dit_load_weight.
int satb_dit_set_conformer(SatbDit* d, int enable) {
  SATB_REQUIRE(d, "null handle");
  SATB_REQUIRE(d->loaded.empty(), "satb_dit_set_conformer must be called before the first weight is loaded");
  SATB_REQUIRE(!enable || d->D <= kConformerMaxDim, "conformer blocks are supported up to embed_dim 1536");
  d->conformer = enable != 0;
  return 0;
}

// Feed-forward options (FeedForward, transformer.py:238-287): call before the first satb_dit_load_weight.
int satb_dit_set_feedforward(SatbDit* d, int inner_dim, int glu, int conv_kernel_size, int bias) {
  SATB_REQUIRE(d, "null handle");
  SATB_REQUIRE(d->loaded.empty(), "satb_dit_set_feedforward must be called before the first weight is loaded");
  SATB_REQUIRE(inner_dim >= 1, "feed-forward inner dim must be >= 1");
  SATB_REQUIRE(glu == 0 || glu == 1, "glu must be 0 or 1");
  SATB_REQUIRE(bias == 0 || bias == 1, "bias must be 0 or 1");
  SATB_REQUIRE(conv_kernel_size >= 0, "conv_kernel_size must be 0 (Linear) or a positive odd kernel size");
  SATB_REQUIRE(conv_kernel_size == 0 || conv_kernel_size % 2 == 1,
               "conv_kernel_size must be odd: an even kernel gives one output position more than the sequence");
  const long long inner_p = (static_cast<long long>(inner_dim) + 63) / 64 * 64;
  SATB_REQUIRE(inner_p * d->D * std::max(conv_kernel_size, 2) <= 0x7fffffffLL, "feed-forward weight too large");
  d->ff_set = true;
  d->ff_inner = inner_dim;
  d->ffi = static_cast<int>(inner_p);
  d->ff_glu = glu != 0;
  d->ff_k = conv_kernel_size;
  d->ff_bias = bias != 0;
  return 0;
}

// Positional options (ContinuousTransformer rotary_pos_emb / use_sinusoidal_emb / use_abs_pos_emb, transformer.py:50-96,
// 737-785): call before the first satb_dit_load_weight.
int satb_dit_set_positions(SatbDit* d, int rotary, int pos_type, int abs_max_len) {
  SATB_REQUIRE(d, "null handle");
  SATB_REQUIRE(d->loaded.empty(), "satb_dit_set_positions must be called before the first weight is loaded");
  SATB_REQUIRE(rotary == 0 || rotary == 1, "rotary must be 0 or 1");
  SATB_REQUIRE(pos_type >= 0 && pos_type <= 2, "pos_type must be 0 (none), 1 (sinusoidal) or 2 (absolute)");
  SATB_REQUIRE(pos_type == 2 ? abs_max_len >= 1 : abs_max_len == 0,
               "abs_max_len must be >= 1 with the absolute embedding (pos_type 2) and 0 otherwise");
  SATB_REQUIRE(static_cast<long long>(abs_max_len) * d->D <= 0x7fffffffLL, "absolute embedding too large");
  d->rotary = rotary != 0;
  d->pos_type = pos_type;
  d->abs_max_len = abs_max_len;
  return 0;
}

// FP8 self-attention (attention_fp8.cu): call before satb_dit_finalize.
int satb_dit_set_attention_fp8(SatbDit* d, int enable) {
  SATB_REQUIRE(d, "null handle");
  SATB_REQUIRE(enable == 0 || enable == 1, "enable must be 0 or 1");
  SATB_REQUIRE(!d->finalized, "satb_dit_set_attention_fp8 must be called before satb_dit_finalize");
  SATB_REQUIRE(!enable || d->dh == 64, "FP8 self-attention is supported with head dim 64 only");
  d->attn_fp8 = enable != 0;
  d->res_R = 0;   // the next forward reserves (and sizes the FP8 operands)
  return 0;
}

// FP8 FF-out (DESIGN.md sections 3-5): call before the first satb_dit_load_weight, after satb_dit_set_feedforward.
int satb_dit_set_ff_out_fp8(SatbDit* d, int enable) {
  SATB_REQUIRE(d, "null handle");
  SATB_REQUIRE(enable == 0 || enable == 1, "enable must be 0 or 1");
  SATB_REQUIRE(d->loaded.empty(), "satb_dit_set_ff_out_fp8 must be called before the first weight is loaded (it decides "
                                  "how ff.ff.2.weight is stored)");
  if (enable) {
    SATB_REQUIRE(d->fp8, "the FP8 FF-out option needs operand_dtype 2 (fp8)");
    SATB_REQUIRE(d->ff_k == 0, "the FP8 FF-out option is not supported with use_conv feed-forwards (FF-out is a token "
                               "convolution there)");
    SATB_REQUIRE(d->ffi % 128 == 0, ("the FP8 FF-out option needs a feed-forward inner width that is a multiple of 128 "
                                     "(padded to 64 it is " + std::to_string(d->ffi) + ")").c_str());
  }
  d->ff_out_fp8 = enable != 0;
  return 0;
}

void satb_dit_destroy(SatbDit* d) {
  if (!d) return;
  for (void* p : d->owned) cudaFree(p);
  for (LayerW& L : d->layers) {
    if (L.cf_pw_src) cudaFree(L.cf_pw_src);
    if (L.cf_glu_src) cudaFree(L.cf_glu_src);
  }
  d->ws_h.release(); d->ws_a16.release(); d->ws_qkv.release(); d->ws_attn.release(); d->ws_q16.release();
  d->ws_ff.release(); d->ws_ain.release(); d->ws_y.release(); d->ws_small.release(); d->ws_cond.release();
  d->ws_kv.release(); d->ws_rope.release(); d->ws_prep.release(); d->ws_a8.release(); d->ws_ascale.release();
  d->ws_pos.release(); d->ws_attn8.release();
  delete d;
}

// Upload one state-dict entry (fp32, device pointer, reference key relative to
// DiffusionTransformer; SURVEY.md 3.3).  Big matrices are cast to the 16-bit operand
// type here, once; small tensors stay fp32.
int satb_dit_load_weight(SatbDit* d, const char* name_c, const float* src, long long numel, void* stream_v) {
  SATB_REQUIRE(d && name_c && src, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  const std::string name(name_c);
  const int D = d->D, C = d->C, Cin = d->Cin;
  auto copy_f32 = [&](float** dst, long long expect) -> int {
    SATB_REQUIRE(numel == expect, ("bad size for " + name).c_str());
    if (!*dst) SATB_PROPAGATE(d->alloc(dst, expect));
    SATB_CHECK_CUDA(cudaMemcpyAsync(*dst, src, expect * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
  };
  auto cast16 = [&](uint16_t** dst, int rows, int cols, const int* perm) -> int {
    SATB_REQUIRE(numel == static_cast<long long>(rows) * cols, ("bad size for " + name).c_str());
    if (!*dst) SATB_PROPAGATE(d->alloc(dst, static_cast<size_t>(rows) * cols));
    return launch_cast_rows(src, *dst, perm, rows, cols, cols, cols, d->bf16, st);
  };
  // FP8 mode: e4m3 rows with one power-of-two scale per stored row, taken after the row permutation
  auto quant8 = [&](uint8_t** dst, float** scale, int rows, int cols, const int* perm) -> int {
    SATB_REQUIRE(numel == static_cast<long long>(rows) * cols, ("bad size for " + name).c_str());
    if (!*dst) SATB_PROPAGATE(d->alloc(dst, static_cast<size_t>(rows) * cols));
    if (!*scale) SATB_PROPAGATE(d->alloc(scale, rows));
    return launch_quant_rows_fp8(src, *dst, *scale, perm, rows, cols, st);
  };
  d->finalized = false;
  d->loaded[name] = 1;
  if (name == "timestep_features.weight") return copy_f32(&d->ts_w, d->F);
  if (name == "to_timestep_embed.0.weight") return copy_f32(&d->te0_w, static_cast<long long>(D) * 2 * d->F);
  if (name == "to_timestep_embed.0.bias") return copy_f32(&d->te0_b, D);
  if (name == "to_timestep_embed.2.weight") return copy_f32(&d->te2_w, static_cast<long long>(D) * D);
  if (name == "to_timestep_embed.2.bias") return copy_f32(&d->te2_b, D);
  if (name == "to_cond_embed.0.weight") return cast16(&d->ce0_w, d->ce, d->ct, nullptr);
  if (name == "to_cond_embed.2.weight") return cast16(&d->ce2_w, d->ce, d->ce, nullptr);
  if (name == "to_global_embed.0.weight") return copy_f32(&d->ge0_w, static_cast<long long>(d->ge) * d->gd);
  if (name == "to_global_embed.2.weight") return copy_f32(&d->ge2_w, static_cast<long long>(d->ge) * d->ge);
  if (name == "preprocess_conv.weight") return copy_f32(&d->pre_w, static_cast<long long>(Cin) * Cin);
  if (name == "to_prepend_embed.0.weight" && d->pdim > 0) return copy_f32(&d->pe0_w, static_cast<long long>(D) * d->pdim);
  if (name == "to_prepend_embed.2.weight" && d->pdim > 0) return copy_f32(&d->pe2_w, static_cast<long long>(D) * D);
  if (name == "postprocess_conv.weight") return copy_f32(&d->post_w, static_cast<long long>(C) * C);
  if (name == "transformer.project_in.weight") return copy_f32(&d->pin_w, static_cast<long long>(D) * Cin);
  if (name == "transformer.project_out.weight") return copy_f32(&d->pout_w, static_cast<long long>(C) * D);
  if (name == "transformer.rotary_pos_emb.inv_freq" && d->rotary) return copy_f32(&d->inv_freq, d->nf);
  // the sinusoid's inv_freq is a non-persistent buffer of the reference: the caller hands it over under this key
  if (d->pos_type == 1 && name == "transformer.pos_emb.scale") return copy_f32(&d->pos_scale, 1);
  if (d->pos_type == 1 && name == "transformer.pos_emb.inv_freq") return copy_f32(&d->pos_inv, D / 2);
  if (d->pos_type == 2 && name == "transformer.pos_emb.emb.weight")
    return copy_f32(&d->pos_emb, static_cast<long long>(d->abs_max_len) * D);
  const std::string lp = "transformer.layers.";
  if (name.compare(0, lp.size(), lp) == 0) {
    const size_t dot = name.find('.', lp.size());
    SATB_REQUIRE(dot != std::string::npos, ("bad key " + name).c_str());
    const int li = atoi(name.substr(lp.size(), dot - lp.size()).c_str());
    SATB_REQUIRE(li >= 0 && li < d->depth, ("layer index out of range in " + name).c_str());
    LayerW& L = d->layers[li];
    const std::string k = name.substr(dot + 1);
    if (k == "pre_norm.gamma") return copy_f32(&L.pre_g, D);
    if (k == "pre_norm.beta") return copy_f32(&L.pre_b, D);
    if (k == "cross_attend_norm.gamma") return copy_f32(&L.ca_g, D);
    if (k == "cross_attend_norm.beta") return copy_f32(&L.ca_b, D);
    if (k == "ff_norm.gamma") return copy_f32(&L.ff_g, D);
    if (k == "ff_norm.beta") return copy_f32(&L.ff_b, D);
    if (d->ff_set && k.compare(0, 3, "ff.") == 0) {
      const int rc = load_ff_weight(d, L, name, k, src, numel, st);
      if (rc != 1) return rc;
      d->loaded.erase(name);
      set_last_error("unknown DiT weight key: " + name + " (not a key of this model's feed-forward variant)");
      return -4;
    }
    if (k == "self_attn.to_qkv.weight") {
      if (!d->qkv_perm && d->dh != 32 && d->dh != 64) {
        const std::vector<int> perm = qkv_head_perm(D, d->dh, d->nf);
        SATB_PROPAGATE(d->alloc(&d->qkv_perm, perm.size()));
        SATB_CHECK_CUDA(cudaMemcpy(d->qkv_perm, perm.data(), perm.size() * sizeof(int), cudaMemcpyHostToDevice));
      }
      return d->fp8 ? quant8(&L.w8_qkv, &L.s_qkv, 3 * D, D, d->qkv_perm) : cast16(&L.w_qkv, 3 * D, D, d->qkv_perm);
    }
    if (k == "self_attn.to_out.weight") return cast16(&L.w_o, D, D, nullptr);
    if (k == "cross_attn.to_q.weight") return d->fp8 ? quant8(&L.w8_q, &L.s_q, D, D, nullptr) : cast16(&L.w_q, D, D, nullptr);
    if (k == "cross_attn.to_kv.weight") return cast16(&L.w_kv, 2 * d->ce, d->ce, nullptr);
    if (k == "cross_attn.to_out.weight") return cast16(&L.w_co, D, D, nullptr);
    if (k == "ff.ff.0.proj.weight" || k == "ff.ff.0.proj.bias") {
      if (!d->ff_perm) {
        // interleave so that every 64-row group = 32 value rows then their 32 gate rows
        const std::vector<int> perm = swiglu_perm(d->ffi);
        SATB_PROPAGATE(d->alloc(&d->ff_perm, perm.size()));
        SATB_CHECK_CUDA(cudaMemcpy(d->ff_perm, perm.data(), perm.size() * sizeof(int), cudaMemcpyHostToDevice));
      }
      if (ends_with(k, "weight"))
        return d->fp8 ? quant8(&L.w8_ff1, &L.s_ff1, 2 * d->ffi, D, d->ff_perm) : cast16(&L.w_ff1, 2 * d->ffi, D, d->ff_perm);
      SATB_REQUIRE(numel == 2 * d->ffi, ("bad size for " + name).c_str());
      if (!L.b_ff1) SATB_PROPAGATE(d->alloc(&L.b_ff1, 2 * d->ffi));
      return launch_gather_f32(src, L.b_ff1, d->ff_perm, 2 * d->ffi, st);
    }
    if (k == "ff.ff.2.weight")
      return d->ff_out_fp8 ? quant8(&L.w8_ff2, &L.s_ff2, D, d->ffi, nullptr) : cast16(&L.w_ff2, D, d->ffi, nullptr);
    if (k == "ff.ff.2.bias") return copy_f32(&L.b_ff2, D);
    if (k == "to_scale_shift_gate.1.weight") {
      SATB_REQUIRE(numel == 6LL * D * D, ("bad size for " + name).c_str());
      if (!d->w_ssg) SATB_PROPAGATE(d->alloc(&d->w_ssg, static_cast<size_t>(d->depth) * 6 * D * D));
      SATB_CHECK_CUDA(cudaMemcpyAsync(d->w_ssg + static_cast<size_t>(li) * 6 * D * D, src, numel * sizeof(float),
                                      cudaMemcpyDeviceToDevice, st));
      return 0;
    }
    const std::string cp = "conformer.";
    if (d->conformer && k.compare(0, cp.size(), cp) == 0) {   // transformer.py:557-574
      const std::string c = k.substr(cp.size());
      if (!d->cf_perm) {
        const std::vector<int> perm = swiglu_perm(D);
        SATB_PROPAGATE(d->alloc(&d->cf_perm, perm.size()));
        SATB_CHECK_CUDA(cudaMemcpy(d->cf_perm, perm.data(), perm.size() * sizeof(int), cudaMemcpyHostToDevice));
      }
      if (c == "in_norm.gamma") return copy_f32(&L.cf_in_g, D);
      if (c == "in_norm.beta") return copy_f32(&L.cf_in_b, D);
      if (c == "mid_norm.gamma") return copy_f32(&L.cf_mid_g, D);
      if (c == "mid_norm.beta") return copy_f32(&L.cf_mid_b, D);
      if (c == "depthwise_conv.weight") return copy_f32(&L.cf_dw, 17LL * D);   // [D, 1, 17]
      if (c == "pointwise_conv_2.weight") return cast16(&L.cf_w2, D, D, nullptr);   // [D, D, 1]
      if (c == "glu.proj.bias") {
        SATB_REQUIRE(numel == 2LL * D, ("bad size for " + name).c_str());
        if (!L.cf_b1) SATB_PROPAGATE(d->alloc(&L.cf_b1, 2 * D));
        return launch_gather_f32(src, L.cf_b1, d->cf_perm, 2 * D, st);
      }
      if (c == "pointwise_conv.weight" || c == "glu.proj.weight") {
        const bool pw = c == "pointwise_conv.weight";
        float** dst = pw ? &L.cf_pw_src : &L.cf_glu_src;
        const long long n = (pw ? 1LL : 2LL) * D * D;
        SATB_REQUIRE(numel == n, ("bad size for " + name).c_str());
        if (!*dst) SATB_CHECK_CUDA(cudaMalloc(dst, n * sizeof(float)));
        SATB_CHECK_CUDA(cudaMemcpyAsync(*dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
        if (L.cf_pw_src && L.cf_glu_src) return fold_conformer_glu(d, L, st);
        return 0;
      }
    }
  }
  d->loaded.erase(name);
  set_last_error("unknown DiT weight key: " + name);
  return -4;
}

// Folds the 1x1 pre/post convolutions into project_in / project_out
// (x + Wpre x then Win: Win (I + Wpre); Wout then y + Wpost y: (I + Wpost) Wout;
// models/dit.py:197,224 with transformer.py:778,807) and checks completeness.
int satb_dit_finalize(SatbDit* d, void* stream_v) {
  SATB_REQUIRE(d, "null handle");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  const int D = d->D, C = d->C;
  if (d->conformer) {
    for (int i = 0; i < d->depth; ++i) {
      const LayerW& L = d->layers[i];
      // cf_w1 is the fold of pointwise_conv and glu.proj; a source still pending means its partner is missing
      if (!(L.cf_in_g && L.cf_in_b && L.cf_w1 && !L.cf_pw_src && !L.cf_glu_src && L.cf_b1 && L.cf_dw && L.cf_mid_g &&
            L.cf_mid_b && L.cf_w2)) {
        set_last_error("conformer weights missing in layer " + std::to_string(i) + ": every block needs conformer." +
                       "{in_norm.gamma, in_norm.beta, pointwise_conv.weight, glu.proj.weight, glu.proj.bias, "
                       "depthwise_conv.weight, mid_norm.gamma, mid_norm.beta, pointwise_conv_2.weight}");
        return -1;
      }
    }
  }
  if (d->ff_set) {
    const bool in8 = d->fp8 && !d->ff_conv_in();
    for (int i = 0; i < d->depth; ++i) {
      const LayerW& L = d->layers[i];
      const std::string p = "transformer.layers." + std::to_string(i) + ".ff.ff.";
      std::string miss;
      auto need = [&](bool ok, const char* key) { if (!ok) miss += (miss.empty() ? "" : ", ") + p + key; };
      need(in8 ? L.w8_ff1 != nullptr : L.w_ff1 != nullptr, d->ff_glu ? "0.proj.weight" : "0.1.weight");
      if (d->ff_glu) need(L.b_ff1 != nullptr, "0.proj.bias");
      else if (d->ff_bias) need(L.b_ff1 != nullptr, "0.1.bias");
      need(d->ff_out_fp8 ? L.w8_ff2 != nullptr : L.w_ff2 != nullptr, "2.weight");
      if (d->ff_bias) need(L.b_ff2 != nullptr, "2.bias");
      if (!miss.empty()) {
        set_last_error("feed-forward weights missing in layer " + std::to_string(i) + ": " + miss);
        return -1;
      }
    }
  }
  if (d->pos_type == 1 && !(d->pos_scale && d->pos_inv)) {
    set_last_error(std::string("sinusoidal positional embedding missing: ") +
                   (d->pos_scale ? "" : "transformer.pos_emb.scale ") + (d->pos_inv ? "" : "transformer.pos_emb.inv_freq"));
    return -1;
  }
  if (d->pos_type == 2) SATB_REQUIRE(d->pos_emb, "absolute positional embedding missing: transformer.pos_emb.emb.weight");
  // satb_dit_set_feedforward may follow satb_dit_set_ff_out_fp8
  SATB_REQUIRE(!d->ff_out_fp8 || (d->ff_k == 0 && d->ffi % 128 == 0),
               "the FP8 FF-out option needs a Linear feed-forward whose inner width is a multiple of 128");
  SATB_REQUIRE(d->ts_w && d->te0_w && d->te0_b && d->te2_w && d->te2_b, "timestep embedding weights missing");
  SATB_REQUIRE(d->pin_w && d->pout_w && d->pre_w && d->post_w, "project_in/out or pre/post conv weights missing");
  if (d->rotary) SATB_REQUIRE(d->inv_freq, "rotary inv_freq missing");
  d->pos_len = 0;   // rebuilt from the (re)loaded scale / embedding by the next satb_dit_reserve
  if (d->ct > 0) SATB_REQUIRE(d->ce0_w && d->ce2_w, "to_cond_embed weights missing");
  if (d->gd > 0) SATB_REQUIRE(d->ge0_w && d->ge2_w, "to_global_embed weights missing");
  for (int i = 0; i < d->depth; ++i) {
    const LayerW& L = d->layers[i];
    const bool ff_in8 = d->fp8 && !d->ff_conv_in();   // a token-convolution FF-in keeps 16-bit weights in every mode
    SATB_REQUIRE(L.pre_g && L.ff_g && (d->fp8 ? L.w8_qkv != nullptr : L.w_qkv != nullptr) &&
                     (ff_in8 ? L.w8_ff1 != nullptr : L.w_ff1 != nullptr) && L.w_o &&
                     (d->ff_out_fp8 ? L.w8_ff2 != nullptr : L.w_ff2 != nullptr),
                 "transformer layer weights missing");
    if (d->ct > 0)
      SATB_REQUIRE(L.ca_g && (d->fp8 ? L.w8_q != nullptr : L.w_q != nullptr) && L.w_kv && L.w_co,
                   "cross-attention weights missing");
  }
  if (d->adaln) SATB_REQUIRE(d->w_ssg, "adaLN to_scale_shift_gate weights missing");
  SATB_CHECK_CUDA(cudaStreamSynchronize(st));
  const int Cin = d->Cin;
  if (d->pdim > 0) SATB_REQUIRE(d->pe0_w && d->pe2_w, "to_prepend_embed weights missing");
  std::vector<float> pin(static_cast<size_t>(D) * Cin), pout(static_cast<size_t>(C) * D), pre(Cin * Cin), post(C * C);
  SATB_CHECK_CUDA(cudaMemcpy(pin.data(), d->pin_w, pin.size() * 4, cudaMemcpyDeviceToHost));
  SATB_CHECK_CUDA(cudaMemcpy(pout.data(), d->pout_w, pout.size() * 4, cudaMemcpyDeviceToHost));
  SATB_CHECK_CUDA(cudaMemcpy(pre.data(), d->pre_w, pre.size() * 4, cudaMemcpyDeviceToHost));
  SATB_CHECK_CUDA(cudaMemcpy(post.data(), d->post_w, post.size() * 4, cudaMemcpyDeviceToHost));
  // stored at the padded pitches: fin [D, Cin_p] with zero columns Cin .., fout [C_p, D] with zero rows C ..
  const int Cin_p = d->Cin_p, C_p = d->C_p;
  std::vector<float> fin(static_cast<size_t>(D) * Cin_p, 0.f), fout(static_cast<size_t>(C_p) * D, 0.f);
  for (int n = 0; n < D; ++n)
    for (int c = 0; c < Cin; ++c) {
      double acc = pin[static_cast<size_t>(n) * Cin + c];
      for (int j = 0; j < Cin; ++j) acc += static_cast<double>(pin[static_cast<size_t>(n) * Cin + j]) * pre[j * Cin + c];
      fin[static_cast<size_t>(n) * Cin_p + c] = static_cast<float>(acc);
    }
  for (int c = 0; c < C; ++c)
    for (int k = 0; k < D; ++k) {
      double acc = pout[static_cast<size_t>(c) * D + k];
      for (int j = 0; j < C; ++j) acc += static_cast<double>(post[c * C + j]) * pout[static_cast<size_t>(j) * D + k];
      fout[static_cast<size_t>(c) * D + k] = static_cast<float>(acc);
    }
  float *tmp_in = nullptr, *tmp_out = nullptr;
  SATB_CHECK_CUDA(cudaMalloc(&tmp_in, fin.size() * 4));
  SATB_CHECK_CUDA(cudaMalloc(&tmp_out, fout.size() * 4));
  SATB_CHECK_CUDA(cudaMemcpy(tmp_in, fin.data(), fin.size() * 4, cudaMemcpyHostToDevice));
  SATB_CHECK_CUDA(cudaMemcpy(tmp_out, fout.data(), fout.size() * 4, cudaMemcpyHostToDevice));
  if (!d->w_in16) SATB_PROPAGATE(d->alloc(&d->w_in16, fin.size()));
  if (!d->w_out16) SATB_PROPAGATE(d->alloc(&d->w_out16, fout.size()));
  int rc = launch_cast_rows(tmp_in, d->w_in16, nullptr, D, Cin_p, Cin_p, Cin_p, d->bf16, st);
  if (rc == 0) rc = launch_cast_rows(tmp_out, d->w_out16, nullptr, C_p, D, D, D, d->bf16, st);
  cudaStreamSynchronize(st);
  cudaFree(tmp_in);
  cudaFree(tmp_out);
  SATB_PROPAGATE(rc);
  d->tmaps.maps.clear();
  d->finalized = true;
  ++d->gen;
  return 0;
}

}  // extern "C"

static int ensure_rope(SatbDit* d, int N_seq) {
  if (d->rope_len == N_seq) return 0;
  // models/transformer.py:130-155: freqs[p, j] = float(p) * inv_freq[j] in fp32; cos/sin in fp32.
  std::vector<float> inv(d->nf), tab(static_cast<size_t>(2) * N_seq * d->nf);
  SATB_CHECK_CUDA(cudaMemcpy(inv.data(), d->inv_freq, d->nf * 4, cudaMemcpyDeviceToHost));
  for (int p = 0; p < N_seq; ++p)
    for (int j = 0; j < d->nf; ++j) {
      const float f = static_cast<float>(p) * inv[j];
      tab[static_cast<size_t>(p) * d->nf + j] = cosf(f);
      tab[static_cast<size_t>(N_seq) * d->nf + static_cast<size_t>(p) * d->nf + j] = sinf(f);
    }
  SATB_PROPAGATE(d->ws_rope.ensure(tab.size() * 4));
  SATB_CHECK_CUDA(cudaMemcpy(d->ws_rope.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
  d->rope_len = N_seq;
  return 0;
}

// The [N_seq, D] fp32 table project_in adds (transformer.py:784-785), position p = row within the item, prepended rows
// included.  Sinusoidal (:74-96): cat(sin(p inv_freq), cos(p inv_freq)) * scale, with the product p * inv_freq in fp32
// and the reference's own inv_freq.  Absolute (:50-71): emb.weight[p] * fp32(D ** -0.5).
static int ensure_pos(SatbDit* d, int N_seq) {
  if (d->pos_len == N_seq) return 0;
  const int D = d->D, half = D / 2;
  std::vector<float> tab(static_cast<size_t>(N_seq) * D);
  if (d->pos_type == 1) {
    std::vector<float> inv(half);
    float scale = 0.f;
    SATB_CHECK_CUDA(cudaMemcpy(inv.data(), d->pos_inv, half * 4, cudaMemcpyDeviceToHost));
    SATB_CHECK_CUDA(cudaMemcpy(&scale, d->pos_scale, 4, cudaMemcpyDeviceToHost));
    for (int p = 0; p < N_seq; ++p)
      for (int j = 0; j < half; ++j) {
        const float f = static_cast<float>(p) * inv[j];
        tab[static_cast<size_t>(p) * D + j] = sinf(f) * scale;
        tab[static_cast<size_t>(p) * D + half + j] = cosf(f) * scale;
      }
  } else {
    SATB_CHECK_CUDA(cudaMemcpy(tab.data(), d->pos_emb, tab.size() * 4, cudaMemcpyDeviceToHost));
    const float s = static_cast<float>(std::pow(static_cast<double>(D), -0.5));
    for (float& v : tab) v *= s;
  }
  SATB_PROPAGATE(d->ws_pos.ensure(tab.size() * 4));
  SATB_CHECK_CUDA(cudaMemcpy(d->ws_pos.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
  d->pos_len = N_seq;
  return 0;
}

// The shape of the last reserve no longer fits, or the position table is stale (weights reloaded).
static bool needs_reserve(const SatbDit* d, int R, int L) {
  return R > d->res_R || L != d->res_L || d->P != d->res_P || (d->pos_type != 0 && d->pos_len != L + d->P);
}

// Every activation buffer for R rows of n tokens, and the rotary / positional tables for tab_len positions (n = tab_len
// for the single-device forward; a rank of a group forward holds n of the tab_len tokens).  Grow-only.
static int reserve_rows(SatbDit* d, int R, int n, int tab_len) {
  const int N_seq = n;
  if (d->pos_type == 2 && tab_len > d->abs_max_len) {
    set_last_error("sequence length " + std::to_string(tab_len) + " (latent tokens + prepended tokens) exceeds the absolute "
                   "positional embedding's max length " + std::to_string(d->abs_max_len));
    return -1;
  }
  const size_t M = static_cast<size_t>(R) * N_seq;
  const int D = d->D;
  SATB_PROPAGATE(d->ws_h.ensure(M * D * 4));
  SATB_PROPAGATE(d->ws_a16.ensure(M * D * 2));
  SATB_PROPAGATE(d->ws_qkv.ensure(M * 3 * D * 2));
  SATB_PROPAGATE(d->ws_attn.ensure(M * D * 2));
  SATB_PROPAGATE(d->ws_q16.ensure(M * D * 2));
  // the FF intermediate [M, ffi] (FP8 FF-out: e4m3 [M, ffi], then its scales [M, ffi / 128], in fewer bytes), and the
  // conformer branch's two [M, D] intermediates
  SATB_PROPAGATE(d->ws_ff.ensure(M * std::max(d->ffi, d->conformer ? 2 * D : 0) * 2));
  SATB_PROPAGATE(d->ws_ain.ensure(M * d->Cin_p * 2));
  SATB_PROPAGATE(d->ws_y.ensure(M * d->C_p * 4));
  if (d->fp8) {
    SATB_PROPAGATE(d->ws_a8.ensure(M * D));
    SATB_PROPAGATE(d->ws_ascale.ensure(M * 4));
  }
  if (d->attn_fp8) {
    SATB_PROPAGATE(d->ws_attn8.ensure(attn_fp8_workspace_bytes(R, d->H, N_seq, N_seq)));
    // the q / k scales past each item's tokens are never written (the core masks those keys): zero, once
    SATB_CHECK_CUDA(cudaMemset(d->ws_attn8.p, 0, attn_fp8_workspace_bytes(R, d->H, N_seq, N_seq)));
    SATB_PROPAGATE(make_attention_fp8_maps(&d->attn8_maps, attn_fp8_bufs(d->ws_attn8.p, R, d->H, N_seq, N_seq), R, d->H,
                                           N_seq, N_seq));
    d->attn8_R = R;
  }
  if (d->rotary) SATB_PROPAGATE(ensure_rope(d, tab_len));
  if (d->pos_type != 0) SATB_PROPAGATE(ensure_pos(d, tab_len));
  d->tmaps.maps.clear();
  ++d->gen;
  return 0;
}

extern "C" {

// Reserve every activation buffer for R rows of L latent tokens (synchronous; call
// before capturing a CUDA graph).  Grow-only.
int satb_dit_reserve(SatbDit* d, int R, int L) {
  SATB_REQUIRE(d && d->finalized, "weights not finalized");
  SATB_REQUIRE(R >= 1 && L >= 1, "bad shape");
  SATB_PROPAGATE(reserve_rows(d, R, L + d->P, L + d->P));
  d->res_R = R;
  d->res_L = L;
  d->res_P = d->P;
  return 0;
}

}  // extern "C"

struct SmallWs {
  float *fourier, *te_h, *tok, *ge_h, *ge, *ssg;
};
static SmallWs small_ws(SatbDit* d, int R) {
  SmallWs s;
  float* p = d->ws_small.as<float>();
  s.fourier = p; p += static_cast<size_t>(R) * 2 * d->F;
  s.te_h = p;    p += static_cast<size_t>(R) * d->D;
  s.tok = p;     p += static_cast<size_t>(R) * d->D;
  s.ge_h = p;    p += static_cast<size_t>(R) * d->D;
  s.ge = p;      p += static_cast<size_t>(R) * d->D;
  s.ssg = p;
  return s;
}

extern "C" {

// Prepend conditioning of the next prepare_cond: embeds = W2 silu(W0 prepend) (dit.py:75-81,157-161), kept as fp32
// tokens [B, Pp, D]; the unconditional CFG rows use zeros (to_prepend_embed is bias-free, so MLP(0) = 0, dit.py:309-311).
int satb_dit_set_prepend_cond(SatbDit* d, const float* prepend, int B, int n_tokens, void* stream_v) {
  SATB_REQUIRE(d && d->finalized, "weights not finalized");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  ++d->gen;
  if (!prepend || n_tokens <= 0) {
    d->Pp = 0;
    d->P = d->adaln ? 0 : 1;
    return 0;
  }
  SATB_REQUIRE(d->pdim > 0 && !d->adaln, "this model has no prepend conditioning");
  SATB_REQUIRE(B >= 1, "bad batch");
  const size_t rows = static_cast<size_t>(B) * n_tokens;
  SATB_REQUIRE(rows <= 4096, "too many prepend tokens");
  SATB_PROPAGATE(d->ws_prep.ensure(2 * rows * d->D * sizeof(float)));
  float* emb = d->ws_prep.as<float>();
  float* hid = emb + rows * d->D;
  SATB_PROPAGATE(launch_skinny_linear(prepend, d->pe0_w, nullptr, nullptr, hid, static_cast<int>(rows), d->pdim, d->D, 1, st));
  SATB_PROPAGATE(launch_skinny_linear(hid, d->pe2_w, nullptr, nullptr, emb, static_cast<int>(rows), d->D, d->D, 0, st));
  d->Pp = n_tokens;
  d->P = 1 + n_tokens;
  return 0;
}

// Step-invariant conditioning work hoisted out of the sampler loop (SURVEY.md 8a a2/a8):
// to_cond_embed, to_global_embed and every layer's cross-attention k/v projection.
//   cross [B, Mctx, ct] fp32 or null; neg_cross [B, Mctx, ct] fp32 or null (already masked);
//   global [B, gd] fp32 or null; use_cfg: rows are doubled (cond rows first, uncond rows second).
int satb_dit_prepare_cond(SatbDit* d, const float* cross, const float* neg_cross, const float* global, int B, int Mctx,
                          int use_cfg, void* stream_v) {
  SATB_REQUIRE(d && d->finalized, "weights not finalized");
  SATB_REQUIRE(B >= 1, "bad batch");
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  const int D = d->D;
  ++d->gen;
  d->B = B;
  d->cfg_on = use_cfg != 0;
  d->has_cross = cross != nullptr && d->ct > 0;
  d->has_global = global != nullptr && d->gd > 0;
  d->Mctx = d->has_cross ? Mctx : 0;
  // rows with a non-null context: cond rows, plus the uncond rows iff a negative prompt is given
  // (a null (zero) context makes the bias-free cross-attention branch exactly 0: SURVEY.md H5)
  d->Rc = d->has_cross ? ((d->cfg_on && neg_cross) ? 2 * B : B) : 0;
  SATB_REQUIRE(!(neg_cross && !d->cfg_on), "negative conditioning requires CFG");
  SATB_PROPAGATE(d->ws_small.ensure(static_cast<size_t>(2 * B) * (2 * d->F + 4 * D + 6 * D * d->depth) * 4 + 4096));
  SmallWs sw = small_ws(d, 2 * B);
  if (d->has_global) {
    SATB_PROPAGATE(launch_skinny_linear(global, d->ge0_w, nullptr, nullptr, sw.ge_h, B, d->gd, d->ge, 1, st));
    SATB_PROPAGATE(launch_skinny_linear(sw.ge_h, d->ge2_w, nullptr, nullptr, sw.ge, B, d->ge, d->ge, 0, st));
  }
  if (d->has_cross) {
    SATB_REQUIRE(Mctx >= 1, "empty cross-attention context");
    const size_t rows = static_cast<size_t>(d->Rc) * Mctx;
    const size_t in_b = rows * d->ct * 2, mid_b = rows * d->ce * 2;
    SATB_PROPAGATE(d->ws_cond.ensure(in_b + 2 * mid_b + 1024));
    uint16_t* in16 = d->ws_cond.as<uint16_t>();
    uint16_t* mid16 = in16 + rows * d->ct;
    uint16_t* ce16 = mid16 + rows * d->ce;
    SATB_PROPAGATE(launch_cast_rows(cross, in16, nullptr, B * Mctx, d->ct, d->ct, d->ct, d->bf16, st));
    if (d->Rc == 2 * B)
      SATB_PROPAGATE(launch_cast_rows(neg_cross, in16 + static_cast<size_t>(B) * Mctx * d->ct, nullptr, B * Mctx,
                                      d->ct, d->ct, d->ct, d->bf16, st));
    SATB_PROPAGATE(d->ws_kv.ensure(static_cast<size_t>(d->depth) * rows * 2 * d->ce * 2));
    d->tmaps.maps.clear();
    const int Mr = static_cast<int>(rows);
    if (d->bf16) {
      typedef EpiStore16<true> E;
      SATB_PROPAGATE((linear<E, 128, true>(d->tmaps, in16, d->ct, Mr, d->ct, d->ce0_w, d->ce, E::Params{mid16, d->ce, nullptr, 1}, st)));
      SATB_PROPAGATE((linear<E, 128, true>(d->tmaps, mid16, d->ce, Mr, d->ce, d->ce2_w, d->ce, E::Params{ce16, d->ce, nullptr, 0}, st)));
      for (int i = 0; i < d->depth; ++i) {
        uint16_t* kv = d->ws_kv.as<uint16_t>() + static_cast<size_t>(i) * rows * 2 * d->ce;
        if (d->qk_norm) {
          typedef EpiHeadNorm16<true> EN;   // k heads normalised (transformer.py:433-436), v as is
          SATB_PROPAGATE((linear<EN, 128, true>(d->tmaps, ce16, d->ce, Mr, d->ce, d->layers[i].w_kv, 2 * d->ce,
                                                 EN::Params{kv, 2 * d->ce, d->ce, 0, 1, nullptr, nullptr}, st)));
        } else {
          SATB_PROPAGATE((linear<E, 128, true>(d->tmaps, ce16, d->ce, Mr, d->ce, d->layers[i].w_kv, 2 * d->ce, E::Params{kv, 2 * d->ce, nullptr, 0}, st)));
        }
      }
    } else {
      typedef EpiStore16<false> E;
      SATB_PROPAGATE((linear<E, 128, false>(d->tmaps, in16, d->ct, Mr, d->ct, d->ce0_w, d->ce, E::Params{mid16, d->ce, nullptr, 1}, st)));
      SATB_PROPAGATE((linear<E, 128, false>(d->tmaps, mid16, d->ce, Mr, d->ce, d->ce2_w, d->ce, E::Params{ce16, d->ce, nullptr, 0}, st)));
      for (int i = 0; i < d->depth; ++i) {
        uint16_t* kv = d->ws_kv.as<uint16_t>() + static_cast<size_t>(i) * rows * 2 * d->ce;
        if (d->qk_norm) {
          typedef EpiHeadNorm16<false> EN;   // k heads normalised (transformer.py:433-436), v as is
          SATB_PROPAGATE((linear<EN, 128, false>(d->tmaps, ce16, d->ce, Mr, d->ce, d->layers[i].w_kv, 2 * d->ce,
                                                 EN::Params{kv, 2 * d->ce, d->ce, 0, 1, nullptr, nullptr}, st)));
        } else {
          SATB_PROPAGATE((linear<E, 128, false>(d->tmaps, ce16, d->ce, Mr, d->ce, d->layers[i].w_kv, 2 * d->ce, E::Params{kv, 2 * d->ce, nullptr, 0}, st)));
        }
      }
    }
  }
  return 0;
}

}  // extern "C"

// RAII helper: records a start/stop event pair around a kernel sequence when profiling is on
struct ProfScope {
  SatbDit* d; int cat; cudaStream_t st; cudaEvent_t a = nullptr, b = nullptr;
  ProfScope(SatbDit* d_, int cat_, cudaStream_t st_) : d(d_), cat(cat_), st(st_) {
    if (d->prof_on) { a = d->prof_event(); b = d->prof_event(); cudaEventRecord(a, st); }
  }
  ~ProfScope() {
    if (a) { cudaEventRecord(b, st); d->prof_recs.push_back({cat, a, b}); }
  }
};
enum { PROF_FF_IN = 0, PROF_FF_OUT, PROF_QKV, PROF_ATTN_SELF, PROF_ATTN_OUT, PROF_CROSS, PROF_LN, PROF_CONFORMER, PROF_NCAT };

// The token rows one forward runs on one handle: R rows (B items, doubled under CFG) of n tokens each, the first P of
// which are the prepended ones (global-conditioning and prepend-conditioning tokens).  The tokens are positions
// pos0 .. pos0 + n - 1 of the rotary and positional tables, which hold tab_len positions.  The single-device forward is
// the one shard that holds every token: P = d->P, n = tab_len = L + P, pos0 = 0.  A rank of a group forward holds a
// contiguous range of every item's tokens, with the prepended ones on rank 0 only.  half: -1 runs every row of the
// conditioning (2 B under CFG); 0 / 1 runs only the conditional / unconditional half of a CFG call (R = B rows, a rank
// of the CFG-split group forward), with conditioning rows half * B .. half * B + B - 1: their cross-attention K / V,
// prepend tokens (zeros on the unconditional half) and adaLN rows, exactly as the batched CFG forward uses them.
struct FwdShape {
  int B, R, L, P, n, pos0, tab_len;
  int half = -1;
};

// One forward as its stages: input (timestep embedding, project_in, prepended rows), then per block self_qkv, self_attn
// and block_rest (cross-attention, conformer branch, feed-forward), then output (project_out, CFG combine).  The
// single-device forward runs them in that order on one stream; the group forward interleaves the ranks' stages with the
// K/V gather between self_qkv and self_attn.
// FP8 = true: the QKV, cross-attention q and FF-in GEMMs read e4m3 LayerNorm rows (a8, one scale per row in a_scale)
// and the e4m3 weights; everything else runs as in fp16 mode (BF16 = false).
template <bool BF16, bool FP8 = false>
struct DitFwd {
  SatbDit* d;
  FwdShape s;
  cudaStream_t st;
  int D, C, H, M, Mc;   // Mc: rows running cross-attention (a prefix of the row space)
  int Rc, kv_row0;      // the Rc rows running cross-attention read conditioning K / V rows kv_row0 .. kv_row0 + Rc - 1
  int64_t ssg_ld;
  SmallWs sw;
  float* h;
  uint16_t* a16;
  uint8_t* a8;
  float* a_scale;
  const void* a_in;
  uint16_t *qkv, *att, *q16, *ff, *ain;
  BlockE4m3Out ff8;     // FP8 FF-out: the e4m3 FF intermediate and its block scales, in ws_ff in place of ff
  float* y;
  const float *cos_tab, *sin_tab, *pos_tab;

  DitFwd(SatbDit* d_, const FwdShape& s_, cudaStream_t st_) : d(d_), s(s_), st(st_) {
    D = d->D; C = d->C; H = d->H;
    M = s.R * s.n;
    // the conditional half holds the cross-attention rows of the batched CFG forward that fall in its B rows; the
    // unconditional half has some only with a negative prompt (Rc = 2 B)
    Rc = s.half < 0 ? d->Rc : s.half == 0 ? std::min(d->Rc, s.B) : (d->Rc == 2 * s.B ? s.B : 0);
    kv_row0 = s.half == 1 ? s.B : 0;
    Mc = Rc * s.n;
    ssg_ld = static_cast<int64_t>(d->depth) * 6 * D;
    sw = small_ws(d, 2 * d->B);
    h = d->ws_h.as<float>();
    a16 = d->ws_a16.as<uint16_t>();
    a8 = d->ws_a8.as<uint8_t>();
    a_scale = d->ws_ascale.as<float>();
    a_in = FP8 ? static_cast<const void*>(a8) : static_cast<const void*>(a16);
    qkv = d->ws_qkv.as<uint16_t>();
    att = d->ws_attn.as<uint16_t>();
    q16 = d->ws_q16.as<uint16_t>();
    ff = d->ws_ff.as<uint16_t>();
    uint8_t* ff_bytes = d->ws_ff.as<uint8_t>();
    ff8 = BlockE4m3Out{ff_bytes, reinterpret_cast<float*>(ff_bytes + static_cast<size_t>(M) * d->ffi), d->ffi};
    ain = d->ws_ain.as<uint16_t>();
    y = d->ws_y.as<float>();
    // rotary off (satb_dit_set_positions): null tables, which the QKV epilogues take as no rotation
    const float* rope = d->ws_rope.as<float>();
    cos_tab = d->rotary ? rope + static_cast<size_t>(s.pos0) * d->nf : nullptr;
    sin_tab = d->rotary ? rope + static_cast<size_t>(s.tab_len + s.pos0) * d->nf : nullptr;
    pos_tab = d->pos_type != 0 ? d->ws_pos.as<float>() + static_cast<size_t>(s.pos0) * D : nullptr;
  }

  // LayerNorm rows for one of the three FP8-capable GEMMs: e4m3 + row scales in FP8 mode, 16-bit otherwise
  int layernorm_in(const float* g, const float* b, int rows, const float* mod_scale, const float* mod_shift,
                   int64_t mod_ld, int n_items) {
    if (FP8) return launch_layernorm_fp8(h, g, b, a8, a_scale, rows, D, mod_scale, mod_shift, mod_ld, s.n, n_items, st);
    return launch_layernorm(h, g, b, a16, rows, D, mod_scale, mod_shift, mod_ld, s.n, n_items, BF16, st);
  }

  const float* ssg(int i) const { return d->adaln ? sw.ssg + static_cast<size_t>(i) * 6 * D : nullptr; }

  int input(const float* x, const float* t) {
    const int B = s.B;
    // timestep embedding (+ global embedding) -> conditioning token / adaLN vector  (dit.py:176-195)
    SATB_PROPAGATE(launch_fourier(t, d->ts_w, sw.fourier, B, d->F, st));
    // te_h = silu(W0 f + b0); tok = W2 te_h + b2 (+ global embed); in adaLN mode only silu(tok) is consumed
    SATB_PROPAGATE(launch_skinny_linear(sw.fourier, d->te0_w, d->te0_b, nullptr, sw.te_h, B, 2 * d->F, D, 1, st));
    SATB_PROPAGATE(launch_skinny_linear(sw.te_h, d->te2_w, d->te2_b, d->has_global ? sw.ge : nullptr, sw.tok, B, D, D,
                                        d->adaln ? 1 : 0, st));
    // latent -> token rows, project_in (with the 1x1 pre-conv folded), prepend token; a positional embedding is added
    // to every row, prepended ones included, in project_in's epilogue and by write_prepend.  K is Cin_p: the pad
    // columns of ain (zeroed by dit_pre) meet the zero columns of w_in16.
    const int Kin = d->Cin_p;
    SATB_PROPAGATE(launch_dit_pre(x, ain, s.R, B, d->Cin, Kin, s.L, s.P, BF16, st));
    if (pos_tab)
      SATB_PROPAGATE((linear<EpiStore32Pos, 256, BF16>(d->tmaps, ain, Kin, M, Kin, d->w_in16, D,
                                                       EpiStore32Pos::Params{h, D, nullptr, pos_tab, s.n}, st)));
    else
      SATB_PROPAGATE((linear<EpiStore32, 256, BF16>(d->tmaps, ain, Kin, M, Kin, d->w_in16, D, EpiStore32::Params{h, D, nullptr}, st)));
    if (d->P > 0) {
      if (s.P > 0)
        SATB_PROPAGATE(launch_write_prepend(sw.tok, d->Pp > 0 && s.half != 1 ? d->ws_prep.as<float>() : nullptr,
                                            pos_tab, h, s.R, B, s.n, D, d->Pp, st));
    } else {
      // adaLN: all layers' scale/shift/gate in one skinny GEMM (transformer.py:648-651,667)
      SATB_PROPAGATE(launch_skinny_linear(sw.tok, d->w_ssg, nullptr, nullptr, sw.ssg, B, D, d->depth * 6 * D, 0, st));
      SATB_PROPAGATE(launch_gate_sigmoid(sw.ssg, B, d->depth, D, st));
    }
    return 0;
  }

  // ---- self-attention, first half: LN -> QKV GEMM (+RoPE) into qkv
  int self_qkv(int i) {
    const LayerW& W = d->layers[i];
    const float* ssg_l = ssg(i);
    {
      ProfScope ps(d, PROF_LN, st);
      SATB_PROPAGATE(layernorm_in(W.pre_g, W.pre_b, M, ssg_l, ssg_l ? ssg_l + D : nullptr, ssg_ld, s.B));
    }
    ProfScope ps(d, PROF_QKV, st);
    const void* w = FP8 ? static_cast<const void*>(W.w8_qkv) : static_cast<const void*>(W.w_qkv);
    const Fp8Scales sc{a_scale, W.s_qkv};
    // FP8 self-attention: q and k leave the epilogue as e4m3 with their scales, v in 16 bits as always
    const AttnFp8Bufs b8 = d->attn_fp8 ? attn_fp8_bufs(d->ws_attn8.p, d->attn8_R, H, s.n, s.n) : AttnFp8Bufs{};
    const QkE4m3Out o8{b8.q8, b8.k8, b8.sq, b8.sk, H, attn_fp8_pad(s.n)};
    if (d->qk_norm) {
      typedef EpiHeadNorm16<BF16> E;   // q, k heads L2-normalised, then rotary
      typename E::Params ep{qkv, 3 * D, 2 * D, 2 * D, s.n, cos_tab, sin_tab};
      // FP8: BN 128 (the instance the cross q GEMM also runs; the BN 256 one spills a few registers)
      constexpr int kBn = FP8 ? 128 : 256;
      if (d->attn_fp8)
        SATB_PROPAGATE((linear<EpiHeadNormE4m3<BF16>, kBn, BF16, FP8>(d->tmaps, a_in, D, M, D, w, 3 * D,
                                                                       {ep, o8}, st, 1, sc)));
      else
        SATB_PROPAGATE((linear<E, kBn, BF16, FP8>(d->tmaps, a_in, D, M, D, w, 3 * D, ep, st, 1, sc)));
    } else {
      typedef EpiQkvRope<BF16> E;
      typename E::Params ep{qkv, 3 * D, 2 * D, s.n, d->dh, d->nf, cos_tab, sin_tab};
      if (d->attn_fp8)
        SATB_PROPAGATE((linear<EpiQkvRopeE4m3<BF16>, 256, BF16, FP8>(d->tmaps, a_in, D, M, D, w, 3 * D, {ep, o8}, st,
                                                                      1, sc)));
      else
        SATB_PROPAGATE((linear<E, 256, BF16, FP8>(d->tmaps, a_in, D, M, D, w, 3 * D, ep, st, 1, sc)));
    }
    return 0;
  }

  // ---- self-attention, second half: attention core -> out-proj (+residual).  kv null: the keys and values are the
  // k / v columns of this handle's own qkv (the single-device forward).  Else kv [R, Nk, 2D] holds every token's k | v
  // (the group forward's gathered buffer) and the local queries attend to all of them.
  int self_attn(int i, const uint16_t* kv, int Nk) {
    const LayerW& W = d->layers[i];
    const float* ssg_l = ssg(i);
    {
      ProfScope ps(d, PROF_ATTN_SELF, st);
      const int64_t qs = static_cast<int64_t>(s.n) * 3 * D;
      if (d->attn_fp8) {   // e4m3 operands in the workspace carved for attn8_R rows; the maps were made for them
        const AttnFp8Bufs b8 = attn_fp8_bufs(d->ws_attn8.p, d->attn8_R, H, s.n, s.n);
        SATB_PROPAGATE(launch_attention_fp8_vt(qkv + 2 * D, 3 * D, qs, b8, s.R, H, s.n, BF16, st));
        SATB_PROPAGATE(launch_attention_fp8(d->attn8_maps, b8, att, D, static_cast<int64_t>(s.n) * D, s.R, H, s.n,
                                            s.n, BF16, st));
      } else if (!kv) {
        const CUtensorMap* tm = nullptr;   // q, k and v are column ranges of one buffer: one map
        if (d->dh == 64) SATB_PROPAGATE(d->tmaps.get_a(qkv, 3 * D, s.n, s.R, 3 * D, qs, &tm));
        SATB_PROPAGATE(launch_attention_tc(qkv, qkv, qkv, att, 3 * D, 3 * D, 3 * D, D, qs, qs, qs,
                                           static_cast<int64_t>(s.n) * D, 3 * D, 3 * D, 3 * D, 0, D, 2 * D, s.R, H, H,
                                           s.n, s.n, d->dh, BF16, st, tm, tm, tm));
      } else {
        const int64_t kvs = static_cast<int64_t>(Nk) * 2 * D;
        const CUtensorMap *tq = nullptr, *tkv = nullptr;   // k and v are column ranges of one buffer: one map
        if (d->dh == 64) {
          SATB_PROPAGATE(d->tmaps.get_a(qkv, 3 * D, s.n, s.R, 3 * D, qs, &tq));
          SATB_PROPAGATE(d->tmaps.get_a(kv, 2 * D, Nk, s.R, 2 * D, kvs, &tkv));
        }
        SATB_PROPAGATE(launch_attention_tc(qkv, kv, kv, att, 3 * D, 2 * D, 2 * D, D, qs, kvs, kvs,
                                           static_cast<int64_t>(s.n) * D, 3 * D, 2 * D, 2 * D, 0, 0, D, s.R, H, H,
                                           s.n, Nk, d->dh, BF16, st, tq, tkv, tkv));
      }
    }
    ProfScope ps(d, PROF_ATTN_OUT, st);
    EpiResidual::Params ep{h, D, nullptr, ssg_l ? ssg_l + 2 * D : nullptr, s.n, static_cast<int>(ssg_ld), s.B};
    SATB_PROPAGATE((linear_auto<EpiResidual, BF16>(d->tmaps, att, D, M, D, W.w_o, D, ep, st)));
    return 0;
  }

  // ---- the rest of a block: cross-attention, conformer branch, feed-forward
  int block_rest(int i) {
    const LayerW& W = d->layers[i];
    const float* ssg_l = ssg(i);
    const int n = s.n;
    // ---- cross-attention on the rows that have a non-null context
    if (Mc > 0) {
      ProfScope ps(d, PROF_CROSS, st);
      const int Hkv = d->ce / d->dh;
      SATB_PROPAGATE(layernorm_in(W.ca_g, W.ca_b, Mc, nullptr, nullptr, 0, 1));
      const void* wq = FP8 ? static_cast<const void*>(W.w8_q) : static_cast<const void*>(W.w_q);
      const Fp8Scales sc{a_scale, W.s_q};
      if (d->qk_norm) {
        typedef EpiHeadNorm16<BF16> E;
        typename E::Params ep{q16, D, D, 0, n, nullptr, nullptr};
        if (FP8)   // BN 128 only, as for the QKV GEMM above
          SATB_PROPAGATE((linear<E, 128, BF16, FP8>(d->tmaps, a_in, D, Mc, D, wq, D, ep, st, 1, sc)));
        else
          SATB_PROPAGATE((linear_auto<E, BF16>(d->tmaps, a_in, D, Mc, D, wq, D, ep, st)));
      } else {
        typedef EpiStore16<BF16> E;
        typename E::Params ep{q16, D, nullptr, 0};
        SATB_PROPAGATE((linear_auto<E, BF16, FP8>(d->tmaps, a_in, D, Mc, D, wq, D, ep, st, sc)));
      }
      const uint16_t* kv = d->ws_kv.as<uint16_t>() +
                           (static_cast<size_t>(i) * d->Rc + kv_row0) * d->Mctx * 2 * d->ce;
      const int64_t kvs = static_cast<int64_t>(d->Mctx) * 2 * d->ce;
      const CUtensorMap *tq = nullptr, *tkv = nullptr;   // k and v are column ranges of one buffer: one map
      if (d->dh == 64) {
        SATB_PROPAGATE(d->tmaps.get_a(q16, D, n, Rc, D, static_cast<int64_t>(n) * D, &tq));
        SATB_PROPAGATE(d->tmaps.get_a(kv, 2 * d->ce, d->Mctx, Rc, 2 * d->ce, kvs, &tkv));
      }
      SATB_PROPAGATE(launch_attention_tc(q16, kv, kv, att, D, 2 * d->ce, 2 * d->ce, D, static_cast<int64_t>(n) * D,
                                         kvs, kvs, static_cast<int64_t>(n) * D, D, 2 * d->ce, 2 * d->ce, 0, 0,
                                         d->ce, Rc, H, Hkv, n, d->Mctx, d->dh, BF16, st, tq, tkv, tkv));
      EpiResidual::Params ep{h, D, nullptr, nullptr, n, 0, 1};
      SATB_PROPAGATE((linear_auto<EpiResidual, BF16>(d->tmaps, att, D, Mc, D, W.w_co, D, ep, st)));
    }
    // ---- conformer branch (transformer.py:576-591, added at :680-681 / :697-698 with no modulation or gate):
    // in_norm -> one GEMM for pointwise_conv + glu.proj (+bias, SwiGLU) -> depthwise conv + mid_norm + SiLU ->
    // pointwise_conv_2 (+residual).  16-bit operands in every mode (fp16 in the FP8 mode).  Its two [M, D] 16-bit
    // intermediates live in ws_ff, which is idle between cross-attention and the feed-forward.
    if (d->conformer) {
      ProfScope ps(d, PROF_CONFORMER, st);
      uint16_t* glu = ff;
      uint16_t* cv = ff + static_cast<size_t>(M) * D;
      SATB_PROPAGATE(launch_layernorm(h, W.cf_in_g, W.cf_in_b, a16, M, D, nullptr, nullptr, 0, n, 1, BF16, st));
      typedef EpiSwiglu<BF16> E;
      SATB_PROPAGATE((linear<E, 256, BF16>(d->tmaps, a16, D, M, D, W.cf_w1, 2 * D, typename E::Params{glu, D, W.cf_b1}, st)));
      SATB_PROPAGATE(launch_conformer_dwconv(glu, W.cf_dw, W.cf_mid_g, W.cf_mid_b, cv, s.R, n, D, BF16, st));
      EpiResidual::Params ep{h, D, nullptr, nullptr, n, 0, 1};
      SATB_PROPAGATE((linear_auto<EpiResidual, BF16>(d->tmaps, cv, D, M, D, W.cf_w2, D, ep, st)));
    }
    // ---- feed-forward: LN -> GEMM (+bias, SwiGLU) -> GEMM (+bias, +residual).  satb_dit_set_feedforward variants: a
    // plain FF-in is the GEMM (+bias, SiLU); a token convolution (FF-in and / or FF-out) the k-tap GEMM over each item.
    {
      ProfScope ps(d, PROF_LN, st);
      const float* mod_scale = ssg_l ? ssg_l + 3 * D : nullptr;
      const float* mod_shift = ssg_l ? ssg_l + 4 * D : nullptr;
      if (FP8 && d->ff_conv_in())   // the token convolution takes 16-bit (fp16) operands in every mode
        SATB_PROPAGATE(launch_layernorm(h, W.ff_g, W.ff_b, a16, M, D, mod_scale, mod_shift, ssg_ld, n, s.B, false, st));
      else
        SATB_PROPAGATE(layernorm_in(W.ff_g, W.ff_b, M, mod_scale, mod_shift, ssg_ld, s.B));
    }
    {
      ProfScope ps(d, PROF_FF_IN, st);
      const void* w = FP8 ? static_cast<const void*>(W.w8_ff1) : static_cast<const void*>(W.w_ff1);
      if (FP8 && d->ff_out_fp8) {   // the FF intermediate leaves the epilogue as e4m3 blocks (ff8) for FF-out
        const Fp8Scales sc{a_scale, W.s_ff1};
        if (d->ff_glu)
          SATB_PROPAGATE((linear<EpiSwigluE4m3, 256, false, true>(d->tmaps, a_in, D, M, D, w, 2 * d->ffi,
                                                                   EpiSwigluE4m3::Params{ff8, W.b_ff1}, st, 1, sc)));
        else
          SATB_PROPAGATE((linear_auto<EpiSiluE4m3, false, true>(d->tmaps, a_in, D, M, D, w, d->ffi,
                                                                 EpiSiluE4m3::Params{ff8, W.b_ff1}, st, sc)));
      } else if (d->ff_glu) {
        typedef EpiSwiglu<BF16> E;
        typename E::Params ep{ff, d->ffi, W.b_ff1};
        SATB_PROPAGATE((linear<E, 256, BF16, FP8>(d->tmaps, a_in, D, M, D, w, 2 * d->ffi, ep, st, 1,
                                                   Fp8Scales{a_scale, W.s_ff1})));
      } else if (d->ff_k == 0) {
        typedef EpiStore16<BF16> E;   // silu(x W^T + b), transformer.py:262-268
        typename E::Params ep{ff, d->ffi, W.b_ff1, 1};
        SATB_PROPAGATE((linear_auto<E, BF16, FP8>(d->tmaps, a_in, D, M, D, w, d->ffi, ep, st, Fp8Scales{a_scale, W.s_ff1})));
      } else {
        typedef EpiStore16<BF16> E;
        typename E::Params ep{ff, d->ffi, W.b_ff1, 1};
        SATB_PROPAGATE((token_conv<E, BF16>(d->tmaps, a16, n, s.R, n, D, W.w_ff1, d->ffi, d->ff_k, ep, st)));
      }
    }
    ProfScope ps(d, PROF_FF_OUT, st);
    EpiResidual::Params ep{h, D, W.b_ff2, ssg_l ? ssg_l + 5 * D : nullptr, n, static_cast<int>(ssg_ld), s.B};
    if (FP8 && d->ff_out_fp8)
      SATB_PROPAGATE((linear<BlockScaledA<EpiResidual>, 128, false, true>(d->tmaps, ff8.q, d->ffi, M, d->ffi, W.w8_ff2, D,
                                                                         ep, st, 1, Fp8Scales{ff8.scale, W.s_ff2})));
    else if (d->ff_k == 0)
      SATB_PROPAGATE((linear_auto<EpiResidual, BF16>(d->tmaps, ff, d->ffi, M, d->ffi, W.w_ff2, D, ep, st)));
    else
      SATB_PROPAGATE((token_conv<EpiResidual, BF16>(d->tmaps, ff, n, s.R, n, d->ffi, W.w_ff2, D, d->ff_k, ep, st)));
    return 0;
  }

  // project_out (with the 1x1 post-conv folded) reads a 16-bit copy of h; its N is C_p (zero weight rows past C)
  int project_out(float* hidden_out) {
    if (hidden_out)
      SATB_CHECK_CUDA(cudaMemcpyAsync(hidden_out, h, static_cast<size_t>(M) * D * 4, cudaMemcpyDeviceToDevice, st));
    const int Cp = d->C_p;
    SATB_PROPAGATE(launch_cast_rows(h, a16, nullptr, M, D, D, D, BF16, st));
    SATB_PROPAGATE((linear<EpiStore32, 64, BF16>(d->tmaps, a16, D, M, D, d->w_out16, Cp, EpiStore32::Params{y, Cp, nullptr}, st)));
    return 0;
  }

  // dit_post: the C real channels of each y row of the first B rows -> out, combined with the unconditional rows yu
  // (same shape and row pitch) under CFG; yu null: no CFG
  int combine(float* out, const float* yu, float cfg_scale, float scale_phi) {
    return launch_dit_post(y, yu, d->C_p, out, s.B, C, s.L, s.n, s.P, yu ? 1 : 0, cfg_scale, scale_phi, st);
  }

  int output(float* out, float cfg_scale, float scale_phi, float* hidden_out) {
    SATB_PROPAGATE(project_out(hidden_out));
    return combine(out, d->cfg_on ? y + static_cast<size_t>(s.B) * s.n * d->C_p : nullptr, cfg_scale, scale_phi);
  }
};

template <bool BF16, bool FP8 = false>
static int dit_forward_impl(SatbDit* d, const float* x, const float* t, float* out, int B, int L, float cfg_scale,
                            float scale_phi, cudaStream_t st, float* hidden_out) {
  const int N_seq = L + d->P;
  DitFwd<BF16, FP8> f(d, FwdShape{B, d->cfg_on ? 2 * B : B, L, d->P, N_seq, 0, N_seq}, st);
  SATB_PROPAGATE(f.input(x, t));
  for (int i = 0; i < d->depth; ++i) {
    SATB_PROPAGATE(f.self_qkv(i));
    SATB_PROPAGATE(f.self_attn(i, nullptr, N_seq));
    SATB_PROPAGATE(f.block_rest(i));
  }
  return f.output(out, cfg_scale, scale_phi, hidden_out);
}

static int dit_forward_dispatch(SatbDit* d, const float* x, const float* t, float* out, int B, int L, float cfg_scale,
                                float scale_phi, cudaStream_t st, float* hidden) {
  if (d->fp8) return dit_forward_impl<false, true>(d, x, t, out, B, L, cfg_scale, scale_phi, st, hidden);
  return d->bf16 ? dit_forward_impl<true>(d, x, t, out, B, L, cfg_scale, scale_phi, st, hidden)
                 : dit_forward_impl<false>(d, x, t, out, B, L, cfg_scale, scale_phi, st, hidden);
}

extern "C" {

// One denoiser call: x [B, C, L] fp32, t [B] fp32 -> out [B, C, L] fp32 (all device
// pointers, caller-owned).  Mirrors DiffusionTransformer.forward (models/dit.py:228-364)
// for the conditioning registered by satb_dit_prepare_cond.
int satb_dit_forward(SatbDit* d, const float* x, const float* t, float* out, int B, int L, float cfg_scale,
                     float scale_phi, void* stream_v) {
  SATB_REQUIRE(d && d->finalized, "weights not finalized");
  SATB_REQUIRE(B == d->B, "batch size differs from satb_dit_prepare_cond");
  const int R = d->cfg_on ? 2 * B : B;
  if (needs_reserve(d, R, L)) SATB_PROPAGATE(satb_dit_reserve(d, R, L));
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  return dit_forward_dispatch(d, x, t, out, B, L, cfg_scale, scale_phi, st, nullptr);
}

// Per-category kernel timing with CUDA events on the launching stream (bench.py roofline):
// categories 0 ff_in GEMM, 1 ff_out GEMM, 2 qkv GEMM, 3 self-attention core, 4 attn out GEMM,
// 5 cross-attention (LN + q GEMM + core + out GEMM), 6 LayerNorm, 7 conformer branch (all four of its launches).
int satb_dit_profile(SatbDit* d, int enable) {
  SATB_REQUIRE(d, "null handle");
  d->prof_on = enable != 0;
  return 0;
}
// Synchronises, sums the recorded intervals per category into ms[8] / count[8], and clears them.
int satb_dit_profile_read(SatbDit* d, float* ms, int* count) {
  SATB_REQUIRE(d && ms && count, "null argument");
  for (int i = 0; i < PROF_NCAT; ++i) { ms[i] = 0.f; count[i] = 0; }
  for (auto& r : d->prof_recs) {
    SATB_CHECK_CUDA(cudaEventSynchronize(r.b));
    float t = 0.f;
    SATB_CHECK_CUDA(cudaEventElapsedTime(&t, r.a, r.b));
    ms[r.cat] += t;
    count[r.cat] += 1;
    d->prof_pool.push_back(r.a);
    d->prof_pool.push_back(r.b);
  }
  d->prof_recs.clear();
  return 0;
}

// Debug/test variant that also returns the residual stream after the last block
// ([R * (L + P), D] fp32) for comparison with the reference's hidden_states.
int satb_dit_forward_debug(SatbDit* d, const float* x, const float* t, float* out, float* hidden, int B, int L,
                           float cfg_scale, float scale_phi, void* stream_v) {
  SATB_REQUIRE(d && d->finalized, "weights not finalized");
  SATB_REQUIRE(B == d->B, "batch size differs from satb_dit_prepare_cond");
  const int R = d->cfg_on ? 2 * B : B;
  if (needs_reserve(d, R, L)) SATB_PROPAGATE(satb_dit_reserve(d, R, L));
  cudaStream_t st = static_cast<cudaStream_t>(stream_v);
  return dit_forward_dispatch(d, x, t, out, B, L, cfg_scale, scale_phi, st, hidden);
}

// ---- Token-sharded forward: one process drives `world` ranks, each a finalized handle with a full copy of the weights
// on its device (several ranks may share a device).  Rank r holds tokens token_begin[r] .. token_begin[r + 1] - 1 of
// every item, the prepended ones on rank 0.  Every stage works per token except self-attention, which needs every
// token's k and v: once per layer each rank gathers them into its kv buffer [R, N, 2D] and attends its own queries
// against all N keys.
int satb_dit_group_plan(int world, int n_prepend, int L, int* token_begin) {
  SATB_REQUIRE(token_begin, "null argument");
  SATB_REQUIRE(world >= 1 && world <= kKvGatherMaxRanks, "world must be 1 .. 8");
  SATB_REQUIRE(n_prepend >= 0 && L >= 1, "need n_prepend >= 0 and L >= 1");
  const int N = n_prepend + L;
  if (world > N) {
    set_last_error("world " + std::to_string(world) + " exceeds the " + std::to_string(N) +
                   " tokens of an item: every rank needs at least one token");
    return -1;
  }
  // as even as possible in units of `unit` tokens, rank 0 taking at least the prepended tokens
  auto split = [&](int unit) -> int {
    const int nu = ceil_div(N, unit);   // units; the last may be partial
    const int p0 = ceil_div(n_prepend, unit);
    for (int r = 0; r <= world; ++r) token_begin[r] = static_cast<int>(static_cast<long long>(r) * nu / world) * unit;
    if (token_begin[1] < n_prepend) {   // rank 0 takes the prepended units, the others share the rest evenly
      if (nu - p0 < world - 1) return -1;
      for (int r = 1; r <= world; ++r)
        token_begin[r] = (p0 + static_cast<int>(static_cast<long long>(r - 1) * (nu - p0) / (world - 1))) * unit;
    }
    token_begin[world] = N;
    return 0;
  };
  // GEMM row tiles and attention query tiles are 128 rows (kBlockM): whole tiles per rank when every rank can have one
  if (N >= kBlockM * world && split(kBlockM) == 0) return 0;
  if (split(1) == 0) return 0;
  set_last_error("the " + std::to_string(n_prepend) + " prepended tokens leave fewer than one token for each of the other " +
                 std::to_string(world - 1) + " ranks");
  return -1;
}

}  // extern "C"

// The whole-tensor arguments of satb_dit_group_graph_forward, on the home device (rank 0's)
struct GraphKey {
  const float *x = nullptr, *t = nullptr;
  float* out = nullptr;
  int B = 0, L = 0;
  float cfg_scale = 0.f, scale_phi = 0.f;
  bool operator==(const GraphKey& o) const {
    return x == o.x && t == o.t && out == o.out && B == o.B && L == o.L && cfg_scale == o.cfg_scale &&
           scale_phi == o.scale_phi;
  }
};

struct SatbDitGroup {
  int world = 0;                             // ranks of one row (the token split)
  // satb_dit_group_create_cfg: two rows of `world` ranks, row 0 (ranks 0 .. world - 1) running the conditional half
  // of each CFG call and row 1 (ranks world .. 2 world - 1) the unconditional half; a call without CFG runs row 0 only
  bool cfg = false;
  int ranks = 0;                             // handles: world, or 2 world for a CFG group
  std::vector<SatbDit*> h;
  std::vector<int> dev;
  std::vector<DevBuf> kv;                    // per rank, on its device: [R, N, 2D] 16-bit
  // Per rank, recorded by eager calls only: its QKV GEMM done / its gather done (the last enqueued) / its last work
  // of the call done / (CFG group, row 0) its combine done.  A captured graph records its own events (gev_*): an event
  // last recorded inside a capture cannot be waited on outside it.  ev_y / gev_y (CFG group, row 1): its project_out
  // done.
  std::vector<cudaEvent_t> ev_qkv, ev_read, ev_done, ev_y, ev_comb;
  std::vector<cudaEvent_t> gev_qkv, gev_read, gev_join, gev_y;
  std::vector<int> res_R, res_L, res_P;      // per rank: the shape its workspace was last reserved for
  // satb_dit_group_graph_forward: the instantiated graph, what it was captured for, and the fixed per-rank slices of
  // x, t and out it reads and writes (on each rank's device)
  cudaGraphExec_t exec = nullptr;
  GraphKey key;
  std::vector<unsigned long long> gens;      // every handle's gen at capture
  unsigned long long graph_launches = 0;     // kernel launches in the graph
  long long captures = 0, replays = 0;
  std::vector<DevBuf> gx, gt, gout;
  cudaEvent_t ev_fork = nullptr;             // home device: the capture's fork
  cudaEvent_t ev_graph = nullptr;            // home device: recorded after each graph launch (and before a warm-up)
  cudaStream_t cap = nullptr;                // home device: the capture stream
};

// Every per-rank event vector of a group.
static std::vector<std::vector<cudaEvent_t>*> group_events(SatbDitGroup* g) {
  return {&g->ev_qkv, &g->ev_read, &g->ev_done, &g->ev_y, &g->ev_comb, &g->gev_qkv, &g->gev_read, &g->gev_join,
          &g->gev_y};
}

// The option a group forward cannot run on this handle, or null.  Token convolutions (conformer blocks, use_conv
// feed-forwards) need the neighbouring ranks' tokens (halos); FP8 self-attention's v channel scales span all of an
// item's tokens.
static const char* group_refusal(const SatbDit* d) {
  if (d->conformer) return "conformer blocks are not supported by the token-sharded forward (their depthwise "
                           "convolution needs the neighbouring ranks' tokens)";
  if (d->ff_k > 0) return "use_conv feed-forwards are not supported by the token-sharded forward (their token "
                          "convolution needs the neighbouring ranks' tokens)";
  if (d->attn_fp8) return "attention_dtype \"fp8\" is not supported by the token-sharded forward (its v channel scales "
                          "span all of an item's tokens)";
  return nullptr;
}

static bool same_model(const SatbDit* a, const SatbDit* b) {
  return std::memcmp(&a->cfg, &b->cfg, sizeof(SatbDitConfig)) == 0 && a->ff_inner == b->ff_inner &&
         a->ff_glu == b->ff_glu && a->ff_bias == b->ff_bias && a->ff_k == b->ff_k && a->rotary == b->rotary &&
         a->pos_type == b->pos_type && a->abs_max_len == b->abs_max_len && a->conformer == b->conformer &&
         a->attn_fp8 == b->attn_fp8 && a->ff_out_fp8 == b->ff_out_fp8;
}

static void group_drop_graph(SatbDitGroup* g) {
  if (g->exec) cudaGraphExecDestroy(g->exec);   // a launch still in flight completes; the memory is freed after it
  g->exec = nullptr;
  g->key = GraphKey();
  g->gens.clear();
}

static void group_release(SatbDitGroup* g) {
  int cur = 0;
  cudaGetDevice(&cur);
  group_drop_graph(g);
  for (int r = 0; r < g->ranks; ++r) {
    cudaSetDevice(g->dev[r]);
    for (std::vector<DevBuf>* b : {&g->kv, &g->gx, &g->gt, &g->gout})
      if (r < static_cast<int>(b->size())) (*b)[r].release();
    for (std::vector<cudaEvent_t>* e : group_events(g))
      if (r < static_cast<int>(e->size()) && (*e)[r]) cudaEventDestroy((*e)[r]);
  }
  if (g->ranks > 0) {
    cudaSetDevice(g->dev[0]);
    if (g->ev_fork) cudaEventDestroy(g->ev_fork);
    if (g->ev_graph) cudaEventDestroy(g->ev_graph);
    if (g->cap) cudaStreamDestroy(g->cap);
  }
  cudaSetDevice(cur);
}

// Sets each rank's device in turn and restores the caller's on scope exit.
struct DeviceRestore {
  int cur = 0;
  DeviceRestore() { cudaGetDevice(&cur); }
  ~DeviceRestore() { cudaSetDevice(cur); }
};

// The group forward, layer-major across the ranks.  Hazards between ranks, ordered with events only:
//   RAW: rank r's gather of layer l reads every rank's qkv, so it waits for every rank's QKV GEMM of layer l (ev_qkv).
//   WAR: rank s's QKV GEMM of layer l + 1 overwrites its qkv, so it waits until every rank has finished gathering
//        layer l (ev_read).  The first layer of a call waits likewise for the last gathers of the previous call.
// Within a rank, its own stream orders everything else (its kv buffer is rewritten only after its own attention of the
// previous layer, on the same stream).
// split (a CFG call on a CFG group): both rows run, each on its half of the rows, and the pairs above hold within a
// row (the ranks of a row gather only each other's K / V).  After the last block, row-0 rank j combines its y with
// row-1 rank j's y (same tokens), read through a peer pointer, and two more pairs order that:
//   RAW: row-0 rank j's combine waits for row-1 rank j's project_out (ev_y).
//   WAR: row-1 rank j's project_out of the next call waits for row-0 rank j's combine of this call (ev_comb).
// in_graph: the stages are being captured.  The same pairs are recorded on the graph's own events (they become graph
// edges), and the waits on the previous call (the first layer's WAR, the combine's WAR) are skipped: the previous
// call was recorded outside the capture, and a graph launch runs only after everything before it on its stream
// (satb_dit_group_graph_forward).
template <bool BF16, bool FP8>
static int group_forward_impl(SatbDitGroup* g, const float* const* x, const float* const* t, float* const* out, int B,
                              int L, float cfg_scale, float scale_phi, cudaStream_t const* st, const int* tb,
                              bool split, bool in_graph) {
  const int W = g->world, NR = split ? 2 * W : W, P = g->h[0]->P, N = L + P;
  const std::vector<cudaEvent_t>& ev_qkv = in_graph ? g->gev_qkv : g->ev_qkv;
  const std::vector<cudaEvent_t>& ev_read = in_graph ? g->gev_read : g->ev_read;
  const std::vector<cudaEvent_t>& ev_y = in_graph ? g->gev_y : g->ev_y;
  const int R = split ? B : g->h[0]->cfg_on ? 2 * B : B;
  std::vector<DitFwd<BF16, FP8>> f;
  f.reserve(NR);
  std::vector<const void*> qkv(NR);
  for (int r = 0; r < NR; ++r) {
    const int j = r % W, p = j == 0 ? P : 0, n = tb[j + 1] - tb[j];
    FwdShape s{B, R, n - p, p, n, tb[j], N};
    s.half = split ? r / W : -1;
    f.emplace_back(g->h[r], s, st[r]);
    qkv[r] = g->h[r]->ws_qkv.p;
  }
  for (int r = 0; r < NR; ++r) {
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
    SATB_PROPAGATE(f[r].input(x[r], t[r]));
  }
  const int D = g->h[0]->D;
  for (int i = 0; i < g->h[0]->depth; ++i) {
    for (int r = 0; r < NR; ++r) {
      const int row0 = r / W * W;   // the first rank of r's row
      SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
      if (!(in_graph && i == 0))
        for (int s = row0; s < row0 + W; ++s) SATB_CHECK_CUDA(cudaStreamWaitEvent(st[r], ev_read[s], 0));   // WAR
      SATB_PROPAGATE(f[r].self_qkv(i));
      SATB_CHECK_CUDA(cudaEventRecord(ev_qkv[r], st[r]));
    }
    for (int r = 0; r < NR; ++r) {
      const int row0 = r / W * W;
      SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
      for (int s = row0; s < row0 + W; ++s) SATB_CHECK_CUDA(cudaStreamWaitEvent(st[r], ev_qkv[s], 0));    // RAW
      SATB_PROPAGATE(launch_kv_gather(qkv.data() + row0, tb, W, g->kv[r].p, R, D, st[r]));
      SATB_CHECK_CUDA(cudaEventRecord(ev_read[r], st[r]));
      SATB_PROPAGATE(f[r].self_attn(i, g->kv[r].as<uint16_t>(), N));
      SATB_PROPAGATE(f[r].block_rest(i));
    }
  }
  if (!split) {
    for (int r = 0; r < W; ++r) {
      SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
      SATB_PROPAGATE(f[r].output(out[r], cfg_scale, scale_phi, nullptr));
    }
    return 0;
  }
  for (int r = W; r < NR; ++r) {   // the unconditional half: project_out only
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
    if (!in_graph) SATB_CHECK_CUDA(cudaStreamWaitEvent(st[r], g->ev_comb[r - W], 0));   // WAR
    SATB_PROPAGATE(f[r].project_out(nullptr));
    SATB_CHECK_CUDA(cudaEventRecord(ev_y[r], st[r]));
  }
  for (int r = 0; r < W; ++r) {    // the conditional half: project_out, then the combine
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
    SATB_PROPAGATE(f[r].project_out(nullptr));
    SATB_CHECK_CUDA(cudaStreamWaitEvent(st[r], ev_y[W + r], 0));                          // RAW
    SATB_PROPAGATE(f[r].combine(out[r], g->h[W + r]->ws_y.as<float>(), cfg_scale, scale_phi));
    if (!in_graph) SATB_CHECK_CUDA(cudaEventRecord(g->ev_comb[r], st[r]));
  }
  return 0;
}

// Checks the handles of one group (satb_dit_group_create: one row; satb_dit_group_create_cfg: two rows) and makes it.
// refuse_halo: refuse the options whose token convolutions or V scales span the token split (-5).
static int group_create(SatbDit* const* handles, const int* devices, int world, bool cfg, bool refuse_halo,
                        SatbDitGroup** out) {
  const int ranks = cfg ? 2 * world : world;
  for (int r = 0; r < ranks; ++r) {
    SATB_REQUIRE(handles[r], "null handle");
    const char* why = refuse_halo ? group_refusal(handles[r]) : nullptr;
    if (why) {
      set_last_error(why);
      return -5;
    }
    if (!same_model(handles[0], handles[r])) {
      set_last_error("rank " + std::to_string(r) + "'s handle has another config or model option than rank 0's");
      return -1;
    }
    for (int s = 0; s < r; ++s)
      SATB_REQUIRE(handles[s] != handles[r], "every rank needs its own handle (its own workspace)");
  }
  for (int r = 0; r < ranks; ++r) SATB_REQUIRE(handles[r]->finalized, "weights not finalized");
  DeviceRestore restore;
  int n_dev = 0;
  SATB_CHECK_CUDA(cudaGetDeviceCount(&n_dev));
  for (int r = 0; r < ranks; ++r) SATB_REQUIRE(devices[r] >= 0 && devices[r] < n_dev, "no such device");
  // every rank reads every other rank's qkv: peer access between each pair of distinct devices (in a CFG group also
  // between the rows: the combine reads the other half's y, the graph copies x and t from rank 0's device)
  for (int r = 0; r < ranks; ++r)
    for (int s = 0; s < ranks; ++s) {
      if (devices[r] == devices[s]) continue;
      int ok = 0;
      SATB_CHECK_CUDA(cudaDeviceCanAccessPeer(&ok, devices[r], devices[s]));
      if (!ok) {
        set_last_error("device " + std::to_string(devices[r]) + " cannot access device " + std::to_string(devices[s]) +
                       " peer to peer: the token-sharded forward reads every rank's K/V over peer links");
        return -1;
      }
    }
  for (int r = 0; r < ranks; ++r) {
    SATB_CHECK_CUDA(cudaSetDevice(devices[r]));
    for (int s = 0; s < ranks; ++s) {
      if (devices[r] == devices[s]) continue;
      const cudaError_t e = cudaDeviceEnablePeerAccess(devices[s], 0);   // this process's context only
      if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();
      } else {
        SATB_CHECK_CUDA(e);
      }
    }
  }
  SatbDitGroup* g = new SatbDitGroup();
  g->world = world;
  g->cfg = cfg;
  g->ranks = ranks;
  g->h.assign(handles, handles + ranks);
  g->dev.assign(devices, devices + ranks);
  g->kv.resize(ranks);
  g->gx.resize(ranks);
  g->gt.resize(ranks);
  g->gout.resize(ranks);
  g->res_R.assign(ranks, 0);
  g->res_L.assign(ranks, 0);
  g->res_P.assign(ranks, -1);
  for (std::vector<cudaEvent_t>* ev : group_events(g)) ev->assign(ranks, nullptr);
  cudaError_t e = cudaSuccess;
  for (int r = 0; r < ranks && e == cudaSuccess; ++r) {
    e = cudaSetDevice(devices[r]);
    for (std::vector<cudaEvent_t>* ev : group_events(g))
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&(*ev)[r], cudaEventDisableTiming);
  }
  if (e == cudaSuccess) e = cudaSetDevice(devices[0]);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_graph, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&g->cap, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    group_release(g);
    delete g;
    set_last_error(std::string(cfg ? "satb_dit_group_create_cfg: " : "satb_dit_group_create: ") +
                   cudaGetErrorString(e));
    return -2;
  }
  *out = g;
  return 0;
}

extern "C" {

int satb_dit_group_create(SatbDit* const* handles, const int* devices, int world, SatbDitGroup** out) {
  SATB_REQUIRE(handles && devices && out, "null argument");
  SATB_REQUIRE(world >= 1 && world <= kKvGatherMaxRanks, "world must be 1 .. 8");
  return group_create(handles, devices, world, false, true, out);
}

int satb_dit_group_create_cfg(SatbDit* const* handles, const int* devices, int world, SatbDitGroup** out) {
  SATB_REQUIRE(handles && devices && out, "null argument");
  SATB_REQUIRE(world >= 1 && world <= kKvGatherMaxRanks, "world must be 1 .. 8");
  // a row of one rank holds every token: its token convolutions and FP8 V scales see the whole item
  return group_create(handles, devices, world, true, world > 1, out);
}

void satb_dit_group_destroy(SatbDitGroup* g) {
  if (!g) return;
  group_release(g);
  delete g;
}

}  // extern "C"

// Checks one call's arguments against the conditioning of every rank it runs and fills the token split tb.  split: a
// CFG call on a CFG group (both rows run); otherwise only row 0 runs.
static int group_check(SatbDitGroup* g, int B, int L, int* tb, bool* split) {
  const int W = g->world;
  SatbDit* d0 = g->h[0];
  *split = g->cfg && d0->cfg_on;
  for (int r = 0; r < (*split ? 2 * W : W); ++r) {
    const SatbDit* d = g->h[r];
    SATB_REQUIRE(d->finalized, "weights not finalized");
    SATB_REQUIRE(B == d->B, "batch size differs from satb_dit_prepare_cond");
    SATB_REQUIRE(d->cfg_on == d0->cfg_on && d->P == d0->P && d->Rc == d0->Rc && d->Mctx == d0->Mctx &&
                     d->has_global == d0->has_global,
                 "every rank needs the same conditioning (satb_dit_set_prepend_cond / satb_dit_prepare_cond)");
  }
  SATB_REQUIRE(L >= 1, "bad shape");
  return satb_dit_group_plan(W, d0->P, L, tb);
}

// Grows the workspace and kv buffer of every rank the call runs to its shape when they do not fit (synchronous when
// it allocates).  A rank of a split call runs B rows (its half), else R = 2 B under CFG.
static int group_reserve(SatbDitGroup* g, int B, int L, const int* tb, bool split) {
  SatbDit* d0 = g->h[0];
  const int N = L + d0->P, R = !split && d0->cfg_on ? 2 * B : B;
  for (int r = 0; r < (split ? 2 * g->world : g->world); ++r) {
    SatbDit* d = g->h[r];
    const int j = r % g->world;
    // (the FP8 attention operands are carved for the rows of the last reserve, which may be fewer than res_R)
    const bool fresh = R <= g->res_R[r] && L == g->res_L[r] && d0->P == g->res_P[r] && (!d->attn_fp8 || R <= d->attn8_R);
    // res_R 0: no single-device forward has reserved since; and the table check of needs_reserve (a reload of the
    // weights marks the position table stale)
    if (!(fresh && d->res_R == 0 && !(d->pos_type != 0 && d->pos_len != N))) {
      SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
      SATB_PROPAGATE(reserve_rows(d, R, tb[j + 1] - tb[j], N));
      SATB_PROPAGATE(g->kv[r].ensure(static_cast<size_t>(R) * N * 2 * d->D * 2));
      d->res_R = 0;   // the workspace no longer has the single-device forward's shape: its next call reserves again
    }
    g->res_R[r] = std::max(g->res_R[r], R);
    g->res_L[r] = L;
    g->res_P[r] = d0->P;
  }
  return 0;
}

// The whole tensors of satb_dit_group_graph_forward: each rank's slice is copied into (x, t) and out of (out) the
// group's fixed per-rank buffers on that rank's stream, over peer access between devices.
struct GroupIo {
  const float *x, *t;
  float* out;
};

// Rank r's latent tokens lo .. lo + n - 1 of every item (rank 0 holds the prepended ones besides).
static void rank_latents(const int* tb, int P, int r, int* lo, int* n) {
  *lo = std::max(tb[r] - P, 0);
  *n = tb[r + 1] - P - *lo;
}

// One group forward on the streams of the ranks it runs (both rows of a split call, else row 0): every rank stream
// first waits for the last graph launch (ev_graph), then the optional input slices, the stages, and the optional
// output slices (row 0's).  Eager calls record each rank's ev_done last.
static int group_run(SatbDitGroup* g, const float* const* x, const float* const* t, float* const* out, int B, int L,
                     float cfg_scale, float scale_phi, cudaStream_t const* st, const int* tb, bool split, bool in_graph,
                     const GroupIo* io) {
  const int W = g->world, NR = split ? 2 * W : W;
  SatbDit* d0 = g->h[0];
  const int P = d0->P, Cin = d0->Cin, C = d0->C;
  for (int r = 0; r < NR; ++r) {
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
    if (!in_graph) SATB_CHECK_CUDA(cudaStreamWaitEvent(st[r], g->ev_graph, 0));
    if (!io) continue;
    int lo, n;
    rank_latents(tb, P, r % W, &lo, &n);
    if (n > 0)
      SATB_CHECK_CUDA(cudaMemcpy2DAsync(g->gx[r].p, static_cast<size_t>(n) * 4, io->x + lo, static_cast<size_t>(L) * 4,
                                        static_cast<size_t>(n) * 4, static_cast<size_t>(B) * Cin, cudaMemcpyDefault,
                                        st[r]));
    SATB_CHECK_CUDA(cudaMemcpyAsync(g->gt[r].p, io->t, static_cast<size_t>(B) * 4, cudaMemcpyDefault, st[r]));
  }
  int rc;
  if (d0->fp8)
    rc = group_forward_impl<false, true>(g, x, t, out, B, L, cfg_scale, scale_phi, st, tb, split, in_graph);
  else if (d0->bf16)
    rc = group_forward_impl<true, false>(g, x, t, out, B, L, cfg_scale, scale_phi, st, tb, split, in_graph);
  else
    rc = group_forward_impl<false, false>(g, x, t, out, B, L, cfg_scale, scale_phi, st, tb, split, in_graph);
  SATB_PROPAGATE(rc);
  for (int r = 0; r < NR; ++r) {
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
    int lo, n;
    rank_latents(tb, P, r % W, &lo, &n);
    if (io && n > 0 && r < W)
      SATB_CHECK_CUDA(cudaMemcpy2DAsync(io->out + lo, static_cast<size_t>(L) * 4, g->gout[r].p,
                                        static_cast<size_t>(n) * 4, static_cast<size_t>(n) * 4,
                                        static_cast<size_t>(B) * C, cudaMemcpyDefault, st[r]));
    if (!in_graph) SATB_CHECK_CUDA(cudaEventRecord(g->ev_done[r], st[r]));
  }
  return 0;
}

// Enqueues the group forward on g->cap while it captures, ending the capture on every path.  The rank streams fork
// from g->cap and join it again, so the graph holds every rank's nodes on its own device.
static int group_capture(SatbDitGroup* g, const float* const* x, const float* const* t, float* const* out, int B,
                         int L, float cfg_scale, float scale_phi, cudaStream_t const* st, const int* tb, bool split,
                         const GroupIo& io, cudaGraph_t* graph, unsigned long long* launches) {
  const int NR = split ? 2 * g->world : g->world;
  SATB_CHECK_CUDA(cudaSetDevice(g->dev[0]));
  SATB_CHECK_CUDA(cudaStreamBeginCapture(g->cap, cudaStreamCaptureModeThreadLocal));
  const unsigned long long n0 = g_launch_count;
  int rc = 0;
  cudaError_t e = cudaEventRecord(g->ev_fork, g->cap);
  for (int r = 0; r < NR && e == cudaSuccess; ++r) {
    e = cudaSetDevice(g->dev[r]);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st[r], g->ev_fork, 0);
  }
  if (e == cudaSuccess) {
    rc = group_run(g, x, t, out, B, L, cfg_scale, scale_phi, st, tb, split, true, &io);
    for (int r = 0; r < NR && rc == 0 && e == cudaSuccess; ++r) {
      e = cudaSetDevice(g->dev[r]);
      if (e == cudaSuccess) e = cudaEventRecord(g->gev_join[r], st[r]);
      if (e == cudaSuccess) e = cudaSetDevice(g->dev[0]);
      if (e == cudaSuccess) e = cudaStreamWaitEvent(g->cap, g->gev_join[r], 0);
    }
  }
  *launches = g_launch_count - n0;
  const std::string inner = rc != 0 ? satb_last_error() : "";
  cudaSetDevice(g->dev[0]);
  const cudaError_t e_end = cudaStreamEndCapture(g->cap, graph);   // also ends an invalidated capture
  if (rc != 0 || e != cudaSuccess || e_end != cudaSuccess) {
    if (e_end == cudaSuccess && *graph) cudaGraphDestroy(*graph);
    *graph = nullptr;
    cudaGetLastError();
    if (rc != 0) {
      set_last_error("capturing the group forward: " + inner);
      return rc;
    }
    set_last_error(std::string("capturing the group forward: ") + cudaGetErrorString(e != cudaSuccess ? e : e_end));
    return -3;
  }
  return 0;
}

extern "C" {

int satb_dit_group_forward(SatbDitGroup* g, const float* const* x, const float* const* t, float* const* out, int B,
                           int L, float cfg_scale, float scale_phi, void* const* streams) {
  SATB_REQUIRE(g && x && t && out && streams, "null argument");
  int tb[kKvGatherMaxRanks + 1];
  bool split = false;
  SATB_PROPAGATE(group_check(g, B, L, tb, &split));
  const int W = g->world, NR = split ? 2 * W : W;
  for (int r = 0; r < NR; ++r) SATB_REQUIRE(x[r] && t[r] && (r >= W || out[r]), "null argument");
  DeviceRestore restore;
  SATB_PROPAGATE(group_reserve(g, B, L, tb, split));
  cudaStream_t st[2 * kKvGatherMaxRanks];
  for (int r = 0; r < NR; ++r) st[r] = static_cast<cudaStream_t>(streams[r]);
  return group_run(g, x, t, out, B, L, cfg_scale, scale_phi, st, tb, split, false, nullptr);
}

// Ordering against eager calls, which may run on distinct devices and alternate with graph launches:
//   * before each launch, home_stream waits for every rank's ev_done, the end of its last eager call (its output
//     stage, after which that rank touches no buffer of the call), so the graph never overwrites a workspace, a qkv
//     or a kv buffer an eager call still reads;
//   * after each launch, ev_graph is recorded on home_stream, and every eager call makes each rank stream wait for
//     it before its first launch (group_run), so an eager call never overwrites what the graph still reads.
// The graph's own cross-rank hazards are the eager path's event pairs, captured as edges; successive launches on one
// stream run one after the other, which stands for the first layer's WAR waits (and, in a CFG group, the combine's).
// With virtual ranks everything is on one device, so these waits are ordinary same-device waits there; between devices
// they are the same events.  In a CFG group both rows count as ranks here.
int satb_dit_group_graph_forward(SatbDitGroup* g, const float* x, const float* t, float* out, int B, int L,
                                 float cfg_scale, float scale_phi, void* const* rank_streams, void* home_stream) {
  SATB_REQUIRE(g && x && t && out && rank_streams, "null argument");
  const int W = g->world, NH = g->ranks;
  for (int r = 0; r < NH; ++r)
    SATB_REQUIRE(rank_streams[r], "rank streams must be created streams (the legacy default stream cannot be captured)");
  for (int r = 0; r < NH; ++r)
    SATB_REQUIRE(!g->h[r]->prof_on, "satb_dit_group_graph_forward: profiling (satb_dit_profile) is on for a rank; "
                                    "its event timing cannot be captured");
  int tb[kKvGatherMaxRanks + 1];
  bool split = false;
  SATB_PROPAGATE(group_check(g, B, L, tb, &split));
  const int NR = split ? 2 * W : W;
  DeviceRestore restore;
  cudaStream_t st[2 * kKvGatherMaxRanks];
  for (int r = 0; r < NH; ++r) st[r] = static_cast<cudaStream_t>(rank_streams[r]);
  cudaStream_t home = static_cast<cudaStream_t>(home_stream);
  GraphKey key;
  key.x = x; key.t = t; key.out = out; key.B = B; key.L = L; key.cfg_scale = cfg_scale; key.scale_phi = scale_phi;
  bool stale = !g->exec || !(key == g->key) || static_cast<int>(g->gens.size()) != NH;
  for (int r = 0; r < NH && !stale; ++r) stale = g->gens[r] != g->h[r]->gen;
  if (stale) {
    group_drop_graph(g);
    SatbDit* d0 = g->h[0];
    const GroupIo io{x, t, out};
    const float* xs[2 * kKvGatherMaxRanks];
    const float* ts[2 * kKvGatherMaxRanks];
    float* os[2 * kKvGatherMaxRanks] = {};
    for (int r = 0; r < NR; ++r) {   // the fixed per-rank slices (at least 256 bytes: a rank may hold no latent token)
      int lo, n;
      rank_latents(tb, d0->P, r % W, &lo, &n);
      SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
      SATB_PROPAGATE(g->gx[r].ensure(std::max<size_t>(static_cast<size_t>(B) * d0->Cin * n * 4, 256)));
      SATB_PROPAGATE(g->gt[r].ensure(std::max<size_t>(static_cast<size_t>(B) * 4, 256)));
      xs[r] = g->gx[r].as<float>();
      ts[r] = g->gt[r].as<float>();
      if (r >= W) continue;          // only row 0 writes output
      SATB_PROPAGATE(g->gout[r].ensure(std::max<size_t>(static_cast<size_t>(B) * d0->C * n * 4, 256)));
      os[r] = g->gout[r].as<float>();
    }
    // warm-up: one eager call at this shape, so that nothing allocates, makes a tensor map or sets a function
    // attribute during the capture.  The rank streams start after home_stream's work so far (the caller's inputs).
    SATB_PROPAGATE(group_reserve(g, B, L, tb, split));
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[0]));
    SATB_CHECK_CUDA(cudaEventRecord(g->ev_graph, home));
    SATB_PROPAGATE(group_run(g, xs, ts, os, B, L, cfg_scale, scale_phi, st, tb, split, false, &io));
    cudaGraph_t graph = nullptr;
    unsigned long long launches = 0;
    SATB_PROPAGATE(group_capture(g, xs, ts, os, B, L, cfg_scale, scale_phi, st, tb, split, io, &graph, &launches));
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[0]));
    const cudaError_t e = cudaGraphInstantiate(&g->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
      g->exec = nullptr;
      cudaGetLastError();
      set_last_error(std::string("instantiating the group forward's graph: ") + cudaGetErrorString(e));
      return -3;
    }
    g->key = key;
    g->gens.resize(NH);
    for (int r = 0; r < NH; ++r) g->gens[r] = g->h[r]->gen;
    g->graph_launches = launches;
    ++g->captures;
  }
  SATB_CHECK_CUDA(cudaSetDevice(g->dev[0]));
  for (int r = 0; r < NH; ++r) SATB_CHECK_CUDA(cudaStreamWaitEvent(home, g->ev_done[r], 0));
  SATB_CHECK_CUDA(cudaGraphLaunch(g->exec, home));
  SATB_CHECK_CUDA(cudaEventRecord(g->ev_graph, home));
  g_launch_count += g->graph_launches;
  ++g->replays;
  return 0;
}

int satb_dit_group_graph_reset(SatbDitGroup* g) {
  SATB_REQUIRE(g, "null argument");
  group_drop_graph(g);
  return 0;
}

int satb_dit_group_graph_stats(const SatbDitGroup* g, long long* captures, long long* replays,
                               unsigned long long* launches) {
  SATB_REQUIRE(g && captures && replays && launches, "null argument");
  *captures = g->captures;
  *replays = g->replays;
  *launches = g->exec ? g->graph_launches : 0;
  return 0;
}

}  // extern "C"

// ---- satb_gemm_probe: one fused-epilogue GEMM for the tests.  It lives in this file so that it launches the very
// gemm_wgmma_kernel instances the forward and satb_dit_prepare_cond launch (another .cu file would compile its own
// copies); it instantiates no kernel the forward does not.
static bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

template <class E, int BN, bool BF16, bool FP8 = false>
static int probe_run(const void* a, const void* w, int M, int N, int K, const typename E::Params& ep, int b_static,
                     cudaStream_t st, const Fp8Scales& sc = Fp8Scales{}) {
  SATB_REQUIRE(N % E::kCols == 0, ("gemm probe: N must be a multiple of " + std::to_string(E::kCols)).c_str());
  TmapCache tc;
  return linear<E, BN, BF16, FP8>(tc, a, K, M, K, w, N, ep, st, b_static, sc);
}

static int probe_check_outputs(const SatbGemmProbe& p, int N) {
  const int out_elem = p.epi == SATB_EPI_STORE32 || p.epi == SATB_EPI_STORE32_POS ? 4 : 2;
  if (p.epi != SATB_EPI_RESIDUAL) {
    SATB_REQUIRE(p.out && aligned16(p.out), "gemm probe: out must be a 16-byte aligned device pointer");
    SATB_REQUIRE(p.ld >= (p.epi == SATB_EPI_SWIGLU ? N / 2 : N) && (p.ld * out_elem) % 16 == 0,
                 "gemm probe: ld must cover the output row and keep rows 16-byte aligned");
  } else {
    SATB_REQUIRE(p.h && aligned16(p.h) && p.ld >= N && p.ld % 4 == 0, "gemm probe: h must be 16-byte aligned, ld >= N, ld % 4 == 0");
  }
  for (const void* q : std::initializer_list<const void*>{p.bias, p.gate, p.cos_tab, p.sin_tab})
    SATB_REQUIRE(aligned16(q), "gemm probe: every vector must be 16-byte aligned");
  return 0;
}

template <bool BF16>
static int gemm_probe(const void* a, const void* w, int M, int N, int K, const SatbGemmProbe& p, cudaStream_t st) {
  const int bn = p.bn;
  SATB_PROPAGATE(probe_check_outputs(p, N));
  switch (p.epi) {
    case SATB_EPI_STORE32: {
      const EpiStore32::Params ep{static_cast<float*>(p.out), p.ld, p.bias};
      if (bn == 64) return probe_run<EpiStore32, 64, BF16>(a, w, M, N, K, ep, p.b_static, st);
      if (bn == 256) return probe_run<EpiStore32, 256, BF16>(a, w, M, N, K, ep, p.b_static, st);
      break;
    }
    case SATB_EPI_STORE32_POS: {
      SATB_REQUIRE(p.pos_tab && aligned16(p.pos_tab) && p.seq_len >= 1,
                   "gemm probe: store32_pos needs a 16-byte aligned pos_tab and seq_len >= 1");
      const EpiStore32Pos::Params ep{static_cast<float*>(p.out), p.ld, p.bias, p.pos_tab, p.seq_len};
      if (bn == 256) return probe_run<EpiStore32Pos, 256, BF16>(a, w, M, N, K, ep, p.b_static, st);
      break;
    }
    case SATB_EPI_STORE16: {
      typedef EpiStore16<BF16> E;
      const typename E::Params ep{p.out, p.ld, p.bias, p.act};
      if (bn == 128) return probe_run<E, 128, BF16>(a, w, M, N, K, ep, p.b_static, st);
      if (bn == 256) return probe_run<E, 256, BF16>(a, w, M, N, K, ep, p.b_static, st);
      break;
    }
    case SATB_EPI_HEAD_NORM16: {
      SATB_REQUIRE(!p.cos_tab || (p.sin_tab && p.seq_len >= 1), "gemm probe: rotary needs sin_tab and seq_len");
      typedef EpiHeadNorm16<BF16> E;
      const typename E::Params ep{p.out, p.ld, p.norm_cols, p.rope_cols, p.seq_len, p.cos_tab, p.sin_tab};
      if (bn == 128) return probe_run<E, 128, BF16>(a, w, M, N, K, ep, p.b_static, st);
      if (bn == 256) return probe_run<E, 256, BF16>(a, w, M, N, K, ep, p.b_static, st);
      break;
    }
    case SATB_EPI_QKV_ROPE: {
      SATB_REQUIRE(p.head_dim >= 32 && p.head_dim % 32 == 0 && p.nf % 4 == 0 && p.nf >= 4 && 2 * p.nf <= p.head_dim,
                   "gemm probe: head_dim must be a multiple of 32 and nf a multiple of 4 with 2 nf <= head_dim");
      SATB_REQUIRE(!p.cos_tab || (p.sin_tab && p.seq_len >= 1), "gemm probe: rotary needs sin_tab and seq_len");
      if (bn == 256) {
        typedef EpiQkvRope<BF16> E;
        const typename E::Params ep{p.out, p.ld, p.rope_cols, p.seq_len, p.head_dim, p.nf, p.cos_tab, p.sin_tab};
        return probe_run<E, 256, BF16>(a, w, M, N, K, ep, p.b_static, st);
      }
      break;
    }
    case SATB_EPI_SWIGLU: {
      if (bn == 256) {
        typedef EpiSwiglu<BF16> E;
        return probe_run<E, 256, BF16>(a, w, M, N, K, typename E::Params{p.out, p.ld, p.bias}, p.b_static, st);
      }
      break;
    }
    case SATB_EPI_RESIDUAL: {
      SATB_REQUIRE(!p.gate || (p.rows_per_item >= 1 && p.n_items >= 1 && p.gate_ld % 4 == 0),
                   "gemm probe: the gate needs rows_per_item, n_items >= 1 and gate_ld % 4 == 0");
      const EpiResidual::Params ep{p.h, p.ld, p.bias, p.gate, p.rows_per_item, p.gate_ld, p.n_items};
      if (bn == 128) return probe_run<EpiResidual, 128, BF16>(a, w, M, N, K, ep, p.b_static, st);
      if (bn == 256) return probe_run<EpiResidual, 256, BF16>(a, w, M, N, K, ep, p.b_static, st);
      break;
    }
    default:
      break;
  }
  set_last_error("gemm probe: no such instance (epi " + std::to_string(p.epi) + ", BN " + std::to_string(bn) +
                 "); the forward's instances are store32 BN 64/256, store16, head_norm16 and residual BN 128/256, "
                 "qkv_rope, swiglu and store32_pos BN 256");
  return -1;
}

extern "C" {

int satb_gemm_probe(const void* a16, const void* w16, int M, int N, int K, const SatbGemmProbe* p, void* stream) {
  SATB_REQUIRE(a16 && w16 && p, "null argument");
  SATB_REQUIRE(M >= 1 && N >= 32 && K >= 8 && K % 8 == 0, "gemm probe: need M >= 1, N >= 32 and K % 8 == 0");
  SATB_REQUIRE(aligned16(a16) && aligned16(w16), "gemm probe: operands must be 16-byte aligned");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return p->bf16 ? gemm_probe<true>(a16, w16, M, N, K, *p, st) : gemm_probe<false>(a16, w16, M, N, K, *p, st);
}

// The FP8 instances of the forward: qkv_rope and swiglu BN 256, store16 BN 128 / 256, head_norm16 BN 128 (fp16 outputs).
int satb_gemm_probe_fp8(const void* a8, const void* w8, const float* a_scale, const float* w_scale, int M, int N, int K,
                        const SatbGemmProbe* p, void* stream) {
  SATB_REQUIRE(a8 && w8 && a_scale && w_scale && p, "null argument");
  SATB_REQUIRE(M >= 1 && N >= 32 && K >= 128 && K % 128 == 0, "gemm probe fp8: need M >= 1, N >= 32 and K % 128 == 0");
  SATB_REQUIRE(aligned16(a8) && aligned16(w8) && aligned16(w_scale), "gemm probe fp8: operands must be 16-byte aligned");
  SATB_REQUIRE(p->bf16 == 0, "gemm probe fp8: the FP8 instances store fp16");
  SATB_PROPAGATE(probe_check_outputs(*p, N));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Fp8Scales sc{a_scale, w_scale};
  const int bn = p->bn;
  switch (p->epi) {
    case SATB_EPI_STORE16: {
      typedef EpiStore16<false> E;
      const E::Params ep{p->out, p->ld, p->bias, p->act};
      if (bn == 128) return probe_run<E, 128, false, true>(a8, w8, M, N, K, ep, p->b_static, st, sc);
      if (bn == 256) return probe_run<E, 256, false, true>(a8, w8, M, N, K, ep, p->b_static, st, sc);
      break;
    }
    case SATB_EPI_HEAD_NORM16: {
      SATB_REQUIRE(!p->cos_tab || (p->sin_tab && p->seq_len >= 1), "gemm probe: rotary needs sin_tab and seq_len");
      typedef EpiHeadNorm16<false> E;
      const E::Params ep{p->out, p->ld, p->norm_cols, p->rope_cols, p->seq_len, p->cos_tab, p->sin_tab};
      if (bn == 128) return probe_run<E, 128, false, true>(a8, w8, M, N, K, ep, p->b_static, st, sc);
      break;
    }
    case SATB_EPI_QKV_ROPE: {
      SATB_REQUIRE(p->head_dim >= 32 && p->head_dim % 32 == 0 && p->nf % 4 == 0 && p->nf >= 4 && 2 * p->nf <= p->head_dim,
                   "gemm probe: head_dim must be a multiple of 32 and nf a multiple of 4 with 2 nf <= head_dim");
      SATB_REQUIRE(!p->cos_tab || (p->sin_tab && p->seq_len >= 1), "gemm probe: rotary needs sin_tab and seq_len");
      if (bn == 256) {
        typedef EpiQkvRope<false> E;
        const E::Params ep{p->out, p->ld, p->rope_cols, p->seq_len, p->head_dim, p->nf, p->cos_tab, p->sin_tab};
        return probe_run<E, 256, false, true>(a8, w8, M, N, K, ep, p->b_static, st, sc);
      }
      break;
    }
    case SATB_EPI_SWIGLU: {
      if (bn == 256) {
        typedef EpiSwiglu<false> E;
        return probe_run<E, 256, false, true>(a8, w8, M, N, K, E::Params{p->out, p->ld, p->bias}, p->b_static, st, sc);
      }
      break;
    }
    default:
      break;
  }
  set_last_error("gemm probe fp8: no such instance (epi " + std::to_string(p->epi) + ", BN " + std::to_string(bn) +
                 "); the forward's FP8 instances are qkv_rope and swiglu BN 256, store16 BN 128 / 256 and head_norm16 BN 128");
  return -1;
}

// The e4m3 QKV epilogues of FP8 self-attention (EpiQkvRopeE4m3 BN 256, EpiHeadNormE4m3 BN 256 / FP8 BN 128), as the
// forward launches them: 16-bit operands when a_scale is null, e4m3 operands with their row scales otherwise.
int satb_gemm_probe_qk8(const void* a, const void* w, const float* a_scale, const float* w_scale, int M, int N, int K,
                        const SatbGemmProbe* p, const SatbQkE4m3* o, void* stream) {
  SATB_REQUIRE(a && w && p && o && o->q8 && o->k8 && o->sq && o->sk, "null argument");
  const bool fp8 = a_scale != nullptr;
  SATB_REQUIRE(!fp8 || w_scale, "gemm probe qk8: a_scale needs w_scale");
  SATB_REQUIRE(aligned16(a) && aligned16(w) && aligned16(o->q8) && aligned16(o->k8) && (!fp8 || aligned16(w_scale)),
               "gemm probe qk8: operands and q8 / k8 must be 16-byte aligned");
  SATB_REQUIRE(M >= 1 && K >= 8 && K % (fp8 ? 128 : 8) == 0, "gemm probe qk8: need M >= 1 and K % 8 == 0 (FP8: 128)");
  SATB_REQUIRE(o->heads >= 1 && N % 64 == 0 && N >= 128 * o->heads, "gemm probe qk8: N must be a multiple of 64 holding "
               "the 2 heads * 64 q / k columns");
  SATB_REQUIRE(p->seq_len >= 1 && o->scale_ld >= p->seq_len, "gemm probe qk8: need seq_len >= 1 and scale_ld >= seq_len");
  SATB_REQUIRE(!fp8 || !p->bf16, "gemm probe qk8: the FP8 instances store fp16");
  SATB_REQUIRE(p->out && aligned16(p->out) && p->ld >= N && p->ld % 8 == 0, "gemm probe qk8: out must be 16-byte aligned, ld >= N");
  SATB_REQUIRE(!p->cos_tab || (p->sin_tab && aligned16(p->cos_tab) && aligned16(p->sin_tab)),
               "gemm probe qk8: rotary needs 16-byte aligned cos_tab and sin_tab");
  const QkE4m3Out q{static_cast<uint8_t*>(o->q8), static_cast<uint8_t*>(o->k8), o->sq, o->sk, o->heads, o->scale_ld};
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Fp8Scales sc{a_scale, w_scale};
  const int bn = p->bn;
  auto rope = [&](auto bf) -> int {
    constexpr bool BF16 = decltype(bf)::value;
    typedef EpiQkvRopeE4m3<BF16> E;
    const typename E::Params ep{{p->out, p->ld, p->rope_cols, p->seq_len, 64, 16, p->cos_tab, p->sin_tab}, q};
    if constexpr (!BF16)   // the FP8 instances store fp16
      if (fp8) return probe_run<E, 256, false, true>(a, w, M, N, K, ep, p->b_static, st, sc);
    return probe_run<E, 256, BF16>(a, w, M, N, K, ep, p->b_static, st);
  };
  auto norm = [&](auto bf) -> int {
    constexpr bool BF16 = decltype(bf)::value;
    typedef EpiHeadNormE4m3<BF16> E;
    const typename E::Params ep{{p->out, p->ld, 128 * o->heads, p->rope_cols, p->seq_len, p->cos_tab, p->sin_tab}, q};
    if constexpr (!BF16)
      if (fp8) return probe_run<E, 128, false, true>(a, w, M, N, K, ep, p->b_static, st, sc);
    return probe_run<E, 256, BF16>(a, w, M, N, K, ep, p->b_static, st);
  };
  if (p->epi == SATB_EPI_QKV_ROPE_E4M3 && bn == 256)
    return p->bf16 ? rope(std::true_type{}) : rope(std::false_type{});
  if (p->epi == SATB_EPI_HEAD_NORM_E4M3 && bn == (fp8 ? 128 : 256))
    return p->bf16 ? norm(std::true_type{}) : norm(std::false_type{});
  set_last_error("gemm probe qk8: no such instance (epi " + std::to_string(p->epi) + ", BN " + std::to_string(bn) +
                 "); the forward's are qkv_rope_e4m3 BN 256 and head_norm_e4m3 BN 256 (FP8 operands: BN 128)");
  return -1;
}

// The GEMMs of the FP8 FF-out option as the forward launches them: FF-in with an e4m3 block epilogue (EpiSwigluE4m3
// BN 256, EpiSiluE4m3 BN 128 / 256) and FF-out on block-scaled A (BlockScaledA<EpiResidual> BN 128).
int satb_gemm_probe_ff8(const void* a8, const void* w8, const float* a_scale, const float* w_scale, int M, int N, int K,
                        const SatbGemmProbe* p, void* ff8, float* ff_scale, void* stream) {
  SATB_REQUIRE(a8 && w8 && a_scale && w_scale && p, "null argument");
  SATB_REQUIRE(M >= 1 && N >= 32 && K >= 128 && K % 128 == 0, "gemm probe ff8: need M >= 1, N >= 32 and K % 128 == 0");
  SATB_REQUIRE(aligned16(a8) && aligned16(w8) && aligned16(w_scale), "gemm probe ff8: operands must be 16-byte aligned");
  SATB_REQUIRE(p->bf16 == 0, "gemm probe ff8: the FP8 instances are fp16-mode instances (bf16 must be 0)");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Fp8Scales sc{a_scale, w_scale};
  const int bn = p->bn;
  if (p->epi == SATB_EPI_SWIGLU_E4M3 || p->epi == SATB_EPI_SILU_E4M3) {
    const bool glu = p->epi == SATB_EPI_SWIGLU_E4M3;
    const int cols = glu ? N / 2 : N;
    SATB_REQUIRE(ff8 && ff_scale && aligned16(ff8) && aligned16(ff_scale) && aligned16(p->bias),
                 "gemm probe ff8: ff8, ff_scale (and bias) must be 16-byte aligned device pointers");
    SATB_REQUIRE(p->ld >= cols && p->ld % 128 == 0, "gemm probe ff8: ld must cover the output row and be a multiple of 128");
    const BlockE4m3Out o{static_cast<uint8_t*>(ff8), ff_scale, p->ld};
    if (glu && bn == 256)
      return probe_run<EpiSwigluE4m3, 256, false, true>(a8, w8, M, N, K, EpiSwigluE4m3::Params{o, p->bias}, p->b_static,
                                                        st, sc);
    if (!glu && bn == 128)
      return probe_run<EpiSiluE4m3, 128, false, true>(a8, w8, M, N, K, EpiSiluE4m3::Params{o, p->bias}, p->b_static, st, sc);
    if (!glu && bn == 256)
      return probe_run<EpiSiluE4m3, 256, false, true>(a8, w8, M, N, K, EpiSiluE4m3::Params{o, p->bias}, p->b_static, st, sc);
  } else if (p->epi == SATB_EPI_RESIDUAL_A8 && bn == 128) {
    SatbGemmProbe q = *p;
    q.epi = SATB_EPI_RESIDUAL;   // the residual epilogue's output checks
    SATB_PROPAGATE(probe_check_outputs(q, N));
    SATB_REQUIRE(!p->gate || (p->rows_per_item >= 1 && p->n_items >= 1 && p->gate_ld % 4 == 0),
                 "gemm probe: the gate needs rows_per_item, n_items >= 1 and gate_ld % 4 == 0");
    const EpiResidual::Params ep{p->h, p->ld, p->bias, p->gate, p->rows_per_item, p->gate_ld, p->n_items};
    return probe_run<BlockScaledA<EpiResidual>, 128, false, true>(a8, w8, M, N, K, ep, p->b_static, st, sc);
  }
  set_last_error("gemm probe ff8: no such instance (epi " + std::to_string(p->epi) + ", BN " + std::to_string(bn) +
                 "); the forward's are swiglu_e4m3 BN 256, silu_e4m3 BN 128 / 256 and residual_a8 BN 128");
  return -1;
}

}  // extern "C"

// The feed-forward's token convolutions, through token_conv as the forward calls it.
template <bool BF16>
static int token_conv_probe(const void* a, long long item_stride, const void* w, int R, int n_seq, int K, int N, int k,
                            const SatbGemmProbe& p, cudaStream_t st) {
  TmapCache tc;
  if (p.epi == SATB_EPI_STORE16) {
    typedef EpiStore16<BF16> E;
    return token_conv<E, BF16>(tc, a, item_stride, R, n_seq, K, w, N, k, typename E::Params{p.out, p.ld, p.bias, p.act},
                               st, p.bn);
  }
  const EpiResidual::Params ep{p.h, p.ld, p.bias, p.gate, p.rows_per_item, p.gate_ld, p.n_items};
  return token_conv<EpiResidual, BF16>(tc, a, item_stride, R, n_seq, K, w, N, k, ep, st, p.bn);
}

extern "C" {

int satb_token_conv_probe(const void* a16, long long item_stride, const void* w16, int R, int n_seq, int K, int N, int k,
                          const SatbGemmProbe* p, void* stream) {
  SATB_REQUIRE(a16 && w16 && p, "null argument");
  SATB_REQUIRE(aligned16(a16) && aligned16(w16), "token conv probe: operands must be 16-byte aligned");
  SATB_REQUIRE(R >= 1 && n_seq >= 1 && item_stride >= n_seq, "token conv probe: need R, n_seq >= 1 and item_stride >= n_seq");
  SATB_REQUIRE(K >= 8 && K % 8 == 0 && N >= 32 && N % 32 == 0, "token conv probe: need K % 8 == 0 and N % 32 == 0");
  SATB_REQUIRE(k >= 1 && k % 2 == 1, "token conv probe: the kernel size must be odd");
  SATB_REQUIRE(p->epi == SATB_EPI_STORE16 || p->epi == SATB_EPI_RESIDUAL,
               "token conv probe: the forward's convolutions run the store16 and residual epilogues only");
  SATB_REQUIRE(p->bn == 0 || p->bn == 128 || p->bn == 256, "token conv probe: bn must be 0 (the forward's pick), 128 or 256");
  SATB_REQUIRE(p->epi == SATB_EPI_STORE16 || !p->gate || (p->rows_per_item >= 1 && p->n_items >= 1 && p->gate_ld % 4 == 0),
               "token conv probe: the gate needs rows_per_item, n_items >= 1 and gate_ld % 4 == 0");
  SATB_PROPAGATE(probe_check_outputs(*p, N));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return p->bf16 ? token_conv_probe<true>(a16, item_stride, w16, R, n_seq, K, N, k, *p, st)
                 : token_conv_probe<false>(a16, item_stride, w16, R, n_seq, K, N, k, *p, st);
}

int satb_dit_pre_probe(const float* x, void* a16, int R, int B_src, int C, int lda, int L, int P, int bf16, void* stream) {
  SATB_REQUIRE(x && a16, "null argument");
  SATB_REQUIRE(R >= 1 && B_src >= 1 && C >= 1 && L >= 1 && P >= 0, "dit pre probe: need R, B_src, C, L >= 1 and P >= 0");
  SATB_REQUIRE(lda >= C && lda % 8 == 0, "dit pre probe: need lda >= C and lda % 8 == 0");
  return launch_dit_pre(x, a16, R, B_src, C, lda, L, P, bf16 != 0, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
