// C-ABI entry points for the stand-alone primitives (see include/satb200.h).
#include "../../include/satb200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.h"

using namespace satb;

extern "C" {

int satb_snake_beta(const float* x, const float* alpha, const float* beta, float* y, int B, int C, long long T,
                    int logscale, void* stream) {
  SATB_REQUIRE(x && alpha && beta && y, "null argument");
  return launch_snake_beta(x, alpha, beta, y, B, C, T, logscale, static_cast<cudaStream_t>(stream));
}

int satb_layernorm(const float* x, const float* gamma, const float* beta, void* out16, int rows, int D, int bf16,
                   void* stream) {
  SATB_REQUIRE(x && gamma && out16, "null argument");
  return launch_layernorm(x, gamma, beta, out16, rows, D, nullptr, nullptr, 0, 1, 1, bf16 != 0,
                          static_cast<cudaStream_t>(stream));
}

int satb_layernorm_fp8(const float* x, const float* gamma, const float* beta, const float* mod_scale,
                       const float* mod_shift, long long mod_stride, int rows_per_item, int n_items, void* out8,
                       float* row_scale, int rows, int D, void* stream) {
  SATB_REQUIRE(x && gamma && out8 && row_scale, "null argument");
  SATB_REQUIRE(!mod_scale || (mod_shift && rows_per_item >= 1 && n_items >= 1 && mod_stride % 4 == 0),
               "adaLN modulation needs shift, rows_per_item >= 1, n_items >= 1 and mod_stride % 4 == 0");
  return launch_layernorm_fp8(x, gamma, beta, out8, row_scale, rows, D, mod_scale, mod_shift, mod_stride,
                              rows_per_item, n_items, static_cast<cudaStream_t>(stream));
}

int satb_linear_f32out(const void* a16, const void* w16, float* c, int M, int N, int K, int bf16, void* stream) {
  SATB_REQUIRE(a16 && w16 && c, "null argument");
  SATB_REQUIRE(M >= 1 && N >= 32 && N % 32 == 0 && K >= 8 && K % 8 == 0, "linear: need N % 32 == 0 and K % 8 == 0");
  CUtensorMap ta, tb;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GemmShape s;
  s.L = M; s.batches = 1; s.N = N; s.K = K; s.n_taps = 1; s.tap_base = 0; s.tap_step = 0; s.b_tap_rows = N; s.stride = 1;
  EpiStore32::Params ep{c, N, nullptr};
  SATB_PROPAGATE(make_tmap_a(&ta, a16, K, M, 1, K, static_cast<int64_t>(M) * K));
  if (N % 256 == 0 || N > 256) {
    SATB_PROPAGATE(make_tmap_b(&tb, w16, K, N, K, 256));
    return bf16 ? launch_gemm<EpiStore32, 256, true>(ta, tb, s, ep, st) : launch_gemm<EpiStore32, 256, false>(ta, tb, s, ep, st);
  } else if (N > 64) {
    SATB_PROPAGATE(make_tmap_b(&tb, w16, K, N, K, 128));
    return bf16 ? launch_gemm<EpiStore32, 128, true>(ta, tb, s, ep, st) : launch_gemm<EpiStore32, 128, false>(ta, tb, s, ep, st);
  }
  SATB_PROPAGATE(make_tmap_b(&tb, w16, K, N, K, 64));
  return bf16 ? launch_gemm<EpiStore32, 64, true>(ta, tb, s, ep, st) : launch_gemm<EpiStore32, 64, false>(ta, tb, s, ep, st);
}

int satb_sampler_update(const float* x, const float* v, const float* den_1, const float* den_2, const float* noise,
                        float* den, float* x_next, float* x_in_next, long long n, float c_skip, float c_out, float a,
                        float b, float c, float d, float s, float c_in_next, void* stream) {
  SATB_REQUIRE(x && v && den && x_next, "null argument");
  return launch_sampler_update(x, v, den_1, den_2, noise, den, x_next, x_in_next, n, c_skip, c_out, a, b, c, d, s,
                               c_in_next, static_cast<cudaStream_t>(stream));
}

int satb_attention(const void* q16, const void* k16, const void* v16, void* o16, int B, int H, int Hkv, int Nq, int Nk,
                   int bf16, void* stream) {
  return satb_attention_hd(q16, k16, v16, o16, B, H, Hkv, Nq, Nk, 64, bf16, stream);
}

int satb_attention_hd(const void* q16, const void* k16, const void* v16, void* o16, int B, int H, int Hkv, int Nq,
                      int Nk, int head_dim, int bf16, void* stream) {
  SATB_REQUIRE(q16 && k16 && v16 && o16, "null argument");
  const int64_t dq = static_cast<int64_t>(H) * head_dim, dk = static_cast<int64_t>(Hkv) * head_dim;
  return launch_attention_tc(q16, k16, v16, o16, dq, dk, dk, dq, Nq * dq, Nk * dk, Nk * dk, Nq * dq, static_cast<int>(dq),
                             static_cast<int>(dk), static_cast<int>(dk), 0, 0, 0, B, H, Hkv, Nq, Nk, head_dim, bf16 != 0,
                             static_cast<cudaStream_t>(stream));
}

int satb_attention_probe(const SatbAttentionProbe* p, void* stream) {
  SATB_REQUIRE(p && p->q && p->k && p->v && p->o, "null argument");
  SATB_REQUIRE(p->B >= 1, "attention needs at least one batch item");
  SATB_REQUIRE(p->q_col >= 0 && p->k_col >= 0 && p->v_col >= 0 && p->ldq >= 0 && p->ldk >= 0 && p->ldv >= 0 &&
                   p->ldo >= 0 && p->q_bs >= 0 && p->k_bs >= 0 && p->v_bs >= 0 && p->o_bs >= 0,
               "attention column offsets and strides must not be negative");
  SATB_REQUIRE(p->q_cols <= p->ldq && p->k_cols <= p->ldk && p->v_cols <= p->ldv,
               "attention operand columns exceed the row pitch");
  return launch_attention_tc(p->q, p->k, p->v, p->o, p->ldq, p->ldk, p->ldv, p->ldo, p->q_bs, p->k_bs, p->v_bs, p->o_bs,
                             p->q_cols, p->k_cols, p->v_cols, p->q_col, p->k_col, p->v_col, p->B, p->H, p->Hkv, p->Nq,
                             p->Nk, p->head_dim, p->bf16 != 0, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
