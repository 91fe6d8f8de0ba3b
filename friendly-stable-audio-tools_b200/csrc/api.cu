// C-ABI entry points for the stand-alone primitives (see include/satb200.h).
#include "../../include/satb200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.h"

using namespace satb;

namespace {
inline bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }
constexpr int kMaxGridYZ = 65535;
}  // namespace

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

// ---- test entry points of the small kernels: argument checks, then the launch function the forward calls
int satb_layernorm_mod(const float* x, const float* gamma, const float* beta, const float* mod_scale,
                       const float* mod_shift, long long mod_stride, int rows_per_item, int n_items, void* out16,
                       int rows, int D, int bf16, void* stream) {
  SATB_REQUIRE(x && gamma && out16, "null argument");
  SATB_REQUIRE(!mod_scale || (mod_shift && rows_per_item >= 1 && n_items >= 1 && mod_stride % 4 == 0),
               "adaLN modulation needs shift, rows_per_item >= 1, n_items >= 1 and mod_stride % 4 == 0");
  SATB_REQUIRE(aligned_to(x, 16) && aligned_to(gamma, 16) && aligned_to(beta, 16) && aligned_to(mod_scale, 16) &&
                   aligned_to(mod_shift, 16) && aligned_to(out16, 8),
               "LayerNorm: x, gamma, beta and the modulation must be 16-byte aligned, out 8-byte aligned");
  SATB_REQUIRE(rows >= 0, "LayerNorm: negative row count");
  return launch_layernorm(x, gamma, beta, out16, rows, D, mod_scale, mod_shift, mod_stride, mod_scale ? rows_per_item : 1,
                          mod_scale ? n_items : 1, bf16 != 0, static_cast<cudaStream_t>(stream));
}

int satb_fourier_probe(const float* t, const float* w, float* out, int B, int F, void* stream) {
  SATB_REQUIRE(t && w && out, "null argument");
  SATB_REQUIRE(B >= 1 && F >= 1 && static_cast<long long>(B) * F <= (1 << 30), "fourier probe: need B, F >= 1");
  return launch_fourier(t, w, out, B, F, static_cast<cudaStream_t>(stream));
}

int satb_skinny_linear_probe(const float* in, const float* W, const float* bias, const float* add, float* out, int R,
                             int K, int N, int silu_out, void* stream) {
  SATB_REQUIRE(in && W && out, "null argument");
  SATB_REQUIRE(aligned_to(in, 16) && aligned_to(W, 16), "skinny linear probe: in and W must be 16-byte aligned");
  SATB_REQUIRE(K >= 4 && N >= 1, "skinny linear probe: need K >= 4 and N >= 1");
  return launch_skinny_linear(in, W, bias, add, out, R, K, N, silu_out, static_cast<cudaStream_t>(stream));
}

int satb_write_prepend_probe(const float* tok, const float* pre, const float* pos, float* h, int R, int B, int N_seq,
                             int D, int Pp, void* stream) {
  SATB_REQUIRE(tok && h, "null argument");
  SATB_REQUIRE(B >= 1 && R >= 1 && R <= kMaxGridYZ && D >= 1, "write prepend probe: need B, D >= 1 and 1 <= R <= 65535");
  SATB_REQUIRE(Pp >= 0 && Pp < kMaxGridYZ && N_seq > Pp, "write prepend probe: need 0 <= Pp < N_seq");
  return launch_write_prepend(tok, pre, pos, h, R, B, N_seq, D, Pp, static_cast<cudaStream_t>(stream));
}

int satb_gate_sigmoid_probe(float* ssg, int rows, int depth, int D, void* stream) {
  SATB_REQUIRE(ssg, "null argument");
  SATB_REQUIRE(rows >= 1 && rows <= kMaxGridYZ && depth >= 1 && D >= 1 &&
                   static_cast<long long>(depth) * 6 * D <= (1 << 30),
               "gate sigmoid probe: need 1 <= rows <= 65535 and depth, D >= 1");
  return launch_gate_sigmoid(ssg, rows, depth, D, static_cast<cudaStream_t>(stream));
}

int satb_dit_post_probe(const float* y, int ldy, float* out, int B, int C, int L, int N_seq, int P, int cfg,
                        float cfg_scale, float scale_phi, void* stream) {
  SATB_REQUIRE(y && out, "null argument");
  SATB_REQUIRE(B >= 1 && B <= kMaxGridYZ && C >= 1 && L >= 1 && P >= 0, "dit post probe: need 1 <= B <= 65535, C, L >= 1 and P >= 0");
  SATB_REQUIRE(N_seq >= P && N_seq - P >= L, "dit post probe: need N_seq >= P + L");
  return launch_dit_post(y, y + static_cast<size_t>(B) * N_seq * ldy, ldy, out, B, C, L, N_seq, P, cfg != 0, cfg_scale,
                         scale_phi, static_cast<cudaStream_t>(stream));
}

int satb_cast_rows_probe(const float* src, void* dst16, const int* perm, int rows, int cols, long long src_ld,
                         long long dst_ld, int bf16, void* stream) {
  SATB_REQUIRE(src && dst16, "null argument");
  SATB_REQUIRE(rows >= 1 && cols >= 1, "cast rows probe: need rows, cols >= 1");
  SATB_REQUIRE(src_ld >= cols && dst_ld >= cols, "cast rows probe: the row pitches must cover the columns");
  return launch_cast_rows(src, dst16, perm, rows, cols, src_ld, dst_ld, bf16 != 0, static_cast<cudaStream_t>(stream));
}

int satb_quant_rows_fp8_probe(const float* src, void* dst8, float* row_scale, const int* perm, int rows, int cols,
                              void* stream) {
  SATB_REQUIRE(src && dst8 && row_scale, "null argument");
  SATB_REQUIRE(rows >= 1 && cols >= 4, "FP8 row quantisation probe: need rows >= 1 and cols >= 4");
  SATB_REQUIRE(aligned_to(dst8, 4), "FP8 row quantisation probe: dst must be 4-byte aligned");
  return launch_quant_rows_fp8(src, dst8, row_scale, perm, rows, cols, static_cast<cudaStream_t>(stream));
}

int satb_matmul_f64_probe(const float* A, const float* B, float* C, int M, int N, int K, void* stream) {
  SATB_REQUIRE(A && B && C, "null argument");
  SATB_REQUIRE(M >= 1 && N >= 1 && K >= 1 && (M + 63) / 64 <= kMaxGridYZ, "matmul probe: need M, N, K >= 1 and M <= 64 * 65535");
  return launch_matmul_f64(A, B, C, M, N, K, static_cast<cudaStream_t>(stream));
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

int satb_vdiffusion_update(const float* x, const float* v, const float* noise, float* x_next, float* pred, long long n,
                           float alpha, float sigma, float alpha_next, float adj_sigma, float ddim_sigma, void* stream) {
  SATB_REQUIRE(x && v, "null argument");
  SATB_REQUIRE(x_next || pred, "v-diffusion update: x_next and pred are both null (nothing to write)");
  SATB_REQUIRE(n >= 1, "v-diffusion update: element count must be positive");
  return launch_vdiffusion_update(x, v, noise, x_next, pred, n, alpha, sigma, alpha_next, adj_sigma, ddim_sigma,
                                  static_cast<cudaStream_t>(stream));
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

// FP8 self-attention pieces (attention_fp8.cu), as the DiT forward launches them, on caller-owned buffers
int satb_attention_fp8_vt(const void* v16, void* vt8, float* sv, int B, int H, int N, int bf16, void* stream) {
  SATB_REQUIRE(v16 && vt8 && sv, "null argument");
  SATB_REQUIRE(B >= 1 && B <= kMaxGridYZ && H >= 1 && H <= kMaxGridYZ && N >= 1,
               "FP8 attention V quantiser: need 1 <= B, H <= 65535 and N >= 1");
  const int64_t D = static_cast<int64_t>(H) * 64;
  const AttnFp8Bufs b{nullptr, nullptr, nullptr, nullptr, static_cast<uint8_t*>(vt8), sv};
  return launch_attention_fp8_vt(v16, D, N * D, b, B, H, N, bf16 != 0, static_cast<cudaStream_t>(stream));
}

int satb_attention_fp8_core(const void* q8, const void* k8, const float* sq, const float* sk, const void* vt8,
                            const float* sv, void* o16, int B, int H, int Nq, int Nk, int bf16, void* stream) {
  SATB_REQUIRE(q8 && k8 && sq && sk && vt8 && sv && o16, "null argument");
  SATB_REQUIRE(B >= 1 && B <= kMaxGridYZ && H >= 1 && H <= kMaxGridYZ && Nq >= 1 && Nk >= 1,
               "FP8 attention: need 1 <= B, H <= 65535 and Nq, Nk >= 1");
  SATB_REQUIRE(aligned_to(q8, 16) && aligned_to(k8, 16) && aligned_to(sq, 16) && aligned_to(sk, 16) &&
                   aligned_to(vt8, 16) && aligned_to(sv, 8),
               "FP8 attention: q8, k8, vt8 and the row scales must be 16-byte aligned, sv 8-byte aligned");
  const AttnFp8Bufs b{const_cast<uint8_t*>(static_cast<const uint8_t*>(q8)), const_cast<uint8_t*>(static_cast<const uint8_t*>(k8)),
                      const_cast<float*>(sq), const_cast<float*>(sk), const_cast<uint8_t*>(static_cast<const uint8_t*>(vt8)),
                      const_cast<float*>(sv)};
  AttnFp8Maps maps;
  SATB_PROPAGATE(make_attention_fp8_maps(&maps, b, B, H, Nq, Nk));
  const int64_t D = static_cast<int64_t>(H) * 64;
  return launch_attention_fp8(maps, b, o16, D, Nq * D, B, H, Nq, Nk, bf16 != 0, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
