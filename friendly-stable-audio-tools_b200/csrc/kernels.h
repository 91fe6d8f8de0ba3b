// Internal launch API between translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

struct SatbSamplerStep;   // include/satb200.h

namespace satb {

// ---- attention_tc.cu (tensor-core flash attention; head_dim 32, 64, 96 or 128)
// Head dim 64 reads q / k / v through tensor maps: make_tmap_a(ptr, cols, rows per item, batch, ld, batch stride) with
// the default box.  tmq / tmk / tmv may pass such maps cached by the caller; null ones are encoded here.
int launch_attention_tc(const void* q, const void* k, const void* v, void* o, int64_t ldq, int64_t ldk, int64_t ldv,
                        int64_t ldo, int64_t q_bs, int64_t k_bs, int64_t v_bs, int64_t o_bs, int q_cols, int k_cols,
                        int v_cols, int q_col, int k_col, int v_col, int batch, int H, int H_kv, int Nq, int Nk,
                        int head_dim, bool bf16, cudaStream_t stream, const CUtensorMap* tmq = nullptr,
                        const CUtensorMap* tmk = nullptr, const CUtensorMap* tmv = nullptr);

// ---- attention_fp8.cu (FP8 self-attention, head dim 64, one kv head per head)
// Operands of B items, H heads, Nq query / Nk key rows per item; pad(n) = n rounded up to a multiple of 128:
//   q8 [B, Nq, H * 64], k8 [B, Nk, H * 64] e4m3 rows;  sq [B * H, pad(Nq)], sk [B * H, pad(Nk)] their power-of-two
//   (row, head) scales;  vt8 [B * H, 64, pad(Nk)] e4m3 V^T (keys of each 32-key group in fp8_key_of order, zero past
//   Nk);  sv [B * H, 64] the (item, head, channel) scales of v.
struct AttnFp8Bufs {
  uint8_t *q8, *k8;
  float *sq, *sk;
  uint8_t* vt8;
  float* sv;
};
struct AttnFp8Maps {
  CUtensorMap q, k, vt, sk;
};
__host__ __device__ constexpr int attn_fp8_pad(int n) { return (n + 127) / 128 * 128; }
size_t attn_fp8_workspace_bytes(int B, int H, int Nq, int Nk);
AttnFp8Bufs attn_fp8_bufs(void* ws, int B, int H, int Nq, int Nk);   // carves a workspace of the size above
// V^T and its channel scales from 16-bit v [B, N, ld] (item stride bs, head h at column
// h * 64); q8 / k8 and their scales come from the QKV GEMM's e4m3 epilogues (gemm.cuh QkE4m3Out)
int launch_attention_fp8_vt(const void* v, int64_t ld, int64_t bs, const AttnFp8Bufs& o, int B, int H, int N, bool bf16,
                            cudaStream_t stream);
int make_attention_fp8_maps(AttnFp8Maps* m, const AttnFp8Bufs& bufs, int B, int H, int Nq, int Nk);
// o [B, Nq, ldo] 16-bit (item stride o_bs), head h at column h * 64
int launch_attention_fp8(const AttnFp8Maps& maps, const AttnFp8Bufs& bufs, void* o, int64_t ldo, int64_t o_bs, int B,
                         int H, int Nq, int Nk, bool bf16, cudaStream_t stream);

// ---- runtime.cu: a 2-D / 3-D tensor map (dims[0] innermost, strides of dims 1.. in bytes), zero OOB fill
int make_tmap_nd(CUtensorMap* m, const void* ptr, int rank, int dtype, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle);

// ---- elementwise.cu
// LayerNorm over the last dim (eps 1e-5), optional adaLN modulation y*(1+scale)+shift, 16-bit output.
int launch_layernorm(const float* x, const float* gamma, const float* beta, void* out16, int rows, int D,
                     const float* scale, const float* shift, int64_t mod_stride, int rows_per_item, int n_items,
                     bool bf16, cudaStream_t stream);
// The same LayerNorm with an e4m3 output and one power-of-two scale per row (elementwise.cu, fp8_row_exp):
// out8[row, :] = e4m3(y / row_scale[row]).
int launch_layernorm_fp8(const float* x, const float* gamma, const float* beta, void* out8, float* row_scale, int rows,
                         int D, const float* scale, const float* shift, int64_t mod_stride, int rows_per_item,
                         int n_items, cudaStream_t stream);
// Weight matrix -> e4m3 rows with power-of-two row scales: dst[r, :] = e4m3(src[perm ? perm[r] : r, :] / row_scale[r]).
int launch_quant_rows_fp8(const float* src, void* dst, float* row_scale, const int* perm, int rows, int cols,
                          cudaStream_t stream);
// Fused VDenoiser scaling + multistep sampler update + noise (see elementwise.cu).
int launch_sampler_update(const float* x, const float* v, const float* d1, const float* d2, const float* nz, float* den,
                          float* x_next, float* x_in, long long n, float c_skip, float c_out, float A, float B, float C,
                          float D, float S, float c_in_next, cudaStream_t stream);
// One model call's sampler arithmetic of the fixed-step samplers, inpainting blend included (see sampler.cu and
// SatbSamplerStep in include/satb200.h).
int launch_sampler_step(const ::SatbSamplerStep& p, cudaStream_t stream);
// One v-diffusion DDIM step in the reference's fp32 operation order (see elementwise.cu).
int launch_vdiffusion_update(const float* x, const float* v, const float* nz, float* x_next, float* pred, long long n,
                             float alpha, float sigma, float alpha_next, float adj_sigma, float ddim_sigma,
                             cudaStream_t stream);
// SnakeBeta on [B, C, T] fp32 (log-scale alpha/beta per channel).
int launch_snake_beta(const float* x, const float* alpha, const float* beta, float* y, int B, int C, int64_t T,
                      int logscale, cudaStream_t stream);
// x[B_src, C, L] fp32 -> a16[(r*N_seq + P + l), c] at row pitch lda >= C (rows r*N_seq .. +P-1 and columns
// C .. lda-1 zero), r < R, source row r % B_src.
int launch_dit_pre(const float* x, void* a16, int R, int B_src, int C, int lda, int L, int P, bool bf16,
                   cudaStream_t stream);
// Fourier timestep features [B, 2*F]: cat(cos(2*pi*t*w), sin(2*pi*t*w)).
int launch_fourier(const float* t, const float* w, float* out, int B, int F, cudaStream_t stream);
// out[r, n] = act_out(sum_k in[r, k] * W[n, k] + bias[n] (+ add[r, n])); fp32 weights; act_out = SiLU if silu_out.
int launch_skinny_linear(const float* in, const float* W, const float* bias, const float* add, float* out, int R,
                         int K, int N, int silu_out, cudaStream_t stream);
// h[r*N_seq + j, :] = pre[r, j, :] (j < Pp; zeros for rows r >= B or pre == null), h[r*N_seq + Pp, :] = tok[r % B, :];
// plus pos[j, :] on every row j <= Pp when pos (the [N_seq, D] positional embedding table) is given
int launch_write_prepend(const float* tok, const float* pre, const float* pos, float* h, int R, int B, int N_seq, int D,
                         int Pp, cudaStream_t stream);
// in place: x = sigmoid(1 - x) on column ranges [c0, c0+D) and [c1, c1+D) of every 6D-wide layer block
int launch_gate_sigmoid(float* ssg, int rows, int depth, int D, cudaStream_t stream);
// y[B*N_seq, ldy] fp32 (its first C columns) -> out[B, C, L] with CFG combine / rescale (models/dit.py:338-347);
// cfg: yu[B*N_seq, ldy] holds the unconditional rows (y + B*N_seq*ldy in the batched CFG forward, or the other
// half's y in the CFG-split group forward)
int launch_dit_post(const float* y, const float* yu, int ldy, float* out, int B, int C, int L, int N_seq, int P, int cfg,
                    float cfg_scale, float scale_phi, cudaStream_t stream);
// generic fp32 -> 16-bit cast with row gather: dst[r, :] = src[perm ? perm[r] : r, :] * row_scale
int launch_cast_rows(const float* src, void* dst, const int* perm, int rows, int cols, int64_t src_ld, int64_t dst_ld,
                     bool bf16, cudaStream_t stream);
int launch_gather_f32(const float* src, float* dst, const int* perm, int n, cudaStream_t stream);
int launch_zero(void* p, size_t bytes, cudaStream_t stream);

// ---- kv_gather.cu (token-sharded DiT forward)
// kv [R, N, 2D] 16-bit = the k | v columns (D .. 3D - 1) of every rank's qkv [R, n_s, 3D], rank s's rows at tokens
// token_begin[s] .. token_begin[s + 1] - 1 of each item (N = token_begin[world]).  qkv[s] may live on another device
// (a peer pointer).
constexpr int kKvGatherMaxRanks = 8;
int launch_kv_gather(const void* const* qkv, const int* token_begin, int world, void* kv, int R, int D,
                     cudaStream_t stream);

// ---- time_gather.cu (time-sharded Oobleck decode / encode)
// out [rows, T] fp32: positions begin[q] .. begin[q + 1] - 1 of every row from rank q's src[q] [rows, src_len[q]],
// starting at its position src_off[q] (begin[0] = 0, begin[world] = T).  src[q] may live on another device (a peer
// pointer).
int launch_time_gather(const float* const* src, const int* src_len, const int* src_off, const int* begin, int world,
                       float* out, int rows, int T, cudaStream_t stream);

// ---- conformer.cu
// out16 = silu(LayerNorm(depthwise_conv17(g16))) per item of n_seq rows (zero padding at each item's ends, eps 1e-5):
// g16, out16 [items * n_seq, D] 16-bit; w fp32 [D][17]; gamma, beta [D] (beta may be null).  D <= kConformerMaxDim.
constexpr int kConformerMaxDim = 1536;
int launch_conformer_dwconv(const void* g16, const float* w, const float* gamma, const float* beta, void* out16,
                            int items, int n_seq, int D, bool bf16, cudaStream_t stream);
// C[M, N] = A[M, K] B[K, N], fp32 in and out, fp64 accumulation (weight folding).
int launch_matmul_f64(const float* A, const float* B, float* C, int M, int N, int K, cudaStream_t stream);

}  // namespace satb
