// Bandwidth-bound kernels of the DiT / Oobleck path: LayerNorm, SnakeBeta, layout
// changes around the transformer, timestep features, tiny conditioning MLPs, CFG.
// All fp32 math; 128-bit global accesses where the layout allows.
#include <cuda_fp8.h>

#include "common.cuh"
#include "fp8.cuh"
#include "kernels.h"
#include "ptx.cuh"

namespace satb {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ----------------------------------------------------------------- LayerNorm
// models/transformer.py:188-206 (F.layer_norm, eps 1e-5, learnable gamma, zero beta
// buffer) with the optional adaLN modulation of :670-672 / :683-684 folded in.
// One warp per row, the row lives in registers (two-pass mean / variance).
constexpr int kLnMaxVec = 16;  // D <= 16 * 128 = 2048

// NV = float4 per lane held in registers (D <= NV * 128).  The kernel is bound by memory-level parallelism
// (ncu: 12 long-scoreboard stalls per issue, 20 resident warps with the old 16-deep register array), so the
// array is sized to the actual row and the register count capped for 8 blocks = 32 rows in flight per SM.
template <bool BF16, int NV>
__global__ void __launch_bounds__(128, NV <= 8 ? 8 : (NV <= 12 ? 7 : 5)) layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, uint16_t* __restrict__ out,
                                                        int rows, int D, const float* __restrict__ scale,
                                                        const float* __restrict__ shift, int64_t mod_stride,
                                                        int rows_per_item, int n_items) {
  // gamma / beta never depend on the previous kernel: the block copies them to shared memory BEFORE the
  // programmatic-dependency wait (it is launched while the producer GEMM is still draining), so that after
  // the wait the critical path is only: row loads -> two warp reductions -> smem reads -> stores.
  extern __shared__ float4 ln_gb[];   // [D / 4] gamma, then [D / 4] beta (if any)
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int nv = D >> 7;  // float4 per lane
  pdl_launch_dependents();
  for (int i = threadIdx.x; i < (D >> 2); i += blockDim.x) {
    ln_gb[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i);
    if (beta) ln_gb[(D >> 2) + i] = __ldg(reinterpret_cast<const float4*>(beta) + i);
  }
  __syncthreads();
  pdl_wait();
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
  float4 v[NV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (i < nv) {
      v[i] = xr[lane + 32 * i];
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(D);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (i < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(D) + 1e-5f);
  const float4* g4 = ln_gb;
  const float4* b4 = beta ? ln_gb + (D >> 2) : nullptr;
  const float4* sc4 = nullptr;
  const float4* sh4 = nullptr;
  if (scale) {
    const int item = (row / rows_per_item) % n_items;
    sc4 = reinterpret_cast<const float4*>(scale + item * mod_stride);
    sh4 = reinterpret_cast<const float4*>(shift + item * mod_stride);
  }
  uint2* o2 = reinterpret_cast<uint2*>(out + static_cast<size_t>(row) * D);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (i < nv) {
      const int idx = lane + 32 * i;
      const float4 g = g4[idx];
      float4 y;
      y.x = (v[i].x - mean) * rstd * g.x;
      y.y = (v[i].y - mean) * rstd * g.y;
      y.z = (v[i].z - mean) * rstd * g.z;
      y.w = (v[i].w - mean) * rstd * g.w;
      if (b4) {
        const float4 b = b4[idx];
        y.x += b.x; y.y += b.y; y.z += b.z; y.w += b.w;
      }
      if (sc4) {
        const float4 s = __ldg(sc4 + idx), t = __ldg(sh4 + idx);
        y.x = y.x * (1.f + s.x) + t.x;
        y.y = y.y * (1.f + s.y) + t.y;
        y.z = y.z * (1.f + s.z) + t.z;
        y.w = y.w * (1.f + s.w) + t.w;
      }
      o2[idx] = make_uint2(Op16<BF16>::pack(y.x, y.y), Op16<BF16>::pack(y.z, y.w));
    }
  }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// layernorm_kernel with an e4m3 output: the same fp32 LayerNorm (and adaLN modulation) of the row held in registers,
// then its absolute maximum, the row scale (written to row_scale[row]) and the e4m3 row.  A separate kernel, so that
// the 16-bit one stays as it is.
template <int NV>
__global__ void __launch_bounds__(128, NV <= 8 ? 8 : (NV <= 12 ? 7 : 5)) layernorm_fp8_kernel(
    const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
    uint8_t* __restrict__ out, float* __restrict__ row_scale, int rows, int D, const float* __restrict__ scale,
    const float* __restrict__ shift, int64_t mod_stride, int rows_per_item, int n_items) {
  extern __shared__ float4 ln_gb[];   // [D / 4] gamma, then [D / 4] beta (if any)
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int nv = D >> 7;
  pdl_launch_dependents();
  for (int i = threadIdx.x; i < (D >> 2); i += blockDim.x) {
    ln_gb[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i);
    if (beta) ln_gb[(D >> 2) + i] = __ldg(reinterpret_cast<const float4*>(beta) + i);
  }
  __syncthreads();
  pdl_wait();
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
  float4 v[NV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (i < nv) {
      v[i] = xr[lane + 32 * i];
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(D);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (i < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(D) + 1e-5f);
  const float4* b4 = beta ? ln_gb + (D >> 2) : nullptr;
  const float4* sc4 = nullptr;
  const float4* sh4 = nullptr;
  if (scale) {
    const int item = (row / rows_per_item) % n_items;
    sc4 = reinterpret_cast<const float4*>(scale + item * mod_stride);
    sh4 = reinterpret_cast<const float4*>(shift + item * mod_stride);
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (i < nv) {
      const int idx = lane + 32 * i;
      const float4 g = ln_gb[idx];
      float4 y;
      y.x = (v[i].x - mean) * rstd * g.x;
      y.y = (v[i].y - mean) * rstd * g.y;
      y.z = (v[i].z - mean) * rstd * g.z;
      y.w = (v[i].w - mean) * rstd * g.w;
      if (b4) {
        const float4 b = b4[idx];
        y.x += b.x; y.y += b.y; y.z += b.z; y.w += b.w;
      }
      if (sc4) {
        const float4 s = __ldg(sc4 + idx), t = __ldg(sh4 + idx);
        y.x = y.x * (1.f + s.x) + t.x;
        y.y = y.y * (1.f + s.y) + t.y;
        y.z = y.z * (1.f + s.z) + t.z;
        y.w = y.w * (1.f + s.w) + t.w;
      }
      v[i] = y;
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(y.x), fabsf(y.y)), fmaxf(fabsf(y.z), fabsf(y.w))));
    }
  }
  const int e = fp8_row_exp(warp_max(amax));
  const float inv = pow2f(-e);
  if (lane == 0) row_scale[row] = pow2f(e);
  uint32_t* o4 = reinterpret_cast<uint32_t*>(out + static_cast<size_t>(row) * D);
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (i < nv) o4[lane + 32 * i] = e4m3x4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
}

// Weight rows -> e4m3 rows with their power-of-two scales (same rule), dst row r = src row perm[r]; one warp per row.
__global__ void __launch_bounds__(128) quant_rows_fp8_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst,
                                                             float* __restrict__ row_scale, const int* __restrict__ perm,
                                                             int rows, int cols) {
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float4* s4 = reinterpret_cast<const float4*>(src + static_cast<size_t>(perm ? perm[r] : r) * cols);
  float amax = 0.f;
  for (int i = lane; i < cols / 4; i += 32) {
    const float4 w = s4[i];
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(w.x), fabsf(w.y)), fmaxf(fabsf(w.z), fabsf(w.w))));
  }
  const int e = fp8_row_exp(warp_max(amax));
  const float inv = pow2f(-e);
  if (lane == 0) row_scale[r] = pow2f(e);
  uint32_t* d4 = reinterpret_cast<uint32_t*>(dst + static_cast<size_t>(r) * cols);
  for (int i = lane; i < cols / 4; i += 32) {
    const float4 w = s4[i];
    d4[i] = e4m3x4(w.x * inv, w.y * inv, w.z * inv, w.w * inv);
  }
}

// ----------------------------------------------------------------- SnakeBeta
// models/blocks.py:318-319,350-358: y = x + sin^2(x * e^alpha) / (e^beta + 1e-9).
__global__ void __launch_bounds__(256) snake_beta_kernel(const float* __restrict__ x, const float* __restrict__ alpha,
                                                         const float* __restrict__ beta, float* __restrict__ y, int C,
                                                         int64_t T, int logscale) {
  const int bc = blockIdx.y;
  const int c = bc % C;
  float a = __ldg(alpha + c), b = __ldg(beta + c);
  if (logscale) {
    a = expf(a);
    b = expf(b);
  }
  const float inv_b = 1.0f / (b + 0.000000001f);
  const float* xr = x + static_cast<size_t>(bc) * T;
  float* yr = y + static_cast<size_t>(bc) * T;
  const bool vec = (T % 4 == 0) && ((reinterpret_cast<uintptr_t>(xr) & 15) == 0) && ((reinterpret_cast<uintptr_t>(yr) & 15) == 0);
  if (vec) {
    const int64_t n4 = T >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(xr);
    float4* y4 = reinterpret_cast<float4*>(yr);
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
      float4 v = x4[i];
      float s;
      s = sinf(v.x * a); v.x = v.x + inv_b * (s * s);
      s = sinf(v.y * a); v.y = v.y + inv_b * (s * s);
      s = sinf(v.z * a); v.z = v.z + inv_b * (s * s);
      s = sinf(v.w * a); v.w = v.w + inv_b * (s * s);
      y4[i] = v;
    }
  } else {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < T;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
      const float v = xr[i];
      const float s = sinf(v * a);
      yr[i] = v + inv_b * (s * s);
    }
  }
}

// ------------------------------------------------------------------ DiT pre
// NCL fp32 latent -> token-major 16-bit rows [R*N_seq, lda]; the P leading rows of every
// item (the prepend slots) are zero so the project_in GEMM leaves them 0.  Columns C .. lda-1
// (the row pitch padded up to 16 bytes for TMA) are written as zeros on every call too, so the
// zero-padded K of project_in never reads stale memory.
template <bool BF16>
__global__ void __launch_bounds__(256) dit_pre_kernel(const float* __restrict__ x, uint16_t* __restrict__ a, int B_src,
                                                      int C, int lda, int L, int P) {
  __shared__ float tile[32][33];
  const int r = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const float* xs = x + static_cast<size_t>(r % B_src) * C * L;
  const int N_seq = L + P;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, l = l0 + tx;
    tile[j][tx] = (c < C && l < L) ? xs[static_cast<size_t>(c) * L + l] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int l = l0 + j, c = c0 + tx;
    if (l < L && c < lda)
    {
      typename Op16<BF16>::T hv = Op16<BF16>::from_float(tile[tx][j]);   // tile holds 0 for c >= C
      a[(static_cast<size_t>(r) * N_seq + P + l) * lda + c] = *reinterpret_cast<uint16_t*>(&hv);
    }
  }
  if (blockIdx.x == 0 && P > 0) {
    for (int j = ty; j < P; j += 8) {
      const int c = c0 + tx;
      if (c < lda) a[(static_cast<size_t>(r) * N_seq + j) * lda + c] = 0;
    }
  }
}

// --------------------------------------------------------- timestep features
// models/blocks.py:95-97: f = (2*pi*t) * w (fp32), out = [cos f | sin f].
__global__ void fourier_kernel(const float* __restrict__ t, const float* __restrict__ w, float* __restrict__ out, int B,
                               int F) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * F) return;
  const int b = i / F, j = i - b * F;
  const float tt = 6.283185307179586f * t[b];
  const float f = tt * w[j];
  out[static_cast<size_t>(b) * 2 * F + j] = cosf(f);
  out[static_cast<size_t>(b) * 2 * F + F + j] = sinf(f);
}

// --------------------------------------------------------------- skinny GEMM
// Tiny-M linear layers (timestep / global embedding MLPs, adaLN projections):
// one warp per output column, fp32 weights and accumulation, up to 8 rows per pass.
__device__ __forceinline__ float silu_acc(float x) { return x / (1.0f + expf(-x)); }

// The (at most 8) input rows of a pass are staged in shared memory once per block; every lane then has all
// its weight loads (K / 128 float4, <= 16) in flight at once instead of a 4-deep loop, which is what made
// the 1536 x 1536 timestep-embedding layer latency-bound (96 us under ncu for 9.4 MB of weights).
constexpr int kSkinnyMaxVec = 16;   // K <= 16 * 128 = 2048 per fast pass; larger K falls back to the loop

__global__ void __launch_bounds__(256) skinny_linear_kernel(const float* __restrict__ in, const float* __restrict__ W,
                                                            const float* __restrict__ bias,
                                                            const float* __restrict__ add, float* __restrict__ out,
                                                            int R, int K, int N, int silu_out) {
  extern __shared__ float4 xs4[];   // [8][K / 4]
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int k4n = K >> 2;
  const bool col_ok = n < N;
  const float4* wr = reinterpret_cast<const float4*>(W + static_cast<size_t>(col_ok ? n : 0) * K);
  float4 w[kSkinnyMaxVec];
  const bool fast = k4n <= kSkinnyMaxVec * 32;
  if (fast) {
#pragma unroll
    for (int i = 0; i < kSkinnyMaxVec; ++i)
      w[i] = (col_ok && lane + 32 * i < k4n) ? __ldg(wr + lane + 32 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int r0 = 0; r0 < R; r0 += 8) {
    const int rows = R - r0 < 8 ? R - r0 : 8;
    __syncthreads();
    for (int i = threadIdx.x; i < rows * k4n; i += blockDim.x)
      xs4[i] = __ldg(reinterpret_cast<const float4*>(in + static_cast<size_t>(r0) * K) + i);
    __syncthreads();
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (fast) {
#pragma unroll
      for (int i = 0; i < kSkinnyMaxVec; ++i) {
        const int k4 = lane + 32 * i;
        if (k4 < k4n) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (j < rows) {
              const float4 x = xs4[j * k4n + k4];
              acc[j] = fmaf(x.x, w[i].x, fmaf(x.y, w[i].y, fmaf(x.z, w[i].z, fmaf(x.w, w[i].w, acc[j]))));
            }
          }
        }
      }
    } else {
      for (int k4 = lane; k4 < k4n; k4 += 32) {
        const float4 wv = col_ok ? __ldg(wr + k4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (j < rows) {
            const float4 x = xs4[j * k4n + k4];
            acc[j] = fmaf(x.x, wv.x, fmaf(x.y, wv.y, fmaf(x.z, wv.z, fmaf(x.w, wv.w, acc[j]))));
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float s = warp_sum(acc[j]);
      if (lane == 0 && col_ok && j < rows) {
        float v = s + (bias ? bias[n] : 0.f);
        if (add) v += add[static_cast<size_t>(r0 + j) * N + n];
        if (silu_out) v = silu_acc(v);
        out[static_cast<size_t>(r0 + j) * N + n] = v;
      }
    }
  }
}

// rows 0 .. Pp-1 of every item: the prepend-conditioning tokens (conditional rows r < B; zeros for the unconditional CFG
// rows, dit.py:309-311); row Pp: the global-conditioning token (dit.py:185-195).  pos (may be null): the positional
// embedding table [N_seq, D]; row j gets pos[j] added, as the reference adds it after the prepend concat
// (transformer.py:770-785).
__global__ void write_prepend_kernel(const float* __restrict__ tok, const float* __restrict__ pre,
                                     const float* __restrict__ pos, float* __restrict__ h, int B, int N_seq, int D, int Pp) {
  const int r = blockIdx.y, j = blockIdx.z;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  float v;
  if (j < Pp) v = (r < B && pre) ? pre[(static_cast<size_t>(r) * Pp + j) * D + d] : 0.f;
  else v = tok[static_cast<size_t>(r % B) * D + d];
  if (pos) v += pos[static_cast<size_t>(j) * D + d];
  h[(static_cast<size_t>(r) * N_seq + j) * D + d] = v;
}

__global__ void gate_sigmoid_kernel(float* __restrict__ ssg, int depth, int D) {
  // ssg: [rows, depth*6D]; transform gate columns (chunks 2 and 5 of every layer) to sigmoid(1 - g)
  const int row = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over depth * 2 * D
  if (i >= depth * 2 * D) return;
  const int layer = i / (2 * D), rem = i - layer * 2 * D;
  const int which = rem / D, d = rem - which * D;
  float* p = ssg + static_cast<size_t>(row) * depth * 6 * D + static_cast<size_t>(layer) * 6 * D + (which ? 5 : 2) * D + d;
  *p = 1.0f / (1.0f + expf(-(1.0f - *p)));
}

// ------------------------------------------------------------------ DiT post
// models/dit.py:219 (drop prepend), :338-347 (CFG combine, std rescale over channels).
// y rows are token-major [R*N_seq, ldy] (ldy >= C: project_out's N padded up to its store width; only the C real
// channels are read); one thread per (b, l).  yu: the unconditional rows [B*N_seq, ldy] of the CFG combine (read only
// when cfg): y + B*N_seq*ldy when both halves are in y, or the unconditional half's own y (a peer pointer allowed).  C = 1 with scale_phi != 0 gives NaN, as torch.std (unbiased) of one
// channel does in the reference.
__global__ void __launch_bounds__(128) dit_post_kernel(const float* __restrict__ y, const float* __restrict__ yu_rows,
                                                       int ldy, float* __restrict__ out, int B, int C, int L, int N_seq,
                                                       int P, int cfg, float cfg_scale, float scale_phi) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (l >= L) return;
  const float* yc = y + (static_cast<size_t>(b) * N_seq + P + l) * ldy;
  float* o = out + static_cast<size_t>(b) * C * L + l;
  if (!cfg) {
    for (int c = 0; c < C; ++c) o[static_cast<size_t>(c) * L] = yc[c];
    return;
  }
  const float* yu = yu_rows + (static_cast<size_t>(b) * N_seq + P + l) * ldy;
  if (scale_phi == 0.f) {
    for (int c = 0; c < C; ++c) {
      const float cv = yc[c], uv = yu[c];
      o[static_cast<size_t>(c) * L] = uv + (cv - uv) * cfg_scale;
    }
    return;
  }
  // unbiased std over the channel dim of cond and of the cfg output (torch.std default)
  float s1 = 0.f, s2 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float cv = yc[c], uv = yu[c];
    s1 += cv;
    s2 += uv + (cv - uv) * cfg_scale;
  }
  const float m1 = s1 / C, m2 = s2 / C;
  float v1 = 0.f, v2 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float cv = yc[c], uv = yu[c];
    const float g = uv + (cv - uv) * cfg_scale;
    v1 += (cv - m1) * (cv - m1);
    v2 += (g - m2) * (g - m2);
  }
  const float ratio = sqrtf(v1 / (C - 1)) / sqrtf(v2 / (C - 1));
  for (int c = 0; c < C; ++c) {
    const float cv = yc[c], uv = yu[c];
    const float g = uv + (cv - uv) * cfg_scale;
    o[static_cast<size_t>(c) * L] = scale_phi * (g * ratio) + (1.f - scale_phi) * g;
  }
}

// ----------------------------------------------------------------- weight prep
template <bool BF16>
__global__ void cast_rows_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, const int* __restrict__ perm,
                                 int rows, int cols, int64_t src_ld, int64_t dst_ld) {
  const int r = blockIdx.y;
  const int sr = perm ? perm[r] : r;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < cols; c += gridDim.x * blockDim.x) {
    typename Op16<BF16>::T h = Op16<BF16>::from_float(src[static_cast<size_t>(sr) * src_ld + c]);
    dst[static_cast<size_t>(r) * dst_ld + c] = *reinterpret_cast<uint16_t*>(&h);
  }
}

__global__ void gather_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ perm,
                                  int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[perm ? perm[i] : i];
}

}  // namespace

int launch_layernorm(const float* x, const float* gamma, const float* beta, void* out16, int rows, int D,
                     const float* scale, const float* shift, int64_t mod_stride, int rows_per_item, int n_items,
                     bool bf16, cudaStream_t stream) {
  SATB_REQUIRE(D % 128 == 0 && D <= kLnMaxVec * 128, "LayerNorm width must be a multiple of 128 and <= 2048");
  if (rows <= 0) return 0;
  const int grid = ceil_div(rows, 4);
  const int items = n_items > 0 ? n_items : 1;
  const int nv = D >> 7;
  auto go = [&](auto kern) -> int {
    SATB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(128), static_cast<size_t>(D) * 8, stream, x, gamma, beta,
                               static_cast<uint16_t*>(out16), rows, D, scale, shift, mod_stride, rows_per_item, items));
    return 0;
  };
  int rc;
  if (bf16)
    rc = nv <= 4 ? go(layernorm_kernel<true, 4>) : nv <= 8 ? go(layernorm_kernel<true, 8>)
         : nv <= 12 ? go(layernorm_kernel<true, 12>) : go(layernorm_kernel<true, 16>);
  else
    rc = nv <= 4 ? go(layernorm_kernel<false, 4>) : nv <= 8 ? go(layernorm_kernel<false, 8>)
         : nv <= 12 ? go(layernorm_kernel<false, 12>) : go(layernorm_kernel<false, 16>);
  SATB_PROPAGATE(rc);
  count_launch();
  return 0;
}

int launch_layernorm_fp8(const float* x, const float* gamma, const float* beta, void* out8, float* row_scale, int rows,
                         int D, const float* scale, const float* shift, int64_t mod_stride, int rows_per_item,
                         int n_items, cudaStream_t stream) {
  SATB_REQUIRE(D % 128 == 0 && D <= kLnMaxVec * 128, "LayerNorm width must be a multiple of 128 and <= 2048");
  if (rows <= 0) return 0;
  const int grid = ceil_div(rows, 4);
  const int items = n_items > 0 ? n_items : 1;
  const int nv = D >> 7;
  auto go = [&](auto kern) -> int {
    SATB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(128), static_cast<size_t>(D) * 8, stream, x, gamma, beta,
                               static_cast<uint8_t*>(out8), row_scale, rows, D, scale, shift, mod_stride, rows_per_item,
                               items));
    return 0;
  };
  SATB_PROPAGATE(nv <= 4 ? go(layernorm_fp8_kernel<4>) : nv <= 8 ? go(layernorm_fp8_kernel<8>)
                 : nv <= 12 ? go(layernorm_fp8_kernel<12>) : go(layernorm_fp8_kernel<16>));
  count_launch();
  return 0;
}

int launch_quant_rows_fp8(const float* src, void* dst, float* row_scale, const int* perm, int rows, int cols,
                          cudaStream_t stream) {
  SATB_REQUIRE(cols % 4 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0,
               "FP8 row quantisation: cols must be a multiple of 4 and src 16-byte aligned");
  if (rows <= 0) return 0;
  quant_rows_fp8_kernel<<<ceil_div(rows, 4), 128, 0, stream>>>(src, static_cast<uint8_t*>(dst), row_scale, perm, rows,
                                                                cols);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// One sampler step of the v-objective k-diffusion samplers as a single pass (inference/sampling.py:
// VDenoiser scalings + the DPM-Solver++ multistep update + noise injection are all linear in the tensors):
//   den    = c_out * v + c_skip * x                      (VDenoiser.forward)
//   x_next = A x + B den + C den_1 + D den_2 + S noise   (scalars from the host-side step-size algebra)
//   x_in   = x_next * c_in_next                          (the next model call's input)
// den_1 / den_2 / noise may be null (their coefficient is then ignored).
__global__ void __launch_bounds__(256) sampler_update_kernel(const float4* __restrict__ x, const float4* __restrict__ v,
                                                             const float4* __restrict__ d1, const float4* __restrict__ d2,
                                                             const float4* __restrict__ nz, float4* __restrict__ den,
                                                             float4* __restrict__ x_next, float4* __restrict__ x_in,
                                                             long long n4, float c_skip, float c_out, float A, float B,
                                                             float C, float D, float S, float c_in_next) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 xv = x[i], vv = v[i];
    float4 dn = make_float4(fmaf(c_out, vv.x, c_skip * xv.x), fmaf(c_out, vv.y, c_skip * xv.y),
                            fmaf(c_out, vv.z, c_skip * xv.z), fmaf(c_out, vv.w, c_skip * xv.w));
    float4 o = make_float4(fmaf(A, xv.x, B * dn.x), fmaf(A, xv.y, B * dn.y), fmaf(A, xv.z, B * dn.z),
                           fmaf(A, xv.w, B * dn.w));
    if (d1) {
      const float4 t = d1[i];
      o.x = fmaf(C, t.x, o.x); o.y = fmaf(C, t.y, o.y); o.z = fmaf(C, t.z, o.z); o.w = fmaf(C, t.w, o.w);
    }
    if (d2) {
      const float4 t = d2[i];
      o.x = fmaf(D, t.x, o.x); o.y = fmaf(D, t.y, o.y); o.z = fmaf(D, t.z, o.z); o.w = fmaf(D, t.w, o.w);
    }
    if (nz) {
      const float4 t = nz[i];
      o.x = fmaf(S, t.x, o.x); o.y = fmaf(S, t.y, o.y); o.z = fmaf(S, t.z, o.z); o.w = fmaf(S, t.w, o.w);
    }
    den[i] = dn;
    x_next[i] = o;
    if (x_in) x_in[i] = make_float4(o.x * c_in_next, o.y * c_in_next, o.z * c_in_next, o.w * c_in_next);
  }
}

int launch_sampler_update(const float* x, const float* v, const float* d1, const float* d2, const float* nz, float* den,
                          float* x_next, float* x_in, long long n, float c_skip, float c_out, float A, float B, float C,
                          float D, float S, float c_in_next, cudaStream_t stream) {
  SATB_REQUIRE(n > 0 && n % 4 == 0, "sampler update: element count must be a positive multiple of 4");
  const long long n4 = n / 4;
  int grid = static_cast<int>(ceil_div64(n4, 256));
  if (grid > 4 * device_sm_count()) grid = 4 * device_sm_count();
  SATB_CHECK_CUDA(launch_pdl(sampler_update_kernel, dim3(grid), dim3(256), 0, stream, reinterpret_cast<const float4*>(x),
                             reinterpret_cast<const float4*>(v), reinterpret_cast<const float4*>(d1),
                             reinterpret_cast<const float4*>(d2), reinterpret_cast<const float4*>(nz),
                             reinterpret_cast<float4*>(den), reinterpret_cast<float4*>(x_next),
                             reinterpret_cast<float4*>(x_in), n4, c_skip, c_out, A, B, C, D, S, c_in_next));
  count_launch();
  return 0;
}

// One step of the v-diffusion DDIM sampler (reference inference/sampling.py:64-118) as a single pass over the state:
//   pred = x alpha - v sigma;  eps = x sigma + v alpha;  x_next = pred alpha_next + eps adj_sigma (+ noise ddim_sigma)
// Every product and sum is rounded on its own (the _rn intrinsics keep nvcc from contracting them into FMAs), in the
// order of the reference's fp32 tensor expressions, so a step equals their torch evaluation bit for bit.  pred and
// x_next may each be null (the last step writes pred only); noise may be null.
__global__ void __launch_bounds__(256) vdiffusion_update_kernel(const float* __restrict__ x, const float* __restrict__ v,
                                                                const float* __restrict__ nz, float* __restrict__ x_next,
                                                                float* __restrict__ pred, long long n, float alpha,
                                                                float sigma, float alpha_next, float adj_sigma,
                                                                float ddim_sigma) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xv = x[i], vv = v[i];
    const float p = __fsub_rn(__fmul_rn(xv, alpha), __fmul_rn(vv, sigma));
    if (pred) pred[i] = p;
    if (x_next) {
      const float e = __fadd_rn(__fmul_rn(xv, sigma), __fmul_rn(vv, alpha));
      float o = __fadd_rn(__fmul_rn(p, alpha_next), __fmul_rn(e, adj_sigma));
      if (nz) o = __fadd_rn(o, __fmul_rn(nz[i], ddim_sigma));
      x_next[i] = o;
    }
  }
}

int launch_vdiffusion_update(const float* x, const float* v, const float* nz, float* x_next, float* pred, long long n,
                             float alpha, float sigma, float alpha_next, float adj_sigma, float ddim_sigma,
                             cudaStream_t stream) {
  SATB_REQUIRE(n > 0, "v-diffusion update: element count must be positive");
  int grid = static_cast<int>(ceil_div64(n, 256));
  if (grid > 4 * device_sm_count()) grid = 4 * device_sm_count();
  SATB_CHECK_CUDA(launch_pdl(vdiffusion_update_kernel, dim3(grid), dim3(256), 0, stream, x, v, nz, x_next, pred, n, alpha,
                             sigma, alpha_next, adj_sigma, ddim_sigma));
  count_launch();
  return 0;
}

int launch_snake_beta(const float* x, const float* alpha, const float* beta, float* y, int B, int C, int64_t T,
                      int logscale, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || T <= 0) return 0;
  SATB_REQUIRE(static_cast<int64_t>(B) * C <= 65535, "snake: B*C exceeds grid.y limit");
  int64_t per_block = 256 * 4 * 4;
  int gx = static_cast<int>(ceil_div64(T, per_block));
  if (gx < 1) gx = 1;
  dim3 grid(gx, B * C);
  snake_beta_kernel<<<grid, 256, 0, stream>>>(x, alpha, beta, y, C, T, logscale);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_dit_pre(const float* x, void* a16, int R, int B_src, int C, int lda, int L, int P, bool bf16,
                   cudaStream_t stream) {
  SATB_REQUIRE(lda >= C, "dit_pre: the row pitch must cover the channels");
  dim3 grid(ceil_div(L, 32), ceil_div(lda, 32), R);
  if (bf16)
    dit_pre_kernel<true><<<grid, 256, 0, stream>>>(x, static_cast<uint16_t*>(a16), B_src, C, lda, L, P);
  else
    dit_pre_kernel<false><<<grid, 256, 0, stream>>>(x, static_cast<uint16_t*>(a16), B_src, C, lda, L, P);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_fourier(const float* t, const float* w, float* out, int B, int F, cudaStream_t stream) {
  fourier_kernel<<<ceil_div(B * F, 128), 128, 0, stream>>>(t, w, out, B, F);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_skinny_linear(const float* in, const float* W, const float* bias, const float* add, float* out, int R,
                         int K, int N, int silu_out, cudaStream_t stream) {
  SATB_REQUIRE(R >= 1 && R <= 4096, "skinny linear: bad row count");
  SATB_REQUIRE(K % 4 == 0, "skinny linear: K must be a multiple of 4");
  const size_t smem = static_cast<size_t>(8) * K * sizeof(float);
  SATB_REQUIRE(smem <= 200 * 1024, "skinny linear: K too large for the shared-memory row stage");
  static PerDeviceOnce attr;
  if (attr.first()) SATB_CHECK_CUDA(cudaFuncSetAttribute(skinny_linear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  skinny_linear_kernel<<<ceil_div(N, 8), 256, smem, stream>>>(in, W, bias, add, out, R, K, N, silu_out);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_write_prepend(const float* tok, const float* pre, const float* pos, float* h, int R, int B, int N_seq, int D,
                         int Pp, cudaStream_t stream) {
  dim3 grid(ceil_div(D, 256), R, Pp + 1);
  write_prepend_kernel<<<grid, 256, 0, stream>>>(tok, pre, pos, h, B, N_seq, D, Pp);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_gate_sigmoid(float* ssg, int rows, int depth, int D, cudaStream_t stream) {
  dim3 grid(ceil_div(depth * 2 * D, 256), rows);
  gate_sigmoid_kernel<<<grid, 256, 0, stream>>>(ssg, depth, D);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_dit_post(const float* y, const float* yu, int ldy, float* out, int B, int C, int L, int N_seq, int P, int cfg,
                    float cfg_scale, float scale_phi, cudaStream_t stream) {
  SATB_REQUIRE(ldy >= C, "dit_post: the row pitch must cover the channels");
  SATB_REQUIRE(!cfg || yu, "dit_post: the CFG combine needs the unconditional rows");
  dim3 grid(ceil_div(L, 128), B);
  dit_post_kernel<<<grid, 128, 0, stream>>>(y, yu, ldy, out, B, C, L, N_seq, P, cfg, cfg_scale, scale_phi);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_cast_rows(const float* src, void* dst, const int* perm, int rows, int cols, int64_t src_ld, int64_t dst_ld,
                     bool bf16, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return 0;
  int gx = ceil_div(cols, 256);
  if (gx > 64) gx = 64;
  for (int r0 = 0; r0 < rows; r0 += 65535) {
    const int nr = rows - r0 < 65535 ? rows - r0 : 65535;
    dim3 grid(gx, nr);
    const float* s = perm ? src : src + static_cast<size_t>(r0) * src_ld;
    uint16_t* d = static_cast<uint16_t*>(dst) + static_cast<size_t>(r0) * dst_ld;
    const int* pm = perm ? perm + r0 : nullptr;
    if (bf16)
      cast_rows_kernel<true><<<grid, 256, 0, stream>>>(s, d, pm, nr, cols, src_ld, dst_ld);
    else
      cast_rows_kernel<false><<<grid, 256, 0, stream>>>(s, d, pm, nr, cols, src_ld, dst_ld);
    count_launch();
  }
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_gather_f32(const float* src, float* dst, const int* perm, int n, cudaStream_t stream) {
  if (n <= 0) return 0;
  gather_f32_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(src, dst, perm, n);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_zero(void* p, size_t bytes, cudaStream_t stream) {
  SATB_CHECK_CUDA(cudaMemsetAsync(p, 0, bytes, stream));
  return 0;
}

}  // namespace satb
