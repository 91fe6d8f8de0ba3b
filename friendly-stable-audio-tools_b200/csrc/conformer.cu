// The conformer branch of a TransformerBlock (reference models/transformer.py:557-591): the depthwise convolution over
// the token axis with the mid LayerNorm and SiLU fused into one pass, and the fp64 fold of the two pointwise maps
// before the GLU.  The GEMMs of the branch are instances the DiT forward already runs (csrc/dit.cu).
#include "common.cuh"
#include "kernels.h"
#include "ptx.cuh"

namespace satb {

namespace {

constexpr int kTaps = 17;   // depthwise_conv kernel_size (transformer.py:571)
constexpr int kPad = 8;     // its zero padding on each side

__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(smem)), "l"(gmem), "r"(valid ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all_but_one() { asm volatile("cp.async.wait_group 1;\n" ::: "memory"); }

// Row sums over the block: every thread has stored its T partial sums in part[j * nthreads + tid] (the caller); warp
// w adds the nthreads partials of rows w, w + nwarps, ... and writes fin(sum) to out[row].  Two block barriers.  The
// partials go through shared memory rather than registers because the taps and accumulators already hold most of the
// register file.
template <int T, class Fin>
__device__ __forceinline__ void block_rows(const float* part, float* out, int lane, int warp, int nthreads, Fin fin) {
  __syncthreads();
  for (int j = warp; j < T; j += nthreads >> 5) {
    float s = 0.f;
    for (int i = lane; i < nthreads; i += 32) s += part[j * nthreads + i];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[j] = fin(s);
  }
  __syncthreads();
}

// silu(mid_norm(depthwise_conv(g))) per item (transformer.py:583-586).  g, out: 16-bit [items * n_seq, D]; w: fp32
// [D][17] (the state dict's [D, 1, 17]); gamma, beta: [D] (beta may be null).
//
// One CTA walks a segment of chunks of T rows of one item; blockDim = D / 2 and thread t owns channels 2t, 2t + 1: its
// 34 taps live in registers for the whole segment, its 2 T conv outputs of the current chunk too.  Input rows stream
// through a ring of 2 T + 16 smem rows with 16-byte cp.async: chunk c reads rows [cT - 8, cT + T + 8) and, while it
// runs, the T rows that chunk c + 1 adds are in flight; rows outside [0, n_seq) are zero-filled (cp.async with a
// source size of 0), so the convolution never reads a neighbouring item.  Then the row mean and the variance about it
// (two passes over the registers, as layernorm_kernel, the partial sums reduced through shared memory), the affine
// map and SiLU, and one 4-byte store per row per thread (a warp writes 128 contiguous bytes).  Taps, gamma and beta are read before griddepcontrol.wait.
template <bool BF16, int T, int kMaxThreads>
__global__ void __launch_bounds__(kMaxThreads, 1) conformer_dwconv_ln_silu_kernel(
    const uint16_t* __restrict__ g, const float* __restrict__ w, const float* __restrict__ gamma,
    const float* __restrict__ beta, uint16_t* __restrict__ out, int n_seq, int D, int segs) {
  constexpr int kRing = 2 * T + 2 * kPad;
  extern __shared__ __align__(16) uint8_t conf_smem[];
  uint16_t* ring = reinterpret_cast<uint16_t*>(conf_smem);                 // [kRing][D]
  float* part = reinterpret_cast<float*>(ring + static_cast<size_t>(kRing) * D);   // [T][blockDim] row partial sums
  float* s_mean = part + static_cast<size_t>(T) * blockDim.x;                     // [T]
  float* s_rstd = s_mean + T;                                                     // [T]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x;
  const int c0 = 2 * tid;
  const int item = blockIdx.x / segs, seg = blockIdx.x - item * segs;
  const int nc = (n_seq + T - 1) / T;
  const int ch_begin = static_cast<int>(static_cast<long long>(seg) * nc / segs);
  const int ch_end = static_cast<int>(static_cast<long long>(seg + 1) * nc / segs);

  pdl_launch_dependents();
  float w0[kTaps], w1[kTaps];
#pragma unroll
  for (int k = 0; k < kTaps; ++k) {
    w0[k] = __ldg(w + c0 * kTaps + k);
    w1[k] = __ldg(w + (c0 + 1) * kTaps + k);
  }
  // gamma / beta: fetched into L1 here, read into registers per chunk where they are used (registers are scarce)
  asm volatile("prefetch.global.L1 [%0];" ::"l"(gamma + c0));
  if (beta) asm volatile("prefetch.global.L1 [%0];" ::"l"(beta + c0));
  pdl_wait();
  if (ch_begin >= ch_end) return;

  const size_t base = static_cast<size_t>(item) * n_seq * D;
  const uint16_t* src = g + base;
  uint16_t* dst = out + base;
  const int vpr = D >> 3;   // 16-byte pieces per row
  auto load_rows = [&](int r0, int r1) {   // item-relative rows [r0, r1) into their ring slots (r mod kRing)
    const int n = (r1 - r0) * vpr;
    for (int i = tid; i < n; i += blockDim.x) {
      const int rr = i / vpr, v = i - rr * vpr;
      const int r = r0 + rr;
      const bool ok = r >= 0 && r < n_seq;
      const int slot = (r + kRing) % kRing;
      cp_async16_zfill(ring + static_cast<size_t>(slot) * D + 8 * v, ok ? src + static_cast<size_t>(r) * D + 8 * v : src,
                       ok);
    }
  };
  load_rows(ch_begin * T - kPad, ch_begin * T + T + kPad);
  cp_async_commit();
  if (ch_begin + 1 < ch_end) load_rows(ch_begin * T + T + kPad, ch_begin * T + 2 * T + kPad);
  cp_async_commit();

  const float inv_d = 1.f / static_cast<float>(D);
  for (int c = ch_begin; c < ch_end; ++c) {
    const int r0 = c * T;
    cp_async_wait_all_but_one();
    __syncthreads();
    float a0[T], a1[T];
#pragma unroll
    for (int j = 0; j < T; ++j) a0[j] = a1[j] = 0.f;
    const int s0 = (r0 - kPad + kRing) % kRing;
#pragma unroll
    for (int i = 0; i < T + 2 * kPad; ++i) {   // window row i = item row r0 - 8 + i feeds outputs j = i - k
      const int s = s0 + i >= kRing ? s0 + i - kRing : s0 + i;
      const float2 x = Op16<BF16>::unpack(*reinterpret_cast<const uint32_t*>(ring + static_cast<size_t>(s) * D + c0));
#pragma unroll
      for (int k = 0; k < kTaps; ++k) {
        const int j = i - k;
        if (j >= 0 && j < T) {
          a0[j] = fmaf(w0[k], x.x, a0[j]);
          a1[j] = fmaf(w1[k], x.y, a1[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < T; ++j) part[j * nthreads + tid] = a0[j] + a1[j];
    block_rows<T>(part, s_mean, lane, warp, nthreads, [&](float s) { return s * inv_d; });
    // every thread is past its reads of rows [r0 - 8, r0 + T - 8): their slots take the rows chunk c + 2 adds
    if (c + 2 < ch_end) load_rows(r0 + 2 * T + kPad, r0 + 3 * T + kPad);
    cp_async_commit();
#pragma unroll
    for (int j = 0; j < T; ++j) {   // a0, a1 become the deviations from the row mean
      const float m = s_mean[j];
      a0[j] -= m;
      a1[j] -= m;
      part[j * nthreads + tid] = a0[j] * a0[j] + a1[j] * a1[j];
    }
    block_rows<T>(part, s_rstd, lane, warp, nthreads, [&](float s) { return rsqrtf(s * inv_d + 1e-5f); });
    const float2 ga = __ldg(reinterpret_cast<const float2*>(gamma) + tid);
    const float2 be = beta ? __ldg(reinterpret_cast<const float2*>(beta) + tid) : make_float2(0.f, 0.f);
#pragma unroll
    for (int j = 0; j < T; ++j) {
      const int r = r0 + j;
      if (r < n_seq) {
        const float rs = s_rstd[j];
        float y0 = a0[j] * rs * ga.x + be.x;
        float y1 = a1[j] * rs * ga.y + be.y;
        y0 = y0 / (1.f + expf(-y0));
        y1 = y1 / (1.f + expf(-y1));
        *reinterpret_cast<uint32_t*>(dst + static_cast<size_t>(r) * D + c0) = Op16<BF16>::pack(y0, y1);
      }
    }
  }
}

// C[M, N] = A[M, K] B[K, N] (fp32 row-major inputs and output) with fp64 products and accumulation; 64 x 64 tiles,
// 4 x 4 outputs per thread.  Runs once per layer when the weights are loaded.
__global__ void __launch_bounds__(256) matmul_f64_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                         float* __restrict__ C, int M, int N, int K) {
  __shared__ double As[16][64];
  __shared__ double Bs[16][64];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int am = i >> 4, ak = i & 15;
      As[ak][am] = (m0 + am < M && k0 + ak < K) ? A[static_cast<size_t>(m0 + am) * K + k0 + ak] : 0.0;
      const int bk = i >> 6, bn = i & 63;
      Bs[bk][bn] = (k0 + bk < K && n0 + bn < N) ? B[static_cast<size_t>(k0 + bk) * N + n0 + bn] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        a[i] = As[kk][ty + 16 * i];
        b[i] = Bs[kk][tx + 16 * i];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
      if (m < M && n < N) C[static_cast<size_t>(m) * N + n] = static_cast<float>(acc[i][j]);
    }
}

template <bool BF16, int T, int kMaxThreads>
int launch_dwconv_instance(const void* g16, const float* w, const float* gamma, const float* beta, void* out16,
                           int items, int n_seq, int D, cudaStream_t stream) {
  auto kern = conformer_dwconv_ln_silu_kernel<BF16, T, kMaxThreads>;
  const int threads = D / 2;
  const size_t smem = static_cast<size_t>(2 * T + 2 * kPad) * D * 2 + (static_cast<size_t>(threads) + 2) * T * sizeof(float);
  static PerDeviceOnce attr;
  static int occ_d[64] = {}, occ_v[64] = {};   // resident CTAs per SM, per device, for the last D seen there
  int dev = 0;
  cudaGetDevice(&dev);
  if (attr.first()) SATB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  int occ = 1;
  if (dev >= 0 && dev < 64 && occ_d[dev] == D) {
    occ = occ_v[dev];
  } else {
    SATB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
    if (occ < 1) occ = 1;
    if (dev >= 0 && dev < 64) { occ_d[dev] = D; occ_v[dev] = occ; }
  }
  // segments per item: as many as fill one wave of resident CTAs, chunks split evenly (differing by at most one)
  const int nc = ceil_div(n_seq, T);
  int segs = device_sm_count() * occ / items;
  if (segs < 1) segs = 1;
  if (segs > nc) segs = nc;
  SATB_CHECK_CUDA(launch_pdl(kern, dim3(items * segs), dim3(threads), smem, stream, static_cast<const uint16_t*>(g16), w,
                             gamma, beta, static_cast<uint16_t*>(out16), n_seq, D, segs));
  count_launch();
  return 0;
}

}  // namespace

int launch_conformer_dwconv(const void* g16, const float* w, const float* gamma, const float* beta, void* out16,
                            int items, int n_seq, int D, bool bf16, cudaStream_t stream) {
  SATB_REQUIRE(D % 128 == 0 && D >= 128 && D <= kConformerMaxDim,
               "conformer depthwise conv: D must be a multiple of 128 and <= 1536");
  SATB_REQUIRE(items >= 1 && n_seq >= 1, "conformer depthwise conv: empty input");
  // T = 12 rows per chunk, D / 2 <= 768 threads: 34 taps + 24 accumulators and the loop state fit the 80 registers
  // a thread of a 768-thread CTA can have without spilling (T = 16 spills)
  return bf16 ? launch_dwconv_instance<true, 12, 768>(g16, w, gamma, beta, out16, items, n_seq, D, stream)
              : launch_dwconv_instance<false, 12, 768>(g16, w, gamma, beta, out16, items, n_seq, D, stream);
}

int launch_matmul_f64(const float* A, const float* B, float* C, int M, int N, int K, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return 0;
  matmul_f64_kernel<<<dim3(ceil_div(N, 64), ceil_div(M, 64)), 256, 0, stream>>>(A, B, C, M, N, K);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace satb

extern "C" {

// Test entry point: the kernel the DiT forward launches for the conformer branch (see include/satb200.h).
int satb_conformer_dwconv(const void* g16, const float* w, const float* gamma, const float* beta, void* out16, int items,
                          int n_seq, int D, int bf16, void* stream) {
  SATB_REQUIRE(g16 && w && gamma && out16, "null argument");
  SATB_REQUIRE(((reinterpret_cast<uintptr_t>(g16) | reinterpret_cast<uintptr_t>(out16)) & 15) == 0 &&
                   ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 7) == 0,
               "conformer depthwise conv: g and out must be 16-byte aligned, gamma and beta 8-byte aligned");
  return satb::launch_conformer_dwconv(g16, w, gamma, beta, out16, items, n_seq, D, bf16 != 0,
                                       static_cast<cudaStream_t>(stream));
}

}  // extern "C"
