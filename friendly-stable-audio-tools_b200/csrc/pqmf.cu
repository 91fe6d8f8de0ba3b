// PQMF filterbank (reference models/pqmf.py, the "pqmf" pretransform of models/pretransforms.py:114-133): polyphase
// analysis (audio -> num_bands critically sampled sub-bands) and synthesis (sub-bands -> audio) in fp32 FMA on the
// CUDA cores.  The reference runs the pretransform in fp32 on raw audio; the work is `taps` MACs per sample, small
// next to the Oobleck convolutions around it, so tensor cores are not used.
//
// With n bands, a [n, F] filter bank h (F = taps, m = F / n taps per polyphase row, m even) and Tn = ceil(T / n) frames,
// the reference's pad_signal -> polyphase_analysis -> apply_alias_cancellation is
//   Y[k, t] = s(k, t) * sum_{p < n} sum_{j < m} h_k[j n + p] x[(t + j - m/2) n + p]        (x zero outside [0, T))
// and apply_alias_cancellation -> polyphase_synthesis (flipped bank, padding m/2 + 1, x n, phase flip, interleave, first
// 2n samples dropped) is, for the Tn * n output samples,
//   out[t n + p] = n * sum_{k < n} sum_{j < m} h_k[j n + p] s(k, t + m/2 - j) Y[k, t + m/2 - j]  (Y zero outside [0, Tn))
// where s(k, t) = -1 for odd k and even t, else 1.  Both are one kernel shape,
//   Z[q, t] = sum_r sum_j W[r][j][q] in(r, t + D - j),
// with W and D per direction (pqmf_prep_kernel builds both W at load time, the factor n folded into the synthesis W).
// The sign s depends on the frame parity as well as the band, so it is applied where the value is touched: on the
// analysis store and on the synthesis input load, not as a pass of its own.
#include <algorithm>
#include <string>

#include "../../include/satb200.h"
#include "common.cuh"
#include "ptx.cuh"

namespace satb {
namespace {

constexpr int kPqmfThreads = 256;
constexpr int kPqmfFrames = 8;            // output frames per thread (strided by G, the frame groups of a block)
constexpr int kPqmfWFloats = 16384;       // filter elements staged per chunk of input rows (64 KB)
constexpr int kPqmfMaxTaps = 16384;
constexpr int kPqmfMaxBands = 256;

// Wa[r][j][q] = h_q[(m - 1 - j) n + r]   (analysis: rows r are input phases, q output bands)
// Ws[r][j][q] = n * h_r[j n + q]         (synthesis: rows r are input bands, q output phases)
__global__ void pqmf_prep_kernel(const float* __restrict__ h, float* __restrict__ wa, float* __restrict__ ws, int n,
                                 int m) {
  const int total = n * m * n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int q = i % n, j = (i / n) % m, r = i / (n * m);
    const int F = n * m;
    wa[i] = h[static_cast<size_t>(q) * F + (m - 1 - j) * n + r];
    ws[i] = static_cast<float>(n) * h[static_cast<size_t>(r) * F + j * n + q];
  }
}

// One block: one (batch item, channel) and TT = G * kPqmfFrames consecutive frames, all n output rows q.  Thread
// (g, qg) = (tid % G, tid / G) owns rows q0 .. q0 + QT - 1 and frames t0 + g + G i.  The input rows are consumed in
// chunks of RC: their W block [RC][m][n] and their input window [RC][TT + m - 1] are staged in shared memory.
//   MODE 0 (analysis): in  = audio x [B*C, T];  out = bands [B*C, n, Tn] with the alias sign; D = m/2 - 1
//   MODE 1 (synthesis): in = bands [B*C, n, Tn] with the alias sign;  out = audio [B*C, Tn * n];  D = m/2
template <int MODE, int QT>
__global__ void __launch_bounds__(kPqmfThreads) pqmf_kernel(const float* __restrict__ in, const float* __restrict__ W,
                                                            float* __restrict__ out, int n, int m, int RC, int G,
                                                            long long T, int Tn) {
  extern __shared__ __align__(16) float pq_smem[];
  const int TT = G * kPqmfFrames, span = TT + m - 1;
  float* w_s = pq_smem;                                // [RC][m][n]
  float* in_s = pq_smem + static_cast<size_t>(RC) * m * n;   // [RC][span]
  const int tid = threadIdx.x, g = tid % G, q0 = (tid / G) * QT;
  const long long bc = blockIdx.y;
  const int t0 = blockIdx.x * TT;
  const int D = MODE == 0 ? m / 2 - 1 : m / 2;
  const long long tau0 = static_cast<long long>(t0) + D - (m - 1);
  pdl_wait();
  float acc[QT][kPqmfFrames];
#pragma unroll
  for (int a = 0; a < QT; ++a)
#pragma unroll
    for (int i = 0; i < kPqmfFrames; ++i) acc[a][i] = 0.f;

  for (int r0 = 0; r0 < n; r0 += RC) {
    __syncthreads();   // the previous chunk has been consumed
    {
      const float4* src = reinterpret_cast<const float4*>(W + static_cast<size_t>(r0) * m * n);
      float4* dst = reinterpret_cast<float4*>(w_s);
      const int n4 = RC * m * n / 4;
      for (int i = tid; i < n4; i += kPqmfThreads) dst[i] = __ldg(src + i);
    }
    if (MODE == 0) {
      // input phase r, frame tau: x[tau n + r]; r fastest so that consecutive threads read consecutive samples
      const float* xb = in + bc * T;
      for (int i = tid; i < RC * span; i += kPqmfThreads) {
        const int rl = i % RC, tl = i / RC;
        const long long pos = (tau0 + tl) * n + r0 + rl;
        in_s[rl * span + tl] = (pos >= 0 && pos < T) ? __ldg(xb + pos) : 0.f;
      }
    } else {
      for (int i = tid; i < RC * span; i += kPqmfThreads) {
        const int rl = i / span, tl = i - rl * span;
        const long long tau = tau0 + tl;
        const int k = r0 + rl;
        float v = 0.f;
        if (tau >= 0 && tau < Tn) {
          v = __ldg(in + (bc * n + k) * Tn + tau);
          if ((k & 1) && !(tau & 1)) v = -v;
        }
        in_s[i] = v;
      }
    }
    __syncthreads();
    for (int rl = 0; rl < RC; ++rl) {
      const float* wr = w_s + static_cast<size_t>(rl) * m * n + q0;
      const float* xr = in_s + rl * span + g + m - 1;
#pragma unroll 4
      for (int j = 0; j < m; ++j) {
        float w[QT];
        if constexpr (QT == 4) {
          const float4 v = *reinterpret_cast<const float4*>(wr + j * n);
          w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
        } else {
          const float2 v = *reinterpret_cast<const float2*>(wr + j * n);
          w[0] = v.x; w[1] = v.y;
        }
#pragma unroll
        for (int i = 0; i < kPqmfFrames; ++i) {
          const float xv = xr[G * i - j];
#pragma unroll
          for (int a = 0; a < QT; ++a) acc[a][i] = fmaf(w[a], xv, acc[a][i]);
        }
      }
    }
  }
  pdl_launch_dependents();
#pragma unroll
  for (int i = 0; i < kPqmfFrames; ++i) {
    const int t = t0 + g + G * i;
    if (t >= Tn) continue;
    if (MODE == 0) {
#pragma unroll
      for (int a = 0; a < QT; ++a) {
        const int q = q0 + a;
        out[(bc * n + q) * Tn + t] = ((q & 1) && !(t & 1)) ? -acc[a][i] : acc[a][i];
      }
    } else {
      float* o = out + bc * Tn * n + static_cast<long long>(t) * n + q0;
      if constexpr (QT == 4)
        *reinterpret_cast<float4*>(o) = make_float4(acc[0][i], acc[1][i], acc[2][i], acc[3][i]);
      else
        *reinterpret_cast<float2*>(o) = make_float2(acc[0][i], acc[1][i]);
    }
  }
}

struct PqmfLaunch {
  int QT, G, RC;
  size_t smem;
};

PqmfLaunch pqmf_plan(int n, int taps) {
  const int m = taps / n;
  PqmfLaunch p;
  p.QT = n >= 4 ? 4 : 2;
  p.G = kPqmfThreads * p.QT / n;
  p.RC = 1;
  while (p.RC * 2 <= n && p.RC * 2 * taps <= kPqmfWFloats) p.RC *= 2;
  p.smem = (static_cast<size_t>(p.RC) * taps + static_cast<size_t>(p.RC) * (p.G * kPqmfFrames + m - 1)) * 4;
  return p;
}

template <int MODE>
int launch_pqmf(const float* in, const float* W, float* out, int n, int taps, long long T, int Tn, int BC,
                cudaStream_t st) {
  const PqmfLaunch p = pqmf_plan(n, taps);
  const int m = taps / n;
  const dim3 grid(static_cast<unsigned>(ceil_div(Tn, p.G * kPqmfFrames)), static_cast<unsigned>(BC));
  if (p.QT == 4) {
    static PerDeviceOnce attr;
    if (attr.first())
      SATB_CHECK_CUDA(cudaFuncSetAttribute(pqmf_kernel<MODE, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    SATB_CHECK_CUDA(launch_pdl(pqmf_kernel<MODE, 4>, grid, dim3(kPqmfThreads), p.smem, st, in, W, out, n, m, p.RC, p.G,
                               T, Tn));
  } else {
    static PerDeviceOnce attr;
    if (attr.first())
      SATB_CHECK_CUDA(cudaFuncSetAttribute(pqmf_kernel<MODE, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    SATB_CHECK_CUDA(launch_pdl(pqmf_kernel<MODE, 2>, grid, dim3(kPqmfThreads), p.smem, st, in, W, out, n, m, p.RC, p.G,
                               T, Tn));
  }
  count_launch();
  return 0;
}

}  // namespace
}  // namespace satb

using namespace satb;

struct SatbPqmf {
  int n = 0, taps = 0;
  float* wa = nullptr;   // [n][m][n] analysis weights
  float* ws = nullptr;   // [n][m][n] synthesis weights
  bool loaded = false;
};

extern "C" {

int satb_pqmf_create(int num_bands, int taps, SatbPqmf** out) {
  SATB_REQUIRE(out, "pqmf: null argument");
  if (num_bands < 2 || num_bands > kPqmfMaxBands || (num_bands & (num_bands - 1)) != 0) {
    set_last_error("pqmf: num_bands must be a power of 2 in [2, " + std::to_string(kPqmfMaxBands) + "], got " +
                   std::to_string(num_bands));
    return -1;
  }
  if (taps < 2 * num_bands || taps > kPqmfMaxTaps || taps % (2 * num_bands) != 0) {
    set_last_error("pqmf: taps must be a multiple of 2 * num_bands (an even number of taps per polyphase row), at most " +
                   std::to_string(kPqmfMaxTaps) + ", got " + std::to_string(taps) + " for " +
                   std::to_string(num_bands) + " bands");
    return -1;
  }
  SatbPqmf* h = new SatbPqmf();
  h->n = num_bands;
  h->taps = taps;
  const size_t bytes = static_cast<size_t>(num_bands) * taps * sizeof(float);
  cudaError_t e = cudaMalloc(&h->wa, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&h->ws, bytes);
  if (e != cudaSuccess) {
    set_last_error(std::string("pqmf: cudaMalloc failed: ") + cudaGetErrorString(e));
    if (h->wa) cudaFree(h->wa);
    delete h;
    return -2;
  }
  *out = h;
  return 0;
}

void satb_pqmf_destroy(SatbPqmf* h) {
  if (!h) return;
  if (h->wa) cudaFree(h->wa);
  if (h->ws) cudaFree(h->ws);
  delete h;
}

int satb_pqmf_load_filter(SatbPqmf* h, const float* filter_bank, void* stream) {
  SATB_REQUIRE(h && filter_bank, "pqmf: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int total = h->n * h->taps;
  pqmf_prep_kernel<<<std::min(ceil_div(total, 256), 1024), 256, 0, st>>>(filter_bank, h->wa, h->ws, h->n,
                                                                         h->taps / h->n);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  h->loaded = true;
  return 0;
}

int satb_pqmf_analysis(SatbPqmf* h, const float* audio, float* bands, int B, int C, long long T, void* stream) {
  SATB_REQUIRE(h, "pqmf: null handle");
  SATB_REQUIRE(h->loaded, "pqmf: no filter bank loaded");
  SATB_REQUIRE(audio && bands, "pqmf: null argument");
  SATB_REQUIRE(B >= 1 && C >= 1 && static_cast<long long>(B) * C <= 65535, "pqmf: need B, C >= 1 and B * C <= 65535");
  SATB_REQUIRE(T >= 1 && (T + h->n - 1) / h->n < (1LL << 31) - 4096, "pqmf: need 1 <= T and ceil(T / num_bands) < 2^31");
  const int Tn = static_cast<int>((T + h->n - 1) / h->n);
  return launch_pqmf<0>(audio, h->wa, bands, h->n, h->taps, T, Tn, B * C, static_cast<cudaStream_t>(stream));
}

int satb_pqmf_synthesis(SatbPqmf* h, const float* bands, float* audio, int B, int C, int frames, void* stream) {
  SATB_REQUIRE(h, "pqmf: null handle");
  SATB_REQUIRE(h->loaded, "pqmf: no filter bank loaded");
  SATB_REQUIRE(audio && bands, "pqmf: null argument");
  SATB_REQUIRE(B >= 1 && C >= 1 && static_cast<long long>(B) * C <= 65535, "pqmf: need B, C >= 1 and B * C <= 65535");
  SATB_REQUIRE(frames >= 1 && frames < (1 << 30), "pqmf: need 1 <= frames < 2^30");
  return launch_pqmf<1>(bands, h->ws, audio, h->n, h->taps, static_cast<long long>(frames) * h->n, frames, B * C,
                        static_cast<cudaStream_t>(stream));
}

}  // extern "C"
