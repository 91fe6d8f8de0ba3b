// Oobleck VAE encoder / decoder (reference models/autoencoders.py:45-194) on the wgmma
// implicit-GEMM convolution of gemm.cuh.
//
// Data layout: activations are channels-last [B, L, C].  Every tensor-core convolution
// reads a 16-bit, already Snake-activated copy of its input (written by the producer's
// epilogue with the consumer's alpha/beta) and, where a ResidualUnit skip needs it, an fp32
// copy of the raw value.  A dilated k=7 convolution is 7 shifted GEMMs accumulated in registers
// (TMA zero-fills the padding); a transposed convolution (k = 2s, stride s) is a 2-tap GEMM
// over N = s*Cout columns; a strided convolution (k = 2s, stride s) is a 2s-tap GEMM whose
// taps address the input as (phase, row) through a 4-D tensor map.  The encoder's first
// convolution (2 -> 128 channels) is bandwidth-bound and stays on CUDA cores; the decoder's last
// one (128 -> 2) runs through the same GEMM with a mostly empty N tile.  Behind a PQMF pretransform the
// encoder reads and the decoder writes channels * num_bands sub-bands (a multiple of 8, up to 128): the
// encoder's first convolution then runs as a GEMM over a 16-bit channels-last copy of its input.
// Weight-norm (w = g * v / ||v||, torch.nn.utils.weight_norm via dac.nn.layers) is folded
// once at load time.
// Block options (satb_oobleck_create_variant): ELU instead of Snake (use_snake=False) is the ACT template parameter of
// every kernel that activates (kActElu: no per-channel parameters); nearest-neighbour upsampling + conv k = 2s 'same'
// (use_nearest_upsample=True) is a 3-tap GEMM over the low-rate input with N = s*Cout (run_conv_gemm kind 3).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <tuple>
#include <type_traits>
#include <map>
#include <string>
#include <vector>

#include "../../include/satb200.h"
#include "common.cuh"
#include "conv_halo.cuh"
#include "kernels.h"
#include "linear.cuh"

namespace satb {

// ---------------------------------------------------------------- small kernels
namespace {

// scale[i] = g[i] / || v[i, :, :] ||   (one block per dim-0 slice)
__global__ void wn_scale_kernel(const float* __restrict__ g, const float* __restrict__ v, float* __restrict__ scale,
                                int slice) {
  __shared__ float red[32];
  const int i = blockIdx.x;
  const float* vs = v + static_cast<size_t>(i) * slice;
  float s = 0.f;
  for (int j = threadIdx.x; j < slice; j += blockDim.x) s += vs[j] * vs[j];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) scale[i] = g[i] / sqrtf(s);
  }
}

// GEMM weight layout [tap][n][k] (16-bit) from a weight-normed conv weight.
//   mode 0: Conv1d  v [cout, cin, kk]      -> dst[t][co][ci]            = v[co, ci, t] * scale[co]
//   mode 1: ConvT1d v [cin, cout, 2*up]    -> dst[tap][ph*cout+co][ci]  = v[ci, co, ph + tap*up] * scale[ci]
template <bool BF16>
__global__ void conv_w_prep_kernel(const float* __restrict__ v, const float* __restrict__ scale,
                                   uint16_t* __restrict__ dst, uint16_t* __restrict__ dst_lo, int mode, int cin, int cout,
                                   int kk, int up, size_t total) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % cin);
    const size_t rest = i / cin;
    float w;
    if (mode == 0) {
      const int co = static_cast<int>(rest % cout);
      const int t = static_cast<int>(rest / cout);
      w = v[(static_cast<size_t>(co) * cin + ci) * kk + t] * scale[co];
    } else {
      const int n = static_cast<int>(rest % (static_cast<size_t>(up) * cout));
      const int tap = static_cast<int>(rest / (static_cast<size_t>(up) * cout));
      const int ph = n / cout, co = n - ph * cout;
      w = v[(static_cast<size_t>(ci) * cout + co) * kk + ph + tap * up] * scale[ci];
    }
    typename Op16<BF16>::T h = Op16<BF16>::from_float(w);
    dst[i] = *reinterpret_cast<uint16_t*>(&h);
    if (dst_lo) {   // split-operand mode: the part of w the 16-bit value lost
      typename Op16<BF16>::T l = Op16<BF16>::from_float(w - Op16<BF16>::to_float(h));
      dst_lo[i] = *reinterpret_cast<uint16_t*>(&l);
    }
  }
}

__global__ void fold_small_kernel(const float* __restrict__ v, const float* __restrict__ scale, float* __restrict__ dst,
                                  int slice, size_t total) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < total) dst[i] = v[i] * scale[i / slice];
}

__global__ void snake_prep_kernel(const float* __restrict__ alpha, const float* __restrict__ beta,
                                  float* __restrict__ a, float* __restrict__ ib, int c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c) {
    a[i] = expf(alpha[i]);
    ib[i] = 1.0f / (expf(beta[i]) + 0.000000001f);
  }
}

// NCL fp32 -> channels-last 16-bit (no activation): the decoder's latent input.
template <bool BF16>
__global__ void __launch_bounds__(256) ncl_to_nlc16_kernel(const float* __restrict__ x, uint16_t* __restrict__ y,
                                                           uint16_t* __restrict__ y_lo, int C, int L) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* xs = x + static_cast<size_t>(b) * C * L;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, l = l0 + tx;
    tile[j][tx] = (c < C && l < L) ? xs[static_cast<size_t>(c) * L + l] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int l = l0 + j, c = c0 + tx;
    if (l < L && c < C) {
      typename Op16<BF16>::T h = Op16<BF16>::from_float(tile[tx][j]);
      y[(static_cast<size_t>(b) * L + l) * C + c] = *reinterpret_cast<uint16_t*>(&h);
      if (y_lo) {
        typename Op16<BF16>::T lo = Op16<BF16>::from_float(tile[tx][j] - Op16<BF16>::to_float(h));
        y_lo[(static_cast<size_t>(b) * L + l) * C + c] = *reinterpret_cast<uint16_t*>(&lo);
      }
    }
  }
}

// Encoder input convolution (audio NCL fp32, Cin = 1 or 2 -> C channels, k taps, pad k/2):
// bandwidth-bound; one thread per output channel, a tile of positions per block.
// Writes raw fp32 and the activated (Snake or ELU: ACT) 16-bit copy, channels-last.
template <bool BF16, int ACT>
__global__ void __launch_bounds__(256) conv_in_kernel(const float* __restrict__ audio, const float* __restrict__ w,
                                                      const float* __restrict__ bias, const float* __restrict__ sn_a,
                                                      const float* __restrict__ sn_ib, void* __restrict__ raw,
                                                      uint16_t* __restrict__ s16, uint16_t* __restrict__ s16_lo, int Cin,
                                                      int C, int64_t T, int kk, int raw16) {
  constexpr int kTile = 64;
  extern __shared__ float sm_in[];  // [Cin][kTile + kk - 1]
  const int b = blockIdx.y;
  const int64_t l0 = static_cast<int64_t>(blockIdx.x) * kTile;
  const int halo = kk / 2, span = kTile + kk - 1;
  for (int i = threadIdx.x; i < Cin * span; i += blockDim.x) {
    const int ci = i / span, j = i - ci * span;
    const int64_t l = l0 + j - halo;
    sm_in[i] = (l >= 0 && l < T) ? audio[(static_cast<size_t>(b) * Cin + ci) * T + l] : 0.f;
  }
  __syncthreads();
  for (int co = threadIdx.x; co < C; co += blockDim.x) {
    float wr[16];  // Cin * kk <= 16 (stereo k7 = 14)
    for (int i = 0; i < Cin * kk; ++i) wr[i] = w[static_cast<size_t>(co) * Cin * kk + i];
    const float bb = bias ? bias[co] : 0.f;
    const float a = ACT == kActSnake ? sn_a[co] : 0.f, ib = ACT == kActSnake ? sn_ib[co] : 0.f;
    for (int j = 0; j < kTile; ++j) {
      const int64_t l = l0 + j;
      if (l >= T) break;
      float acc = bb;
      for (int ci = 0; ci < Cin; ++ci)
        for (int t = 0; t < kk; ++t) acc = fmaf(wr[ci * kk + t], sm_in[ci * span + j + t], acc);
      const size_t o = (static_cast<size_t>(b) * T + l) * C + co;
      if (raw16) {
        typename Op16<BF16>::T r = Op16<BF16>::from_float(acc);
        static_cast<uint16_t*>(raw)[o] = *reinterpret_cast<uint16_t*>(&r);
      } else {
        static_cast<float*>(raw)[o] = acc;
      }
      const float act = act_fast<ACT>(acc, a, ib);
      typename Op16<BF16>::T h = Op16<BF16>::from_float(act);
      s16[o] = *reinterpret_cast<uint16_t*>(&h);
      if (s16_lo) {
        typename Op16<BF16>::T lo = Op16<BF16>::from_float(act - Op16<BF16>::to_float(h));
        s16_lo[o] = *reinterpret_cast<uint16_t*>(&lo);
      }
    }
  }
}
// Nearest-neighbour upsampling by `up` followed by a Conv1d v [cout, cin, 2 up] with padding 'same' (up - 1 zeros on
// the left, up on the right; models/autoencoders.py:95-100) is a 3-tap convolution of the low-rate input over
// N = up * cout columns: output position up * m + ph reads x[m + o], o = -1, 0, 1, through
//   dst[o + 1][ph * cout + co][ci] = sum_{k : floor((ph + k - up + 1) / up) = o} v[co, ci, k] * scale[co]
// The sum runs in fp64 and is rounded to fp32 once; the fp32 value is then stored like every other conv weight (its
// 16-bit rounding, and the 16-bit rounding of the remainder as the lo block in split-operand mode).
template <bool BF16>
__global__ void nearest_w_prep_kernel(const float* __restrict__ v, const float* __restrict__ scale,
                                      uint16_t* __restrict__ dst, uint16_t* __restrict__ dst_lo, int cin, int cout,
                                      int up, size_t total) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % cin);
    const size_t rest = i / cin;
    const int n = static_cast<int>(rest % (static_cast<size_t>(up) * cout));
    const int o = static_cast<int>(rest / (static_cast<size_t>(up) * cout)) - 1;
    const int ph = n / cout, co = n - ph * cout;
    // floor((ph + k - up + 1) / up) = o  <=>  k in [(o + 1) up - ph - 1, (o + 2) up - ph - 1), clipped to [0, 2 up)
    const int k0 = max((o + 1) * up - ph - 1, 0), k1 = min((o + 2) * up - ph - 1, 2 * up);
    const float* vr = v + (static_cast<size_t>(co) * cin + ci) * (2 * up);
    double acc = 0.0;
    for (int k = k0; k < k1; ++k) acc += static_cast<double>(vr[k]) * static_cast<double>(scale[co]);
    const float w = static_cast<float>(acc);
    typename Op16<BF16>::T h = Op16<BF16>::from_float(w);
    dst[i] = *reinterpret_cast<uint16_t*>(&h);
    if (dst_lo) {
      typename Op16<BF16>::T l = Op16<BF16>::from_float(w - Op16<BF16>::to_float(h));
      dst_lo[i] = *reinterpret_cast<uint16_t*>(&l);
    }
  }
}

}  // namespace

struct ConvW {
  int cin = 0, cout = 0, k = 0;
  bool transposed = false, small = false, has_bias = true;
  bool nearest = false;     // nearest-upsample conv (k = 2 * up), stored folded as 3 taps over up * cout rows
  std::string pfx;
  uint16_t* w16 = nullptr;  // [taps][n][cin]
  float* w32 = nullptr;     // small convs: folded [cout][cin][k]
  float* bias = nullptr;
};
struct SnakeW {
  int c = 0;
  std::string pfx;
  float *a = nullptr, *ib = nullptr;
};

}  // namespace satb

using namespace satb;

struct SatbOobleck {
  SatbOobleckConfig cfg;
  int act = kActSnake;             // the blocks' activation (use_snake): kActSnake or kActElu
  bool nearest = false;            // decoder upsampling: nearest + conv (use_nearest_upsample) instead of ConvTranspose1d
  bool bf16 = false;
  int raw16 = 0;                   // 1: the raw skip stream is carried in the 16-bit operand type (fp16 mode), 0: fp32
  bool split3 = false;             // operand_dtype 2 ("fp16x3"): every product as (hi, hi) + (lo, hi) + (hi, lo), see GemmShape
  size_t lo_off = 0;               // bytes from a 16-bit activation buffer to its "lo" half (split3)
  unsigned routes = 0;             // SATB_OOB_ROUTE_* bits of the kernels launched since the last reset (probe report)
  bool wrote_raw = false;          // whether the last step wrote its raw output (probe report)
  std::vector<int> chans;          // c_mults[i] * channels, i = 0..n (c_mults prepended with 1)
  std::map<std::string, std::pair<float*, long long>> raw;   // state-dict entries (device fp32)
  std::vector<void*> owned;
  std::map<std::string, ConvW> convs;
  std::map<std::string, SnakeW> snakes;
  bool finalized = false;
  // workspace
  void *buf_raw = nullptr, *buf_a = nullptr, *buf_b = nullptr;
  size_t cap_raw = 0, cap_a = 0, cap_b = 0;
  std::map<std::tuple<const void*, int, int, int, int64_t, int64_t, int>, CUtensorMap> tmaps;

  int alloc_bytes(void** p, size_t bytes) {
    cudaError_t e = cudaMalloc(p, bytes < 256 ? 256 : bytes);
    if (e != cudaSuccess) {
      set_last_error(std::string("cudaMalloc failed: ") + cudaGetErrorString(e));
      return -2;
    }
    owned.push_back(*p);
    return 0;
  }
  int ensure(void** buf, size_t* cap, size_t need) {
    if (need <= *cap) return 0;
    if (*buf) cudaFree(*buf);
    *buf = nullptr;
    *cap = 0;
    cudaError_t e = cudaMalloc(buf, need);
    if (e != cudaSuccess) {
      set_last_error(std::string("cudaMalloc failed: ") + cudaGetErrorString(e) + " (" + std::to_string(need) + " B)");
      return -2;
    }
    *cap = need;
    tmaps.clear();
    return 0;
  }
};

namespace {

int get_raw(SatbOobleck* h, const std::string& name, long long expect, float** out) {
  auto it = h->raw.find(name);
  if (it == h->raw.end()) {
    set_last_error("oobleck: missing weight " + name);
    return -4;
  }
  if (expect >= 0 && it->second.second != expect) {
    set_last_error("oobleck: bad size for " + name + ": got " + std::to_string(it->second.second) + ", expected " +
                   std::to_string(expect));
    return -4;
  }
  *out = it->second.first;
  return 0;
}

int prep_conv(SatbOobleck* h, const std::string& pfx, int cin, int cout, int k, bool transposed, bool small,
              bool has_bias, int up, cudaStream_t st) {
  ConvW c;
  c.cin = cin; c.cout = cout; c.k = k; c.transposed = transposed; c.small = small; c.has_bias = has_bias; c.pfx = pfx;
  float *g, *v;
  const int d0 = transposed ? cin : cout;
  const int slice = (transposed ? cout : cin) * k;
  SATB_PROPAGATE(get_raw(h, pfx + "weight_g", d0, &g));
  SATB_PROPAGATE(get_raw(h, pfx + "weight_v", static_cast<long long>(d0) * slice, &v));
  if (has_bias) SATB_PROPAGATE(get_raw(h, pfx + "bias", cout, &c.bias));
  float* scale;
  SATB_PROPAGATE(h->alloc_bytes(reinterpret_cast<void**>(&scale), static_cast<size_t>(d0) * 4));
  wn_scale_kernel<<<d0, 256, 0, st>>>(g, v, scale, slice);
  count_launch();
  const size_t total = static_cast<size_t>(cin) * cout * k;
  if (small) {
    SATB_PROPAGATE(h->alloc_bytes(reinterpret_cast<void**>(&c.w32), total * 4));
    fold_small_kernel<<<static_cast<int>(ceil_div64(total, 256)), 256, 0, st>>>(v, scale, c.w32, slice, total);
  } else {
    const size_t parts = h->split3 ? 2 : 1;      // [hi block | lo block]
    SATB_PROPAGATE(h->alloc_bytes(reinterpret_cast<void**>(&c.w16), parts * total * 2 + 256 * 128));  // slack for box overreach
    SATB_CHECK_CUDA(cudaMemsetAsync(c.w16, 0, parts * total * 2 + 256 * 128, st));
    uint16_t* w_lo = h->split3 ? c.w16 + total : nullptr;
    int grid = static_cast<int>(ceil_div64(total, 256));
    if (grid > 8192) grid = 8192;
    if (h->bf16)
      conv_w_prep_kernel<true><<<grid, 256, 0, st>>>(v, scale, c.w16, w_lo, transposed ? 1 : 0, cin, cout, k, up, total);
    else
      conv_w_prep_kernel<false><<<grid, 256, 0, st>>>(v, scale, c.w16, w_lo, transposed ? 1 : 0, cin, cout, k, up, total);
  }
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  h->convs[pfx] = c;
  return 0;
}

// Conv1d k = 2 up after a nearest x up upsample (no bias), folded to the 3-tap block of nearest_w_prep_kernel.
int prep_conv_nearest(SatbOobleck* h, const std::string& pfx, int cin, int cout, int up, cudaStream_t st) {
  ConvW c;
  c.cin = cin; c.cout = cout; c.k = 2 * up; c.has_bias = false; c.nearest = true; c.pfx = pfx;
  float *g, *v;
  const int slice = cin * c.k;
  SATB_PROPAGATE(get_raw(h, pfx + "weight_g", cout, &g));
  SATB_PROPAGATE(get_raw(h, pfx + "weight_v", static_cast<long long>(cout) * slice, &v));
  float* scale;
  SATB_PROPAGATE(h->alloc_bytes(reinterpret_cast<void**>(&scale), static_cast<size_t>(cout) * 4));
  wn_scale_kernel<<<cout, 256, 0, st>>>(g, v, scale, slice);
  count_launch();
  const size_t total = static_cast<size_t>(3) * up * cout * cin;
  const size_t parts = h->split3 ? 2 : 1;      // [hi block | lo block]
  SATB_PROPAGATE(h->alloc_bytes(reinterpret_cast<void**>(&c.w16), parts * total * 2 + 256 * 128));  // slack for box overreach
  SATB_CHECK_CUDA(cudaMemsetAsync(c.w16, 0, parts * total * 2 + 256 * 128, st));
  uint16_t* w_lo = h->split3 ? c.w16 + total : nullptr;
  int grid = static_cast<int>(ceil_div64(total, 256));
  if (grid > 8192) grid = 8192;
  if (h->bf16)
    nearest_w_prep_kernel<true><<<grid, 256, 0, st>>>(v, scale, c.w16, w_lo, cin, cout, up, total);
  else
    nearest_w_prep_kernel<false><<<grid, 256, 0, st>>>(v, scale, c.w16, w_lo, cin, cout, up, total);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  h->convs[pfx] = c;
  return 0;
}

// elements of a finalized conv's stored weight block (one part)
size_t conv_w_elems(const ConvW& c) {
  const size_t n = static_cast<size_t>(c.cin) * c.cout;
  return c.nearest ? n * 3 * (c.k / 2) : n * c.k;
}

int prep_snake(SatbOobleck* h, const std::string& pfx, int c, cudaStream_t st) {
  if (h->act != kActSnake) return 0;     // nn.ELU has no parameters: nothing to look up
  SnakeW s;
  s.c = c; s.pfx = pfx;
  float *al, *be;
  SATB_PROPAGATE(get_raw(h, pfx + "alpha", c, &al));
  SATB_PROPAGATE(get_raw(h, pfx + "beta", c, &be));
  SATB_PROPAGATE(h->alloc_bytes(reinterpret_cast<void**>(&s.a), static_cast<size_t>(c) * 4));
  SATB_PROPAGATE(h->alloc_bytes(reinterpret_cast<void**>(&s.ib), static_cast<size_t>(c) * 4));
  snake_prep_kernel<<<ceil_div(c, 256), 256, 0, st>>>(al, be, s.a, s.ib, c);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  h->snakes[pfx] = s;
  return 0;
}

// The parameters of the activation at `pfx`: the Snake's, or null in an ELU model (nn.ELU sits at the same index of
// the Sequential and has none).
const SnakeW* act_params(const SatbOobleck* h, const std::string& pfx) {
  return h->act == kActSnake ? &h->snakes.at(pfx) : nullptr;
}
const float* act_a(const SnakeW* s) { return s ? s->a : nullptr; }
const float* act_ib(const SnakeW* s) { return s ? s->ib : nullptr; }

int get_tmap_a(SatbOobleck* h, const void* in16, int cin, int a_rows, int B, int L_in, int a_stride, const CUtensorMap** out,
               int box_rows = kBlockM) {
  auto key = std::make_tuple(in16, cin, a_rows, B, static_cast<int64_t>(cin), static_cast<int64_t>(L_in) * cin,
                             a_stride | (box_rows << 8));
  auto it = h->tmaps.find(key);
  if (it == h->tmaps.end()) {
    CUtensorMap m;
    SATB_PROPAGATE(make_tmap_a(&m, in16, cin, a_rows, B, cin, static_cast<int64_t>(L_in) * cin, a_stride, box_rows));
    it = h->tmaps.emplace(key, m).first;
  }
  *out = &it->second;
  return 0;
}

int get_tmap_b(SatbOobleck* h, const ConvW& cw, int b_rows, int box, const CUtensorMap** out) {
  auto key = std::make_tuple(static_cast<const void*>(cw.w16), cw.cin, b_rows, -1, static_cast<int64_t>(cw.cin), int64_t(0), box);
  auto it = h->tmaps.find(key);
  if (it == h->tmaps.end()) {
    CUtensorMap m;
    SATB_PROPAGATE(make_tmap_b(&m, cw.w16, cw.cin, b_rows, cw.cin, box));
    it = h->tmaps.emplace(key, m).first;
  }
  *out = &it->second;
  return 0;
}

// One tensor-core convolution.  in16: [B, L_in, cin] 16-bit.  Output positions per item L_out.
//   kind 0: conv k taps, dilation dil, "same" padding           (L_out = L_in)
//   kind 1: transposed conv k = 2*up, stride up, pad ceil(up/2)  (L_out = L_in * up)
//   kind 2: strided conv k = 2*st, stride st, pad ceil(st/2)     (L_out = L_in / st)
//   kind 3: nearest x up then conv k = 2*up, 'same' padding, as 3 taps over N = up*cout  (L_out = L_in * up)
template <class Epi, bool BF16>
int run_conv_gemm(SatbOobleck* h, const ConvW& cw, const void* in16, int B, int L_in, int kind, int dil, int factor,
                  const typename Epi::Params& ep, cudaStream_t st) {
  // the default 16-bit decode / encode runs the lean-epilogue instantiation of the GEMM kernels (EpiConv<.., MASKED>)
  constexpr bool kGeneralConv =
      std::is_same<Epi, EpiConv<BF16, false>>::value || std::is_same<Epi, EpiConvElu<BF16, false>>::value;
  constexpr bool kLeanConv = std::is_same<Epi, EpiConv<BF16, true>>::value || std::is_same<Epi, EpiConvElu<BF16, true>>::value;
  if constexpr (kGeneralConv) {
    if (Epi::fast_flags(ep))
      return run_conv_gemm<EpiConvFor<BF16, true, Epi::kAct>, BF16>(h, cw, in16, B, L_in, kind, dil, factor, ep, st);
  }
  h->routes |= std::is_same<Epi, EpiStoreNCL>::value ? SATB_OOB_ROUTE_GEMM_NCL
               : kLeanConv                           ? SATB_OOB_ROUTE_GEMM_LEAN
                                                     : SATB_OOB_ROUTE_GEMM;
  GemmShape s;
  s.batches = B;
  s.b_static = 1;   // folded weight-norm weights, written at finalize time
  s.K = cw.cin;
  int a_stride = 1, a_rows = L_in;
  if (kind == 0) {
    s.L = L_in; s.N = cw.cout; s.n_taps = cw.k; s.tap_base = -(cw.k / 2) * dil; s.tap_step = dil; s.b_tap_rows = cw.cout;
    s.stride = 1;
  } else if (kind == 1) {
    s.L = L_in + 1; s.N = factor * cw.cout; s.n_taps = 2; s.tap_base = 0; s.tap_step = -1; s.b_tap_rows = factor * cw.cout;
    s.stride = 1;
  } else if (kind == 3) {
    SATB_REQUIRE(cw.nearest && cw.k == 2 * factor, "nearest upsample: needs the folded 3-tap weights of stride factor");
    s.L = L_in; s.N = factor * cw.cout; s.n_taps = 3; s.tap_base = -1; s.tap_step = 1; s.b_tap_rows = factor * cw.cout;
    s.stride = 1;
  } else {
    SATB_REQUIRE(L_in % factor == 0, "strided conv: length must be a multiple of the stride");
    s.L = L_in / factor; s.N = cw.cout; s.n_taps = cw.k; s.tap_base = -((factor + 1) / 2); s.tap_step = 1;
    s.b_tap_rows = cw.cout; s.stride = factor;
    a_stride = factor; a_rows = L_in / factor;
  }
  const CUtensorMap* tap;
  SATB_PROPAGATE(get_tmap_a(h, in16, cw.cin, a_rows, B, L_in, a_stride, &tap));
  const CUtensorMap& ta = *tap;
  const CUtensorMap* ta2 = nullptr;
  int b_rows = s.n_taps * s.b_tap_rows;
  if (h->split3) {
    SATB_PROPAGATE(get_tmap_a(h, static_cast<const char*>(in16) + h->lo_off, cw.cin, a_rows, B, L_in, a_stride, &ta2));
    s.n_parts = 3;
    s.b_part_rows = b_rows;       // the lo weight block follows the hi block
    b_rows *= 2;
  }
  auto get_b = [&](int box, const CUtensorMap** out) -> int { return get_tmap_b(h, cw, b_rows, box, out); };
  const CUtensorMap* tb;
  if (s.N >= 256) {
    SATB_PROPAGATE(get_b(256, &tb));
    return launch_gemm<Epi, 256, BF16>(ta, *tb, s, ep, st, ta2);
  } else if (s.N > 64) {
    SATB_PROPAGATE(get_b(128, &tb));
    return launch_gemm<Epi, 128, BF16>(ta, *tb, s, ep, st, ta2);
  }
  SATB_PROPAGATE(get_b(64, &tb));
  return launch_gemm<Epi, 64, BF16>(ta, *tb, s, ep, st, ta2);
}

// ResidualUnit (models/autoencoders.py:45-68).  In: snake1(x) as 16-bit in sA, x as fp32 in raw.
// Out: y = x + conv1(snake2(conv7(.))) as fp32 in raw (if keep_raw) and snake_next(y) as 16-bit in sA;
// sT is scratch (the two pointers are swapped when the fused kernel wrote its output there).
// ACT: the model's activation (snake1 / snake2 / the next one are ELUs in an ELU model, with null parameters).
template <bool BF16, int ACT>
int residual_unit(SatbOobleck* h, const std::string& pfx, int C, int B, int L, int dil, void* raw, void*& sA, void*& sT,
                  const SnakeW* next_snake, bool keep_raw, cudaStream_t st) {
  const ConvW& c7 = h->convs.at(pfx + "layers.1.");
  const ConvW& c1 = h->convs.at(pfx + "layers.3.");
  const SnakeW* s2 = act_params(h, pfx + "layers.2.");
  typedef EpiConvFor<BF16, false, ACT> E;
  typename E::Params e1{c1.bias, raw, keep_raw ? raw : nullptr, sA, next_snake ? next_snake->a : nullptr,
                        next_snake ? next_snake->ib : nullptr, C, L, 1, 0, h->split3 ? static_cast<char*>(sA) + h->lo_off : nullptr, h->raw16};
  if ((C == 128 || C == 256) && c7.k == 7 && 6 * dil <= kHaloMax && !h->split3) {
    // one kernel: conv7 -> snake2 -> conv1 -> + skip; reads sA (with a halo), so it must write elsewhere
    const CUtensorMap *ta, *tb7, *tb1;
    SATB_PROPAGATE(get_tmap_a(h, sA, C, L, B, L, 1, &ta, kBlockM + 6 * dil));   // one halo box per k-block
    SATB_PROPAGATE(get_tmap_b(h, c7, c7.k * C, C, &tb7));
    SATB_PROPAGATE(get_tmap_b(h, c1, C, C, &tb1));
    e1.s16_out = sT;
    const HaloShape hs{L, B, C, 7, dil, C};
    const ResUnitPre pre{c7.bias, act_a(s2), act_ib(s2)};
    h->routes |= E::fast_flags(e1) ? SATB_OOB_ROUTE_FUSED_LEAN : SATB_OOB_ROUTE_FUSED;
    if (E::fast_flags(e1)) {
      typedef EpiConvFor<BF16, true, ACT> EM;
      SATB_PROPAGATE(C == 128 ? (launch_conv_halo<EM, 128, BF16, true>(*ta, *tb7, tb1, hs, pre, e1, st))
                              : (launch_conv_halo<EM, 256, BF16, true>(*ta, *tb7, tb1, hs, pre, e1, st)));
    } else {
      SATB_PROPAGATE(C == 128 ? (launch_conv_halo<E, 128, BF16, true>(*ta, *tb7, tb1, hs, pre, e1, st))
                              : (launch_conv_halo<E, 256, BF16, true>(*ta, *tb7, tb1, hs, pre, e1, st)));
    }
    std::swap(sA, sT);
    return 0;
  }
  // conv7(dil) on sA -> snake2 -> sT ; conv1 on sT -> + x -> raw, snake_next -> sA
  typename E::Params e7{c7.bias, nullptr, nullptr, sT, act_a(s2), act_ib(s2), C, L, 1, 0, h->split3 ? static_cast<char*>(sT) + h->lo_off : nullptr, h->raw16};
  SATB_PROPAGATE((run_conv_gemm<E, BF16>(h, c7, sA, B, L, 0, dil, 1, e7, st)));
  SATB_PROPAGATE((run_conv_gemm<E, BF16>(h, c1, sT, B, L, 0, 1, 1, e1, st)));
  return 0;
}

void* lo_half(const SatbOobleck* h, void* p16) { return h->split3 ? static_cast<char*>(p16) + h->lo_off : nullptr; }

// ---- the steps of a decode / encode.  decode_impl / encode_impl run them in order over the handle's workspaces;
// satb_oobleck_probe runs one of them on caller-owned buffers.  Blocks b = 1 .. n, units j = 0 .. 2.

// Decoder input: latents z NCL fp32 [B, latent_dim, L] -> channels-last 16-bit in tmp16 -> conv k7 latent -> chans[n],
// whose epilogue applies block 1's leading activation, into out16.
template <bool BF16, int ACT>
int dec_input(SatbOobleck* h, const float* z, void* tmp16, void* out16, int B, int L, cudaStream_t st) {
  const SatbOobleckConfig& c = h->cfg;
  {
    dim3 grid(ceil_div(L, 32), ceil_div(c.latent_dim, 32), B);
    ncl_to_nlc16_kernel<BF16><<<grid, 256, 0, st>>>(z, static_cast<uint16_t*>(tmp16),
                                                    static_cast<uint16_t*>(lo_half(h, tmp16)), c.latent_dim, L);
    count_launch();
  }
  typedef EpiConvFor<BF16, false, ACT> E;
  const ConvW& c0 = h->convs.at("layers.0.");
  const SnakeW* sn = act_params(h, "layers.1.layers.0.");
  typename E::Params ep{c0.bias, nullptr, nullptr, out16, act_a(sn), act_ib(sn), c0.cout, L, 1, 0, lo_half(h, out16), h->raw16};
  h->wrote_raw = false;
  return run_conv_gemm<E, BF16>(h, c0, tmp16, B, L, 0, 1, 1, ep, st);
}

// Decoder block b: transposed conv (or nearest upsample + conv, folded to 3 taps) of in16 [B, L_in, chans[n-b+1]] ->
// raw and act(unit 0) into out16, both [B, L_in * stride, chans[n-b]].
template <bool BF16, int ACT>
int dec_upsample(SatbOobleck* h, int b, const void* in16, void* raw, void* out16, int B, int L_in, cudaStream_t st) {
  const int n = h->cfg.n_stages, cout = h->chans[n - b], s = h->cfg.strides[n - b];
  const std::string bp = "layers." + std::to_string(b) + ".";
  const ConvW& ct = h->convs.at(bp + (h->nearest ? "layers.1.1." : "layers.1."));
  const SnakeW* s_ru0 = act_params(h, bp + "layers.2.layers.0.");
  const int64_t Lo = static_cast<int64_t>(L_in) * s;
  SATB_REQUIRE(Lo < (int64_t(1) << 31) && static_cast<int64_t>(B) * Lo * cout < (int64_t(1) << 40), "decoder: sequence too long");
  typedef EpiConvFor<BF16, false, ACT> E;
  // nearest: output position s m + ph is row m, column ph * cout + co (no padding to drop, no bias)
  typename E::Params et{ct.bias, nullptr, raw, out16, act_a(s_ru0), act_ib(s_ru0), cout, static_cast<int>(Lo), s,
                        h->nearest ? 0 : (s + 1) / 2, lo_half(h, out16), h->raw16};
  h->wrote_raw = true;
  return run_conv_gemm<E, BF16>(h, ct, in16, B, L_in, h->nearest ? 3 : 1, 1, s, et, st);
}

// Decoder ResidualUnit j of block b over [B, L, chans[n-b]]; the activation applied to its output is the next unit's,
// then the next block's, then the final one.
template <bool BF16, int ACT>
int dec_residual(SatbOobleck* h, int b, int j, int B, int L, void* raw, void*& sA, void*& sT, cudaStream_t st) {
  static const int dils[3] = {1, 3, 9};
  const int n = h->cfg.n_stages;
  const std::string bp = "layers." + std::to_string(b) + ".";
  const SnakeW* next;
  if (j < 2)
    next = act_params(h, bp + "layers." + std::to_string(3 + j) + ".layers.0.");
  else if (b < n)
    next = act_params(h, "layers." + std::to_string(b + 1) + ".layers.0.");
  else
    next = act_params(h, "layers." + std::to_string(n + 1) + ".");
  h->wrote_raw = j < 2;   // the last unit's raw output has no reader: the next step is a transposed or final conv
  return residual_unit<BF16, ACT>(h, bp + "layers." + std::to_string(2 + j) + ".", h->chans[n - b], B, L, dils[j], raw,
                                  sA, sT, next, j < 2, st);
}

// Decoder final conv k7 chans[0] -> audio channels (no bias, optional tanh) of in16 [B, L, chans[0]] into audio NCL.
// The 128 -> 2 contraction runs with the N tile mostly empty (8x wasted MMA work is still ~10x faster than the
// shared-memory-bound CUDA-core version it replaces: 1.21 ms -> bandwidth-bound).  Up to 64 outputs (audio, or the
// sub-bands of a PQMF pretransform) take the halo-tile route; 65 .. 128 sub-bands take the implicit GEMM's 128 tile.
template <bool BF16>
int dec_output(SatbOobleck* h, const void* in16, float* audio, int B, int L, cudaStream_t st) {
  const ConvW& cf = h->convs.at("layers." + std::to_string(h->cfg.n_stages + 2) + ".");
  EpiStoreNCL::Params ep{audio, nullptr, cf.cout, L, h->cfg.final_tanh};
  h->wrote_raw = false;
  if (!h->split3 && cf.cout <= 64 && cf.cin % kBlockK == 0 && cf.k % 2 == 1 && cf.k - 1 <= kHaloMax) {
    // every activation row is fetched once per tile instead of once per tap (see conv_halo.cuh)
    const CUtensorMap *ta, *tb;
    SATB_PROPAGATE(get_tmap_a(h, in16, cf.cin, L, B, L, 1, &ta, kBlockM + cf.k - 1));
    SATB_PROPAGATE(get_tmap_b(h, cf, cf.k * cf.cout, 64, &tb));
    const HaloShape hs{L, B, cf.cin, cf.k, 1, cf.cout};
    h->routes |= SATB_OOB_ROUTE_HALO_NCL;
    return launch_conv_halo<EpiStoreNCL, 64, BF16, false>(*ta, *tb, nullptr, hs, ResUnitPre{}, ep, st);
  }
  return run_conv_gemm<EpiStoreNCL, BF16>(h, cf, in16, B, L, 0, 1, 1, ep, st);
}

// Encoder input conv k7 audio NCL [B, in_channels, T] -> chans[0]: raw, and block 1 / unit 0's activation into out16.
// 1 or 2 channels run on CUDA cores.  Wider inputs (the sub-bands of a PQMF pretransform, a multiple of 8 channels) are
// cast to channels-last 16-bit in tmp16 and run as a 7-tap implicit GEMM with the same epilogue outputs.
template <bool BF16, int ACT>
int enc_input(SatbOobleck* h, const float* audio, void* raw, void* out16, void* tmp16, int B, int64_t T,
              cudaStream_t st) {
  const ConvW& c0 = h->convs.at("layers.0.");
  const SnakeW* sn = act_params(h, "layers.1.layers.0.layers.0.");
  h->wrote_raw = true;
  if (!c0.small) {
    dim3 grid(static_cast<unsigned>(ceil_div64(T, 32)), ceil_div(c0.cin, 32), B);
    ncl_to_nlc16_kernel<BF16><<<grid, 256, 0, st>>>(audio, static_cast<uint16_t*>(tmp16),
                                                    static_cast<uint16_t*>(lo_half(h, tmp16)), c0.cin, static_cast<int>(T));
    count_launch();
    typedef EpiConvFor<BF16, false, ACT> E;
    typename E::Params ep{c0.bias, nullptr, raw, out16, act_a(sn), act_ib(sn), c0.cout, static_cast<int>(T), 1, 0,
                          lo_half(h, out16), h->raw16};
    return run_conv_gemm<E, BF16>(h, c0, tmp16, B, static_cast<int>(T), 0, 1, 1, ep, st);
  }
  SATB_REQUIRE(c0.cin * c0.k <= 16, "encoder input conv: in_channels * kernel must be <= 16");
  const size_t smem = static_cast<size_t>(c0.cin) * (64 + c0.k - 1) * 4;
  dim3 grid(static_cast<unsigned>(ceil_div64(T, 64)), B);
  conv_in_kernel<BF16, ACT><<<grid, 256, smem, st>>>(audio, c0.w32, c0.bias, act_a(sn), act_ib(sn), raw,
                                                      static_cast<uint16_t*>(out16),
                                                      static_cast<uint16_t*>(lo_half(h, out16)), c0.cin, c0.cout, T, c0.k,
                                                      h->raw16);
  count_launch();
  h->routes |= SATB_OOB_ROUTE_CUDA_CORE;
  return 0;
}

// Encoder ResidualUnit j of block b over [B, L, chans[b-1]]; the activation applied to its output is the next unit's,
// then the block's own before its strided conv.
template <bool BF16, int ACT>
int enc_residual(SatbOobleck* h, int b, int j, int B, int L, void* raw, void*& sA, void*& sT, cudaStream_t st) {
  static const int dils[3] = {1, 3, 9};
  const std::string bp = "layers." + std::to_string(b) + ".";
  const SnakeW* next = j < 2 ? act_params(h, bp + "layers." + std::to_string(j + 1) + ".layers.0.")
                             : act_params(h, bp + "layers.3.");
  h->wrote_raw = j < 2;   // the strided conv that follows the last unit has no skip
  return residual_unit<BF16, ACT>(h, bp + "layers." + std::to_string(j) + ".", h->chans[b - 1], B, L, dils[j], raw, sA,
                                  sT, next, j < 2, st);
}

// Encoder block b: strided conv of in16 [B, L_in, chans[b-1]] (already activated) -> [B, L_in / s, chans[b]]:
// raw (when a next block reads it as its first skip) and the next block's (or the final) activation into out16.
template <bool BF16, int ACT>
int enc_downsample(SatbOobleck* h, int b, const void* in16, void* raw, void* out16, int B, int L_in, cudaStream_t st) {
  const int n = h->cfg.n_stages, s = h->cfg.strides[b - 1];
  const ConvW& cs = h->convs.at("layers." + std::to_string(b) + ".layers.4.");
  const int Lo = L_in / s;
  const SnakeW* nx = b < n ? act_params(h, "layers." + std::to_string(b + 1) + ".layers.0.layers.0.")
                           : act_params(h, "layers." + std::to_string(n + 1) + ".");
  typedef EpiConvFor<BF16, false, ACT> E;
  typename E::Params ep{cs.bias, nullptr, b < n ? raw : nullptr, out16, act_a(nx), act_ib(nx), cs.cout, Lo, 1, 0, lo_half(h, out16), h->raw16};
  h->wrote_raw = b < n;
  return run_conv_gemm<E, BF16>(h, cs, in16, B, L_in, 2, 1, s, ep, st);
}

// Encoder final conv k3 chans[n] -> latent_dim of in16 [B, L, chans[n]], NCL fp32 output
template <bool BF16>
int enc_output(SatbOobleck* h, const void* in16, float* latents, int B, int L, cudaStream_t st) {
  const ConvW& cf = h->convs.at("layers." + std::to_string(h->cfg.n_stages + 2) + ".");
  EpiStoreNCL::Params ep{latents, cf.bias, cf.cout, L, 0};
  h->wrote_raw = false;
  return run_conv_gemm<EpiStoreNCL, BF16>(h, cf, in16, B, L, 0, 1, 1, ep, st);
}

template <bool BF16, int ACT>
int decode_impl(SatbOobleck* h, const float* z, float* audio, int B, int L, cudaStream_t st) {
  const SatbOobleckConfig& c = h->cfg;
  const int n = c.n_stages;
  // sizes
  size_t max_elems = static_cast<size_t>(B) * L * std::max(c.latent_dim, h->chans[n]);
  {
    int64_t l = L;
    for (int b = 1; b <= n; ++b) {
      const int s = c.strides[n - b];
      l *= s;
      max_elems = std::max(max_elems, static_cast<size_t>(B) * l * h->chans[n - b]);
    }
  }
  SATB_PROPAGATE(h->ensure(&h->buf_raw, &h->cap_raw, max_elems * 4));
  h->lo_off = h->split3 ? ((max_elems * 2 + 255) & ~static_cast<size_t>(255)) : 0;   // [hi | lo] halves of sA / sB
  SATB_PROPAGATE(h->ensure(&h->buf_a, &h->cap_a, max_elems * 2 + h->lo_off));
  SATB_PROPAGATE(h->ensure(&h->buf_b, &h->cap_b, max_elems * 2 + h->lo_off));
  void* raw = h->buf_raw;
  void* sA = h->buf_a;
  void* sB = h->buf_b;
  SATB_PROPAGATE((dec_input<BF16, ACT>(h, z, sB, sA, B, L, st)));
  int64_t Lc = L;
  for (int b = 1; b <= n; ++b) {
    // transposed conv reads sA [B, Lc, cin], writes raw + snake(ru0) into sB
    SATB_PROPAGATE((dec_upsample<BF16, ACT>(h, b, sA, raw, sB, B, static_cast<int>(Lc), st)));
    std::swap(sA, sB);  // sA now holds the residual units' input
    Lc *= c.strides[n - b];
    for (int j = 0; j < 3; ++j) SATB_PROPAGATE((dec_residual<BF16, ACT>(h, b, j, B, static_cast<int>(Lc), raw, sA, sB, st)));
  }
  SATB_PROPAGATE(dec_output<BF16>(h, sA, audio, B, static_cast<int>(Lc), st));
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

template <bool BF16, int ACT>
int encode_impl(SatbOobleck* h, const float* audio, float* latents, int B, int64_t T, cudaStream_t st) {
  const SatbOobleckConfig& c = h->cfg;
  const int n = c.n_stages;
  int64_t ratio = 1;
  for (int i = 0; i < n; ++i) ratio *= c.strides[i];
  SATB_REQUIRE(T % ratio == 0, "encoder: audio length must be a multiple of the downsampling ratio");
  SATB_REQUIRE(T < (int64_t(1) << 31), "encoder: sequence too long");
  size_t max_elems = static_cast<size_t>(B) * T * c.in_channels;   // a wide input conv's 16-bit copy
  {
    int64_t l = T;
    for (int i = 0; i <= n; ++i) {
      max_elems = std::max(max_elems, static_cast<size_t>(B) * l * h->chans[i]);
      if (i < n) l /= c.strides[i];
    }
  }
  SATB_PROPAGATE(h->ensure(&h->buf_raw, &h->cap_raw, max_elems * 4));
  h->lo_off = h->split3 ? ((max_elems * 2 + 255) & ~static_cast<size_t>(255)) : 0;   // [hi | lo] halves of sA / sB
  SATB_PROPAGATE(h->ensure(&h->buf_a, &h->cap_a, max_elems * 2 + h->lo_off));
  SATB_PROPAGATE(h->ensure(&h->buf_b, &h->cap_b, max_elems * 2 + h->lo_off));
  void* raw = h->buf_raw;
  void* sA = h->buf_a;
  void* sB = h->buf_b;
  SATB_PROPAGATE((enc_input<BF16, ACT>(h, audio, raw, sA, sB, B, T, st)));
  int64_t Lc = T;
  for (int b = 1; b <= n; ++b) {
    for (int j = 0; j < 3; ++j) SATB_PROPAGATE((enc_residual<BF16, ACT>(h, b, j, B, static_cast<int>(Lc), raw, sA, sB, st)));
    // strided conv reads sA [B, Lc, cin] -> [B, Lc/s, cout] in sB
    SATB_PROPAGATE((enc_downsample<BF16, ACT>(h, b, sA, raw, sB, B, static_cast<int>(Lc), st)));
    std::swap(sA, sB);
    Lc /= c.strides[b - 1];
  }
  SATB_PROPAGATE(enc_output<BF16>(h, sA, latents, B, static_cast<int>(Lc), st));
  return 0;
}

// One step on caller-owned buffers (satb_oobleck_probe).
template <bool BF16, int ACT>
int probe_impl(SatbOobleck* h, SatbOobleckProbe* p, cudaStream_t st) {
  const int b = p->block, j = p->unit, B = p->B, L = p->L;
  if (p->step == SATB_OOB_DEC_RES || p->step == SATB_OOB_ENC_RES) {
    const bool dec = p->step == SATB_OOB_DEC_RES;
    const int C = h->chans[dec ? h->cfg.n_stages - b : b - 1];
    if (p->raw_in != p->raw_out)
      SATB_CHECK_CUDA(cudaMemcpyAsync(p->raw_out, p->raw_in, static_cast<size_t>(B) * L * C * (h->raw16 ? 2 : 4),
                                      cudaMemcpyDeviceToDevice, st));
    void* sA = p->in;
    void* sT = p->scratch;
    SATB_PROPAGATE((dec ? dec_residual<BF16, ACT>(h, b, j, B, L, p->raw_out, sA, sT, st)
                       : enc_residual<BF16, ACT>(h, b, j, B, L, p->raw_out, sA, sT, st)));
    p->result_in_scratch = sA == p->scratch;
    return 0;
  }
  switch (p->step) {
    case SATB_OOB_DEC_IN: return dec_input<BF16, ACT>(h, static_cast<const float*>(p->in), p->scratch, p->out16, B, L, st);
    case SATB_OOB_DEC_UP: return dec_upsample<BF16, ACT>(h, b, p->in, p->raw_out, p->out16, B, L, st);
    case SATB_OOB_DEC_OUT: return dec_output<BF16>(h, p->in, p->out32, B, L, st);
    case SATB_OOB_ENC_IN:
      return enc_input<BF16, ACT>(h, static_cast<const float*>(p->in), p->raw_out, p->out16, p->scratch, B, L, st);
    case SATB_OOB_ENC_DOWN: return enc_downsample<BF16, ACT>(h, b, p->in, p->raw_out, p->out16, B, L, st);
    default: return enc_output<BF16>(h, p->in, p->out32, B, L, st);
  }
}

template <int ACT>
int decode_act(SatbOobleck* h, const float* z, float* audio, int B, int L, cudaStream_t st) {
  return h->bf16 ? decode_impl<true, ACT>(h, z, audio, B, L, st) : decode_impl<false, ACT>(h, z, audio, B, L, st);
}
template <int ACT>
int encode_act(SatbOobleck* h, const float* audio, float* latents, int B, int64_t T, cudaStream_t st) {
  return h->bf16 ? encode_impl<true, ACT>(h, audio, latents, B, T, st) : encode_impl<false, ACT>(h, audio, latents, B, T, st);
}
template <int ACT>
int probe_act(SatbOobleck* h, SatbOobleckProbe* p, cudaStream_t st) {
  return h->bf16 ? probe_impl<true, ACT>(h, p, st) : probe_impl<false, ACT>(h, p, st);
}

}  // namespace

extern "C" {

int satb_oobleck_create(const SatbOobleckConfig* cfg, SatbOobleck** out) {
  return satb_oobleck_create_variant(cfg, SATB_OOB_ACT_SNAKE, 0, out);
}

int satb_oobleck_create_variant(const SatbOobleckConfig* cfg, int activation, int nearest_upsample, SatbOobleck** out) {
  SATB_REQUIRE(cfg && out, "null argument");
  SATB_REQUIRE(cfg->n_stages >= 1 && cfg->n_stages <= SATB_MAX_STAGES, "bad number of stages");
  SATB_REQUIRE(cfg->channels % 32 == 0, "channels must be a multiple of 32");
  SATB_REQUIRE(cfg->latent_dim % 8 == 0, "latent_dim must be a multiple of 8");
  if (!(cfg->in_channels >= 1 && cfg->in_channels <= 2) &&
      !(cfg->in_channels % 8 == 0 && cfg->in_channels >= 8 && cfg->in_channels <= 128)) {
    set_last_error("oobleck: in_channels must be 1, 2 (audio) or a multiple of 8 up to 128 (PQMF sub-bands), got " +
                   std::to_string(cfg->in_channels));
    return -1;
  }
  if (activation != SATB_OOB_ACT_SNAKE && activation != SATB_OOB_ACT_ELU) {
    set_last_error("oobleck: unknown activation " + std::to_string(activation) + "; accepted: 0 (snake), 1 (elu)");
    return -1;
  }
  if (nearest_upsample != 0 && nearest_upsample != 1) {
    set_last_error("oobleck: nearest_upsample must be 0 or 1, got " + std::to_string(nearest_upsample));
    return -1;
  }
  SATB_REQUIRE(!nearest_upsample || cfg->is_decoder,
               "oobleck: nearest_upsample applies to a decoder only (an encoder has no upsampling)");
  // A block's conv has kernel 2s, stride s, padding ceil(s/2) (models/autoencoders.py:75,86).  Its output length is
  // L * s (decoder) and L / s (encoder) only for an even decoder stride and an encoder stride >= 2: an odd decoder
  // stride gives L * s - 1, encoder stride 1 gives L + 1.  Nearest upsampling followed by a 'same' conv gives L * s
  // for every s.
  for (int i = 0; i < cfg->n_stages; ++i) {
    const int s = cfg->strides[i];
    if (cfg->is_decoder && nearest_upsample) {
      if (s < 2) {
        set_last_error("decoder: stride " + std::to_string(s) + " is not supported: nearest upsampling needs strides >= 2");
        return -1;
      }
    } else if (cfg->is_decoder ? (s < 2 || s % 2 != 0) : s < 2) {
      set_last_error(std::string(cfg->is_decoder ? "decoder" : "encoder") + ": stride " + std::to_string(s) +
                     " is not supported: " +
                     (cfg->is_decoder ? "strides must be even (a transposed conv with kernel 2s, padding ceil(s/2) "
                                        "gives L * s positions only for even s)"
                                      : "strides must be >= 2 (a conv with kernel 2s, padding ceil(s/2) gives L / s "
                                        "positions only for s >= 2)"));
      return -1;
    }
  }
  SatbOobleck* h = new SatbOobleck();
  h->cfg = *cfg;
  h->act = activation == SATB_OOB_ACT_ELU ? kActElu : kActSnake;
  h->nearest = nearest_upsample != 0;
  h->bf16 = cfg->operand_dtype == 1;
  h->split3 = cfg->operand_dtype == 2;
  // fp16 operands: the un-activated skip stream is carried in fp16 as well (8 instead of 12 bytes per element and
  // channel through a fused ResidualUnit; measured +23 % on the fp16-operand error floor, tests/test_gpu_baseline_size).
  // bf16 (8 mantissa bits) keeps the fp32 stream.
  h->raw16 = (!h->bf16 && !h->split3) ? 1 : 0;
  h->chans.push_back(cfg->channels);
  for (int i = 0; i < cfg->n_stages; ++i) h->chans.push_back(cfg->c_mults[i] * cfg->channels);
  *out = h;
  return 0;
}

void satb_oobleck_destroy(SatbOobleck* h) {
  if (!h) return;
  for (void* p : h->owned) cudaFree(p);
  for (auto& kv : h->raw) cudaFree(kv.second.first);
  if (h->buf_raw) cudaFree(h->buf_raw);
  if (h->buf_a) cudaFree(h->buf_a);
  if (h->buf_b) cudaFree(h->buf_b);
  delete h;
}

int satb_oobleck_load_weight(SatbOobleck* h, const char* name, const float* src, long long numel, void* stream) {
  SATB_REQUIRE(h && name && src && numel > 0, "bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto it = h->raw.find(name);
  if (it != h->raw.end() && it->second.second != numel) {
    cudaFree(it->second.first);
    h->raw.erase(it);
    it = h->raw.end();
  }
  float* dst;
  if (it == h->raw.end()) {
    SATB_CHECK_CUDA(cudaMalloc(&dst, numel * sizeof(float)));
    h->raw[name] = std::make_pair(dst, numel);
  } else {
    dst = it->second.first;
  }
  SATB_CHECK_CUDA(cudaMemcpyAsync(dst, src, numel * sizeof(float), cudaMemcpyDeviceToDevice, st));
  h->finalized = false;
  return 0;
}

int satb_oobleck_finalize(SatbOobleck* h, void* stream) {
  SATB_REQUIRE(h, "null handle");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const SatbOobleckConfig& c = h->cfg;
  const int n = c.n_stages;
  for (void* p : h->owned) cudaFree(p);
  h->owned.clear();
  h->convs.clear();
  h->snakes.clear();
  h->tmaps.clear();
  auto res_unit = [&](const std::string& pfx, int C) -> int {
    SATB_PROPAGATE(prep_snake(h, pfx + "layers.0.", C, st));
    SATB_PROPAGATE(prep_conv(h, pfx + "layers.1.", C, C, 7, false, false, true, 1, st));
    SATB_PROPAGATE(prep_snake(h, pfx + "layers.2.", C, st));
    SATB_PROPAGATE(prep_conv(h, pfx + "layers.3.", C, C, 1, false, false, true, 1, st));
    return 0;
  };
  if (c.is_decoder) {
    SATB_PROPAGATE(prep_conv(h, "layers.0.", c.latent_dim, h->chans[n], 7, false, false, true, 1, st));
    for (int b = 1; b <= n; ++b) {
      const int cin = h->chans[n - b + 1], cout = h->chans[n - b], s = c.strides[n - b];
      const std::string bp = "layers." + std::to_string(b) + ".";
      SATB_PROPAGATE(prep_snake(h, bp + "layers.0.", cin, st));
      if (h->nearest)
        SATB_PROPAGATE(prep_conv_nearest(h, bp + "layers.1.1.", cin, cout, s, st));
      else
        SATB_PROPAGATE(prep_conv(h, bp + "layers.1.", cin, cout, 2 * s, true, false, true, s, st));
      for (int j = 0; j < 3; ++j) SATB_PROPAGATE(res_unit(bp + "layers." + std::to_string(2 + j) + ".", cout));
    }
    SATB_PROPAGATE(prep_snake(h, "layers." + std::to_string(n + 1) + ".", h->chans[0], st));
    SATB_PROPAGATE(prep_conv(h, "layers." + std::to_string(n + 2) + ".", h->chans[0], c.in_channels, 7, false, false, false, 1, st));
    SATB_REQUIRE(h->chans[0] % 2 == 0, "decoder: channels must be even");
  } else {
    SATB_PROPAGATE(prep_conv(h, "layers.0.", c.in_channels, h->chans[0], 7, false, c.in_channels <= 2, true, 1, st));
    for (int b = 1; b <= n; ++b) {
      const int cin = h->chans[b - 1], cout = h->chans[b], s = c.strides[b - 1];
      const std::string bp = "layers." + std::to_string(b) + ".";
      for (int j = 0; j < 3; ++j) SATB_PROPAGATE(res_unit(bp + "layers." + std::to_string(j) + ".", cin));
      SATB_PROPAGATE(prep_snake(h, bp + "layers.3.", cin, st));
      SATB_PROPAGATE(prep_conv(h, bp + "layers.4.", cin, cout, 2 * s, false, false, true, 1, st));
    }
    SATB_PROPAGATE(prep_snake(h, "layers." + std::to_string(n + 1) + ".", h->chans[n], st));
    SATB_PROPAGATE(prep_conv(h, "layers." + std::to_string(n + 2) + ".", h->chans[n], c.latent_dim, 3, false, false, true, 1, st));
  }
  SATB_CHECK_CUDA(cudaStreamSynchronize(st));
  h->finalized = true;
  return 0;
}

int satb_oobleck_decode(SatbOobleck* h, const float* z, float* audio, int B, int L, void* stream) {
  SATB_REQUIRE(h && h->finalized, "oobleck: weights not finalized");
  SATB_REQUIRE(h->cfg.is_decoder, "oobleck: handle is an encoder");
  SATB_REQUIRE(z && audio && B >= 1 && L >= 1, "bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return h->act == kActElu ? decode_act<kActElu>(h, z, audio, B, L, st) : decode_act<kActSnake>(h, z, audio, B, L, st);
}

int satb_oobleck_encode(SatbOobleck* h, const float* audio, float* latents, int B, long long T, void* stream) {
  SATB_REQUIRE(h && h->finalized, "oobleck: weights not finalized");
  SATB_REQUIRE(!h->cfg.is_decoder, "oobleck: handle is a decoder");
  SATB_REQUIRE(audio && latents && B >= 1 && T >= 1, "bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return h->act == kActElu ? encode_act<kActElu>(h, audio, latents, B, T, st)
                           : encode_act<kActSnake>(h, audio, latents, B, T, st);
}

int satb_oobleck_probe(SatbOobleck* h, SatbOobleckProbe* p, void* stream) {
  SATB_REQUIRE(h && h->finalized && p, "oobleck probe: needs a finalized handle and a parameter block");
  const bool dec = h->cfg.is_decoder != 0;
  const int n = h->cfg.n_stages;
  const int step = p->step;
  if (dec ? (step < SATB_OOB_DEC_IN || step > SATB_OOB_DEC_OUT) : (step < SATB_OOB_ENC_IN || step > SATB_OOB_ENC_OUT)) {
    set_last_error(std::string("oobleck probe: unknown step ") + std::to_string(step) + " for " +
                   (dec ? "a decoder; accepted: DEC_IN 0, DEC_UP 1, DEC_RES 2, DEC_OUT 3"
                        : "an encoder; accepted: ENC_IN 4, ENC_RES 5, ENC_DOWN 6, ENC_OUT 7"));
    return -1;
  }
  const bool res = step == SATB_OOB_DEC_RES || step == SATB_OOB_ENC_RES;
  const bool blocked = res || step == SATB_OOB_DEC_UP || step == SATB_OOB_ENC_DOWN;
  if ((blocked && (p->block < 1 || p->block > n)) || (res && (p->unit < 0 || p->unit > 2))) {
    set_last_error("oobleck probe: block " + std::to_string(p->block) + " unit " + std::to_string(p->unit) +
                   " out of range; accepted: block 1 .. " + std::to_string(n) + ", unit 0 .. 2 (ResidualUnit steps)");
    return -1;
  }
  SATB_REQUIRE(p->B >= 1 && p->L >= 1, "oobleck probe: B and L must be >= 1");
  SATB_REQUIRE(!h->split3 || (p->lo_off > 0 && p->lo_off % 16 == 0),
               "oobleck probe: fp16x3 needs lo_off, a positive multiple of 16 bytes");
  if (step == SATB_OOB_ENC_DOWN) {
    const int s = h->cfg.strides[p->block - 1];
    if (p->L % s != 0) {
      set_last_error("oobleck probe: strided conv input length " + std::to_string(p->L) +
                     " is not a multiple of the stride " + std::to_string(s));
      return -1;
    }
  }
  // the buffers each step uses (see include/satb200.h)
  const bool raw_out = step == SATB_OOB_DEC_UP || step == SATB_OOB_ENC_IN || step == SATB_OOB_ENC_DOWN || res;
  const bool out16 = step == SATB_OOB_DEC_IN || step == SATB_OOB_DEC_UP || step == SATB_OOB_ENC_IN || step == SATB_OOB_ENC_DOWN;
  const bool out32 = step == SATB_OOB_DEC_OUT || step == SATB_OOB_ENC_OUT;
  const bool scratch = step == SATB_OOB_DEC_IN || res || (step == SATB_OOB_ENC_IN && h->cfg.in_channels > 2);
  const struct { const char* name; const void* ptr; bool used; } bufs[] = {
      {"in", p->in, true}, {"raw_in", p->raw_in, res}, {"raw_out", p->raw_out, raw_out},
      {"out16", p->out16, out16}, {"scratch", p->scratch, scratch}, {"out32", p->out32, out32}};
  for (const auto& bf : bufs) {
    if (bf.used && (bf.ptr == nullptr || reinterpret_cast<uintptr_t>(bf.ptr) % 16 != 0)) {
      set_last_error(std::string("oobleck probe: ") + bf.name + " must be a non-null, 16-byte aligned device pointer");
      return -1;
    }
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  h->lo_off = h->split3 ? static_cast<size_t>(p->lo_off) : 0;
  h->routes = 0;
  p->result_in_scratch = 0;
  const int rc = h->act == kActElu ? probe_act<kActElu>(h, p, st) : probe_act<kActSnake>(h, p, st);
  p->wrote_raw = h->wrote_raw ? 1 : 0;
  p->routes = static_cast<int>(h->routes);
  SATB_PROPAGATE(rc);
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int satb_oobleck_weights(SatbOobleck* h, const char* prefix, void* dst, long long* bytes, void* stream) {
  SATB_REQUIRE(h && h->finalized && prefix && bytes, "oobleck weights: needs a finalized handle, a prefix and bytes");
  auto it = h->convs.find(prefix);
  if (it == h->convs.end()) {
    set_last_error(std::string("oobleck weights: no conv ") + prefix);
    return -1;
  }
  const ConvW& c = it->second;
  const size_t total = conv_w_elems(c);
  const size_t n = c.small ? total * 4 : total * 2 * (h->split3 ? 2 : 1);
  *bytes = static_cast<long long>(n);
  if (dst) {
    SATB_CHECK_CUDA(cudaMemcpyAsync(dst, c.small ? static_cast<const void*>(c.w32) : static_cast<const void*>(c.w16), n,
                                    cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  }
  return 0;
}

}  // extern "C"

// ---- Time-sharded decode / encode: one process drives `world` ranks, each a finalized handle with a full copy of the
// weights on its device (several ranks may share a device).  Rank r computes latents begin[r] .. begin[r + 1] - 1 of
// every item (their samples for the encoder) by running the ordinary single-device decode / encode on an extended
// slice: its range plus a recompute margin of m latents on each interior side, clipped to the item.  Every kept output
// position then reads the same inputs through the same arithmetic as on one device:
//   * each convolution's output at a position is its k-block x tap accumulation of its own input rows, in the same
//     order for every row of a tile; the tile a row falls in decides nothing (no split-K, no per-tile fast path: the
//     lean epilogue runs the same arithmetic on ragged chunks, and its choice against the general one is per launch);
//   * the route of each layer (fused ResidualUnit, halo-tile final conv, implicit GEMM and its N tile, CUDA-core input
//     conv) depends on the channels, taps, dilation and operand mode only, which are the same on every rank;
//   * an extended slice starts at a whole latent, so at every level of the decoder (encoder) its first position is a
//     multiple of that level's cumulative stride: the transposed convs' phases and the strided convs' taps line up.
// Only the positions within the margin of a slice's interior ends see zeros in place of a neighbour's data, and the
// margin is the receptive field in latents, so none of them is kept.  Recomputing the margin needs no change to any
// convolution kernel or tensor-map route, where a per-layer halo exchange would need one per layer and route.

namespace {

int64_t floor_div(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// The receptive field of one latent (decoder: the latents any output sample of latent 0 reads; encoder: the latents
// whose samples latent 0 reads, in whole latents) on either side, from the layer list: k7 input conv, per block the
// up / down conv and three k7 ResidualUnits at dilations 1, 3, 9 (3 + 9 + 27 positions each way), the final conv (k7
// decoder, k3 encoder).  The interval of positions a layer's outputs [lo, hi] read is walked back from the output.
int receptive_margin(const SatbOobleckConfig& c, bool nearest) {
  const int n = c.n_stages;
  int64_t ratio = 1;
  for (int i = 0; i < n; ++i) ratio *= c.strides[i];
  constexpr int kResUnits = 3 * (1 + 3 + 9);
  if (c.is_decoder) {
    int64_t lo = -3, hi = ratio - 1 + 3;                     // the final conv k7 over the samples of latent 0
    for (int b = n; b >= 1; --b) {
      const int s = c.strides[n - b];
      lo -= kResUnits;
      hi += kResUnits;
      if (nearest) {                                         // output s m + ph reads m - 1 .. m + 1
        lo = floor_div(lo, s) - 1;
        hi = floor_div(hi, s) + 1;
      } else {                                               // output o reads l - 1, l with l = floor((o + pad) / s)
        const int p = (s + 1) / 2;
        lo = floor_div(lo + p, s) - 1;
        hi = floor_div(hi + p, s);
      }
    }
    lo -= 3;                                                 // the input conv k7
    hi += 3;
    return static_cast<int>(std::max(-lo, hi));
  }
  int64_t lo = -1, hi = 1;                                   // the final conv k3 around latent 0
  for (int b = n; b >= 1; --b) {
    const int s = c.strides[b - 1], p = (s + 1) / 2;         // output o reads o s - p .. o s - p + 2 s - 1
    lo = lo * s - p - kResUnits;
    hi = hi * s - p + 2 * s - 1 + kResUnits;
  }
  lo -= 3;                                                   // the input conv k7
  hi += 3;
  return static_cast<int>(std::max(floor_div(-lo + ratio - 1, ratio), floor_div(hi - (ratio - 1) + ratio - 1, ratio)));
}

}  // namespace

extern "C" int satb_oobleck_group_plan(int world, int L, const SatbOobleckConfig* cfg, int nearest_upsample,
                                       int* begin, int* ext, int* margin) {
  SATB_REQUIRE(cfg && begin && ext && margin, "null argument");
  SATB_REQUIRE(world >= 1 && world <= kKvGatherMaxRanks, "world must be 1 .. 8");
  SATB_REQUIRE(L >= 1, "need L >= 1");
  SATB_REQUIRE(cfg->n_stages >= 1 && cfg->n_stages <= SATB_MAX_STAGES, "bad number of stages");
  for (int i = 0; i < cfg->n_stages; ++i) SATB_REQUIRE(cfg->strides[i] >= 2, "strides must be >= 2");
  SATB_REQUIRE(nearest_upsample == 0 || (nearest_upsample == 1 && cfg->is_decoder),
               "nearest_upsample must be 0, or 1 for a decoder");
  if (world > L) {
    set_last_error("world " + std::to_string(world) + " exceeds the " + std::to_string(L) +
                   " latents of an item: every rank needs at least one latent");
    return -1;
  }
  const int m = receptive_margin(*cfg, nearest_upsample != 0);
  for (int r = 0; r <= world; ++r) begin[r] = static_cast<int>(static_cast<int64_t>(r) * L / world);
  for (int r = 0; r < world; ++r) {
    const int n = begin[r + 1] - begin[r];
    if (world > 1 && n < m) {
      set_last_error("rank " + std::to_string(r) + " would hold " + std::to_string(n) + " of the " + std::to_string(L) +
                     " latents, fewer than the recompute margin of " + std::to_string(m) +
                     " latents each rank recomputes on each interior side: use fewer ranks or a longer clip");
      return -1;
    }
    ext[2 * r] = std::max(begin[r] - m, 0);
    ext[2 * r + 1] = std::min(begin[r + 1] + m, L);
  }
  *margin = m;
  return 0;
}

struct SatbOobleckGroup {
  int world = 0;
  std::vector<SatbOobleck*> h;
  std::vector<int> dev;
  std::vector<cudaStream_t> st;        // per rank, on its device (the library's own)
  std::vector<cudaEvent_t> ev_done;    // per rank: its decode / encode of the last call done
  std::vector<DevBuf> in, out;         // per rank, on its device: the extended slice's input and output
  cudaEvent_t ev_in = nullptr;         // home device: the caller's stream reached the call (its input is ready)
  cudaEvent_t ev_gathered = nullptr;   // home device: the last call's gather done
};

namespace {

void group_release(SatbOobleckGroup* g) {
  int cur = 0;
  cudaGetDevice(&cur);
  if (g->ev_gathered) cudaEventSynchronize(g->ev_gathered);   // the last gather may still read the ranks' outputs
  for (int r = 0; r < g->world; ++r) {
    cudaSetDevice(g->dev[r]);
    if (r < static_cast<int>(g->st.size()) && g->st[r]) cudaStreamSynchronize(g->st[r]);
    if (r < static_cast<int>(g->in.size())) g->in[r].release();
    if (r < static_cast<int>(g->out.size())) g->out[r].release();
    if (r < static_cast<int>(g->ev_done.size()) && g->ev_done[r]) cudaEventDestroy(g->ev_done[r]);
    if (r < static_cast<int>(g->st.size()) && g->st[r]) cudaStreamDestroy(g->st[r]);
  }
  if (g->world > 0) {
    cudaSetDevice(g->dev[0]);
    if (g->ev_in) cudaEventDestroy(g->ev_in);
    if (g->ev_gathered) cudaEventDestroy(g->ev_gathered);
  }
  cudaSetDevice(cur);
}

struct CurrentDeviceRestore {
  int cur = 0;
  CurrentDeviceRestore() { cudaGetDevice(&cur); }
  ~CurrentDeviceRestore() { cudaSetDevice(cur); }
};

// One sharded call.  Ordered with events only:
//   RAW: each rank's input copy waits for the caller's stream (ev_in); the gather waits for every rank (ev_done).
//   WAR: each rank's work waits for the previous call's gather (ev_gathered), which reads the rank's output buffer.
// The input slices are 2-D copies on the rank streams (the copy engines move a strided slice over the peer link without
// taking SMs from the rank's decode, as the DiT group graph's copies do); the gather is a kernel on the home device.
int group_run(SatbOobleckGroup* g, bool dec, const float* in, float* out, int B, int L, cudaStream_t home) {
  SatbOobleck* h0 = g->h[0];
  const SatbOobleckConfig& c = h0->cfg;
  const int W = g->world;
  int begin[kKvGatherMaxRanks + 1], ext[2 * kKvGatherMaxRanks], m = 0;
  SATB_PROPAGATE(satb_oobleck_group_plan(W, L, &c, h0->nearest ? 1 : 0, begin, ext, &m));
  int64_t ratio = 1;
  for (int i = 0; i < c.n_stages; ++i) ratio *= c.strides[i];
  // per latent: positions of the input and the output; and their channels
  const int64_t in_rate = dec ? 1 : ratio, out_rate = dec ? ratio : 1;
  const int in_ch = dec ? c.latent_dim : c.in_channels, out_ch = dec ? c.in_channels : c.latent_dim;
  SATB_REQUIRE(static_cast<int64_t>(L) * ratio < (int64_t(1) << 31), "sequence too long");
  CurrentDeviceRestore restore;
  for (int r = 0; r < W; ++r) {   // workspaces at the extended shape; growing one waits for the gather that reads it
    const int64_t n = ext[2 * r + 1] - ext[2 * r];
    const size_t need_in = static_cast<size_t>(B) * in_ch * n * in_rate * 4;
    const size_t need_out = static_cast<size_t>(B) * out_ch * n * out_rate * 4;
    if (need_in > g->in[r].bytes || need_out > g->out[r].bytes) {
      SATB_CHECK_CUDA(cudaEventSynchronize(g->ev_gathered));
      SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
      SATB_PROPAGATE(g->in[r].ensure(need_in));
      SATB_PROPAGATE(g->out[r].ensure(need_out));
    }
  }
  SATB_CHECK_CUDA(cudaSetDevice(g->dev[0]));
  SATB_CHECK_CUDA(cudaEventRecord(g->ev_in, home));
  for (int r = 0; r < W; ++r) {
    const int64_t e0 = ext[2 * r], n = ext[2 * r + 1] - e0;
    SATB_CHECK_CUDA(cudaSetDevice(g->dev[r]));
    SATB_CHECK_CUDA(cudaStreamWaitEvent(g->st[r], g->ev_in, 0));         // RAW: the input
    SATB_CHECK_CUDA(cudaStreamWaitEvent(g->st[r], g->ev_gathered, 0));   // WAR: the previous gather read out[r]
    SATB_CHECK_CUDA(cudaMemcpy2DAsync(g->in[r].p, static_cast<size_t>(n * in_rate) * 4, in + e0 * in_rate,
                                      static_cast<size_t>(L * in_rate) * 4, static_cast<size_t>(n * in_rate) * 4,
                                      static_cast<size_t>(B) * in_ch, cudaMemcpyDefault, g->st[r]));
    if (dec)
      SATB_PROPAGATE(satb_oobleck_decode(g->h[r], g->in[r].as<float>(), g->out[r].as<float>(), B, static_cast<int>(n),
                                         g->st[r]));
    else
      SATB_PROPAGATE(satb_oobleck_encode(g->h[r], g->in[r].as<float>(), g->out[r].as<float>(), B, n * ratio, g->st[r]));
    SATB_CHECK_CUDA(cudaEventRecord(g->ev_done[r], g->st[r]));
  }
  SATB_CHECK_CUDA(cudaSetDevice(g->dev[0]));
  const float* src[kKvGatherMaxRanks];
  int src_len[kKvGatherMaxRanks], src_off[kKvGatherMaxRanks], ob[kKvGatherMaxRanks + 1];
  for (int r = 0; r < W; ++r) {
    SATB_CHECK_CUDA(cudaStreamWaitEvent(home, g->ev_done[r], 0));         // RAW: rank r's output
    src[r] = g->out[r].as<float>();
    src_len[r] = static_cast<int>((ext[2 * r + 1] - ext[2 * r]) * out_rate);
    src_off[r] = static_cast<int>((begin[r] - ext[2 * r]) * out_rate);
    ob[r] = static_cast<int>(begin[r] * out_rate);
  }
  ob[W] = static_cast<int>(L * out_rate);
  SATB_PROPAGATE(launch_time_gather(src, src_len, src_off, ob, W, out, B * out_ch, ob[W], home));
  SATB_CHECK_CUDA(cudaEventRecord(g->ev_gathered, home));
  return 0;
}

}  // namespace

extern "C" {

int satb_oobleck_group_create(SatbOobleck* const* handles, const int* devices, int world, SatbOobleckGroup** out) {
  SATB_REQUIRE(handles && devices && out, "null argument");
  SATB_REQUIRE(world >= 1 && world <= kKvGatherMaxRanks, "world must be 1 .. 8");
  for (int r = 0; r < world; ++r) {
    SATB_REQUIRE(handles[r], "null handle");
    const SatbOobleck* a = handles[0];
    const SatbOobleck* b = handles[r];
    if (std::memcmp(&a->cfg, &b->cfg, sizeof(SatbOobleckConfig)) != 0 || a->act != b->act || a->nearest != b->nearest) {
      set_last_error("rank " + std::to_string(r) + "'s handle has another config or block option than rank 0's");
      return -1;
    }
    for (int s = 0; s < r; ++s)
      SATB_REQUIRE(handles[s] != handles[r], "every rank needs its own handle (its own workspace)");
  }
  for (int r = 0; r < world; ++r) SATB_REQUIRE(handles[r]->finalized, "weights not finalized");
  CurrentDeviceRestore restore;
  int n_dev = 0;
  SATB_CHECK_CUDA(cudaGetDeviceCount(&n_dev));
  for (int r = 0; r < world; ++r) SATB_REQUIRE(devices[r] >= 0 && devices[r] < n_dev, "no such device");
  // the home device reads every rank's output, and every rank copies its input slice from the home device
  for (int r = 1; r < world; ++r) {
    if (devices[r] == devices[0]) continue;
    for (const auto& pr : {std::make_pair(devices[0], devices[r]), std::make_pair(devices[r], devices[0])}) {
      int ok = 0;
      SATB_CHECK_CUDA(cudaDeviceCanAccessPeer(&ok, pr.first, pr.second));
      if (!ok) {
        set_last_error("device " + std::to_string(pr.first) + " cannot access device " + std::to_string(pr.second) +
                       " peer to peer: the time-sharded decode gathers every rank's output over peer links");
        return -1;
      }
      SATB_CHECK_CUDA(cudaSetDevice(pr.first));
      const cudaError_t e = cudaDeviceEnablePeerAccess(pr.second, 0);   // this process's context only
      if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();
      } else {
        SATB_CHECK_CUDA(e);
      }
    }
  }
  SatbOobleckGroup* g = new SatbOobleckGroup();
  g->world = world;
  g->h.assign(handles, handles + world);
  g->dev.assign(devices, devices + world);
  g->st.assign(world, nullptr);
  g->ev_done.assign(world, nullptr);
  g->in.resize(world);
  g->out.resize(world);
  cudaError_t e = cudaSuccess;
  for (int r = 0; r < world && e == cudaSuccess; ++r) {
    e = cudaSetDevice(devices[r]);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&g->st[r], cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_done[r], cudaEventDisableTiming);
  }
  if (e == cudaSuccess) e = cudaSetDevice(devices[0]);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_in, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_gathered, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    group_release(g);
    delete g;
    set_last_error(std::string("satb_oobleck_group_create: ") + cudaGetErrorString(e));
    return -2;
  }
  *out = g;
  return 0;
}

void satb_oobleck_group_destroy(SatbOobleckGroup* g) {
  if (!g) return;
  group_release(g);
  delete g;
}

int satb_oobleck_group_decode(SatbOobleckGroup* g, const float* z, float* audio, int B, int L, void* stream) {
  SATB_REQUIRE(g && z && audio && B >= 1 && L >= 1, "bad argument");
  for (int r = 0; r < g->world; ++r) SATB_REQUIRE(g->h[r]->finalized, "oobleck: weights not finalized");
  SATB_REQUIRE(g->h[0]->cfg.is_decoder, "oobleck group: the handles are encoders");
  return group_run(g, true, z, audio, B, L, static_cast<cudaStream_t>(stream));
}

int satb_oobleck_group_encode(SatbOobleckGroup* g, const float* audio, float* latents, int B, long long T, void* stream) {
  SATB_REQUIRE(g && audio && latents && B >= 1 && T >= 1, "bad argument");
  for (int r = 0; r < g->world; ++r) SATB_REQUIRE(g->h[r]->finalized, "oobleck: weights not finalized");
  SATB_REQUIRE(!g->h[0]->cfg.is_decoder, "oobleck group: the handles are decoders");
  int64_t ratio = 1;
  for (int i = 0; i < g->h[0]->cfg.n_stages; ++i) ratio *= g->h[0]->cfg.strides[i];
  SATB_REQUIRE(T % ratio == 0, "encoder: audio length must be a multiple of the downsampling ratio");
  SATB_REQUIRE(T / ratio < (int64_t(1) << 31), "encoder: sequence too long");
  return group_run(g, false, audio, latents, B, static_cast<int>(T / ratio), static_cast<cudaStream_t>(stream));
}

}  // extern "C"
