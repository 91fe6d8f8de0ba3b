// wgmma / TMA GEMM for sm_90a with fused epilogues.
//
//   C[row, n] = sum_{tap, k} A[batch, l + tap_base + tap*tap_step, k] * B[tap*b_tap_rows + n, k]
//
// A is a K-major 16-bit activation matrix viewed as (K, phase, L, batches) through a
// 4-D TMA tensor map (position = row*stride + phase; out-of-range rows are zero-filled
// by TMA, which is how convolution padding and the ragged M tail are handled); B is the
// K-major weight matrix [taps * N, K].  A plain Linear layer is n_taps = 1,
// batches = 1.  Accumulation is fp32 in registers.
//
// Structure (one persistent CTA per SM, 384 threads, 128 x BN tiles):
//   warpgroup 0      TMA producer      one thread: global -> 128B-swizzled smem ring (mbarrier full/empty)
//   warpgroups 1, 2  MMA + epilogue    64 rows each: wgmma 64xBNx16 from the smem ring into registers, then the
//                                      fused epilogue (accumulator -> smem -> one row per thread -> fused op -> global)
// The producer runs ahead into the next tile's k-blocks while the epilogue of the current one runs.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"

namespace satb {

// Order of the split-operand parts: the two small cross terms (lo, hi), (hi, lo) are accumulated FIRST, into a still
// small accumulator, and the (hi, hi) chain last: the tensor core truncates when it aligns addends to the accumulator,
// so adding 2^-11-sized terms to a full-sized sum costs about one accumulator ulp per k-step each.
__device__ __forceinline__ int split_part(int idx, int n_parts) { return n_parts == 3 ? (idx == 2 ? 0 : idx + 1) : idx; }

struct GemmShape {
  int L;            // rows per batch
  int batches;      // number of batches (1 for flat GEMMs)
  int N;            // output columns
  int K;            // reduction length per tap (multiple of 8)
  int n_taps;       // 1 for Linear, 7 for conv k7, 2 for transposed conv phases
  int tap_base;     // position offset of tap 0 (e.g. -3*dilation, or -padding)
  int tap_step;     // position offset increment per tap (dilation; -1 for transposed conv)
  int b_tap_rows;   // rows of B per tap (= N as stored)
  int stride;       // >1: strided conv; tap position u = l*stride + tap_base + tap*tap_step is
                    // addressed as (phase = u mod stride, row = u div stride) of the 4-D map
  int b_static = 0; // 1: B holds long-lived weights that no kernel still running can be writing, so its first
                    // tiles may be fetched before the programmatic-dependency wait
  int n_parts = 1;  // 3: split-operand products for ~fp32 accuracy from 16-bit tensor-core operands: every tap is
                    // issued three times into the same accumulator, (A_hi, W_hi), (A_lo, W_hi), (A_hi, W_lo), where
                    // x_lo = 16-bit(x - x_hi); A_lo comes through the second tensor map, W_lo sits b_part_rows below W_hi
  int b_part_rows = 0;
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // 64 x 16-bit = 128 B = one swizzle atom row
constexpr int kWgmmaK = 16;
constexpr int kGemmThreads = 384;   // producer warpgroup + 2 MMA / epilogue warpgroups
constexpr int kSmemBudget = 227 * 1024;   // the most shared memory a block may use on sm_90

constexpr int kEpiWarps = 8;
template <int BN, int kCols, int kEpiStage = 0>   // kEpiStage: bytes of epilogue staging smem per epilogue warp
struct GemmCfg {
  static constexpr int kStageA = kBlockM * kBlockK * 2;
  static constexpr int kStageB = BN * kBlockK * 2;
  static constexpr int kStage = kStageA + kStageB;
  static constexpr int kAccLd = kCols + 4;              // fp32 row pitch of the accumulator staging tile
  static constexpr int kAccStage = 2 * 64 * kAccLd * 4;  // per MMA warpgroup: two column chunks of its 64 rows
  static constexpr int kFixed = 1024 /*align slack*/ + 256 /*barriers*/ + 2 * kAccStage + kEpiWarps * kEpiStage;
  static constexpr int kStages = (kSmemBudget - kFixed) / kStage > 8 ? 8 : (kSmemBudget - kFixed) / kStage;
  static constexpr int kSmemBytes = kStages * kStage + kFixed;
  static_assert(BN == 64 || BN == 128 || BN == 256, "BN must be 64/128/256");
  static_assert(kStages >= 2, "shared memory too small for a two-stage ring");
};

struct EpiCtx {
  int row;       // flattened output row = batch * L + l
  int l;         // row within batch
  int batch;
  int col0;      // first output column of this register chunk
  bool valid;    // row < L
  int l0;        // first row (within the batch item) of this warp's 32 rows
  int L;         // rows per batch item
  int lane;
  float* stage;  // per-warp staging smem (Epi::kStageBytes), or nullptr
  int n_tile;    // index of the tile along N
  int half;      // which of the two epilogue warps of the lane quadrant (they take alternate column chunks)
};

// Epilogues may carry per-thread state across the column chunks of one tile (e.g. the row sums that feed the next
// LayerNorm): such an epilogue declares `State`, `tile_begin`, `apply(p, c, r, state)` and `tile_end`; all others keep
// the plain `apply(p, c, r)`.
template <class E, class = void>
struct EpiHasState : std::false_type {};
template <class E>
struct EpiHasState<E, std::void_t<typename E::State>> : std::true_type {};
struct EpiNoStateHolder {
  struct State {};
};
template <class Epi>
struct EpiTile {
  using State = typename std::conditional<EpiHasState<Epi>::value, Epi, EpiNoStateHolder>::type::State;
  template <int N>
  __device__ static __forceinline__ void apply(const typename Epi::Params& p, const EpiCtx& c, const uint32_t (&r)[N], State& st) {
    if constexpr (EpiHasState<Epi>::value) Epi::apply(p, c, r, st);
    else Epi::apply(p, c, r);
  }
  __device__ static __forceinline__ void begin(const typename Epi::Params& p, const EpiCtx& c, State& st) {
    if constexpr (EpiHasState<Epi>::value) Epi::tile_begin(p, c, st);
  }
  __device__ static __forceinline__ void end(const typename Epi::Params& p, const EpiCtx& c, State& st) {
    if constexpr (EpiHasState<Epi>::value) Epi::tile_end(p, c, st);
  }
};

// Epilogue of one 128 x BN tile, run by MMA warpgroup cw (rows [64 cw, 64 cw + 64)) on its accumulator fragment.
// The accumulator goes through shared memory (acc_st: 2 x 64 x (kCols + 4) fp32 per warpgroup) two column chunks at a
// time, so that every epilogue thread receives kCols consecutive columns of ONE row (thread = row, as the epilogues
// expect).  epi_st: the epilogue's own per-warp staging (Epi::kStageBytes), or null.
template <class Epi, int BN>
__device__ __forceinline__ void gemm_tile_epilogue(const float (&acc)[BN / 2], float* acc_st, float* epi_st,
                                                   const typename Epi::Params& ep, int L, int N, int m0, int n0, int nt,
                                                   int batch, int cw, int warp, int lane) {
  const int wq = warp & 3;           // warp within the warpgroup
  const int half = wq >> 1;          // warps 0, 1 take the even column chunks, warps 2, 3 the odd ones
  const int rsub = (wq & 1) * 32;    // rows [rsub, rsub + 32) of the warpgroup's 64
  const int fr = 16 * wq + (lane >> 2);   // accumulator fragment rows fr, fr + 8
  const int fc = 2 * (lane & 3);          // and columns 8 j + fc, + 1
  constexpr int kChunks = BN / Epi::kCols;
  constexpr int kLd = Epi::kCols + 4;
  EpiCtx c;
  c.l0 = m0 + 64 * cw + rsub;
  c.l = c.l0 + lane;
  c.batch = batch;
  c.row = batch * L + c.l;
  c.valid = c.l < L;
  c.L = L;
  c.lane = lane;
  c.n_tile = nt;
  c.half = half;
  c.stage = epi_st;
  int n_valid = (N - n0 + Epi::kCols - 1) / Epi::kCols;   // chunks that hold real columns (warp-uniform)
  if (n_valid > kChunks) n_valid = kChunks;
  typename EpiTile<Epi>::State est;
  EpiTile<Epi>::begin(ep, c, est);
#pragma unroll
  for (int cp = 0; cp < (kChunks + 1) / 2; ++cp) {
    named_bar_sync(1 + cw, 128);   // the previous chunk pair has been read out
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int ch = 2 * cp + hh;
      if (ch < kChunks) {
        float* dst = acc_st + hh * 64 * kLd;
#pragma unroll
        for (int j = 0; j < Epi::kCols / 8; ++j) {
          const int ai = (ch * (Epi::kCols / 8) + j) * 4;
          *reinterpret_cast<float2*>(dst + fr * kLd + 8 * j + fc) = make_float2(acc[ai], acc[ai + 1]);
          *reinterpret_cast<float2*>(dst + (fr + 8) * kLd + 8 * j + fc) = make_float2(acc[ai + 2], acc[ai + 3]);
        }
      }
    }
    named_bar_sync(1 + cw, 128);
    const int ci = 2 * cp + half;
    if (ci < n_valid) {
      uint32_t r[Epi::kCols];
      const float4* src = reinterpret_cast<const float4*>(acc_st + half * 64 * kLd + (rsub + lane) * kLd);
#pragma unroll
      for (int j = 0; j < Epi::kCols / 4; ++j) {
        const float4 v = src[j];
        r[4 * j] = __float_as_uint(v.x);
        r[4 * j + 1] = __float_as_uint(v.y);
        r[4 * j + 2] = __float_as_uint(v.z);
        r[4 * j + 3] = __float_as_uint(v.w);
      }
      c.col0 = n0 + ci * Epi::kCols;
      EpiTile<Epi>::apply(ep, c, r, est);
    }
  }
  EpiTile<Epi>::end(ep, c, est);
}
template <class Epi, int BN, bool BF16>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmA2, const GemmShape s, const typename Epi::Params ep) {
  using Cfg = GemmCfg<BN, Epi::kCols, Epi::kStageBytes>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStage);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;
  uint8_t* epi_smem = smem + Cfg::kStages * Cfg::kStage + 256;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  const int m_tiles = (s.L + kBlockM - 1) / kBlockM;
  const int n_tiles = (s.N + BN - 1) / BN;
  const int tiles_per_n = m_tiles * s.batches;
  const int total_tiles = tiles_per_n * n_tiles;
  const int kb_per_tap = (s.K + kBlockK - 1) / kBlockK;
  const int kb_per_part = kb_per_tap * s.n_taps;
  const int num_kb = kb_per_part * s.n_parts;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrival per MMA warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();   // the next kernel may be scheduled as SMs drain
  // Everything above overlapped the previous kernel's tail.  The B operand (weights) never depends on the
  // previous kernel, so the producer thread also starts the B loads of its first stages before it waits for
  // the dependency; the MMA warpgroups wait right away.

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ------------------------------------------------------------ TMA producer
      int pre = 0;
      if (s.b_static && static_cast<int>(blockIdx.x) < total_tiles) {
        pre = num_kb < Cfg::kStages ? num_kb : Cfg::kStages;
        const int n0 = (static_cast<int>(blockIdx.x) / tiles_per_n) * BN;
        for (int kb = 0; kb < pre; ++kb) {
          const int pidx = kb / kb_per_part, kbp = kb - pidx * kb_per_part;
          const int part = split_part(pidx, s.n_parts);
          const int tap = kbp / kb_per_tap;
          const int k0 = (kbp - tap * kb_per_tap) * kBlockK;
          mbar_expect_tx(&full_bar[kb], Cfg::kStage);
          tma_load_2d(smem + kb * Cfg::kStage + Cfg::kStageA, &tmB, &full_bar[kb], k0,
                      tap * s.b_tap_rows + n0 + (part == 2 ? s.b_part_rows : 0));
        }
      }
      pdl_wait();
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = tile / tiles_per_n;
        const int rem = tile - nt * tiles_per_n;
        const int batch = rem / m_tiles;
        const int m0 = (rem - batch * m_tiles) * kBlockM;
        const int n0 = nt * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          const int pidx = kb / kb_per_part, kbp = kb - pidx * kb_per_part;
          const int part = split_part(pidx, s.n_parts);
          const int tap = kbp / kb_per_tap;
          const int k0 = (kbp - tap * kb_per_tap) * kBlockK;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStage;
          uint8_t* sb = sa + Cfg::kStageA;
          const bool b_done = tile == static_cast<int>(blockIdx.x) && kb < pre;   // issued before the wait
          if (!b_done) mbar_expect_tx(&full_bar[stage], Cfg::kStage);
          const int u = s.tap_base + tap * s.tap_step;
          int ph = 0, ro = u;
          if (s.stride > 1) {
            ro = (u >= 0) ? u / s.stride : -((-u + s.stride - 1) / s.stride);   // floor division
            ph = u - ro * s.stride;
          }
          tma_load_4d(sa, part == 1 ? &tmA2 : &tmA, &full_bar[stage], k0, ph, m0 + ro, batch);
          if (!b_done)
            tma_load_2d(sb, &tmB, &full_bar[stage], k0, tap * s.b_tap_rows + n0 + (part == 2 ? s.b_part_rows : 0));
          if (++stage == Cfg::kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    pdl_wait();
    // ------------------------------------------------------------ MMA + epilogue warpgroups
    const int cw = wg - 1;             // rows [64 cw, 64 cw + 64) of the tile
    float* acc_st = reinterpret_cast<float*>(epi_smem + cw * Cfg::kAccStage);
    float* epi_st = Epi::kStageBytes > 0
                        ? reinterpret_cast<float*>(epi_smem + 2 * Cfg::kAccStage + (warp - 4) * Epi::kStageBytes)
                        : nullptr;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int nt = tile / tiles_per_n;
      const int rem = tile - nt * tiles_per_n;
      const int batch = rem / m_tiles;
      const int m0 = (rem - batch * m_tiles) * kBlockM;
      const int n0 = nt * BN;
      // mainloop: one wgmma group per k-block; the smem slot of k-block kb - 1 is released once group kb is issued
      // and group kb - 1 has retired
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * Cfg::kStage) + cw * 64 * kBlockK * 2;
        const uint32_t b_addr = smem_u32(smem + stage * Cfg::kStage) + Cfg::kStageA;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k)
          wgmma_ss<BN, BF16>(acc, make_desc_kmajor_sw128(a_addr + k * kWgmmaK * 2),
                             make_desc_kmajor_sw128(b_addr + k * kWgmmaK * 2), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>(acc);
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>(acc);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);

      gemm_tile_epilogue<Epi, BN>(acc, acc_st, epi_st, ep, s.L, s.N, m0, n0, nt, batch, cw, warp, lane);
    }
  }
}

// ------------------------------------------------------------------ epilogues
// Every epilogue receives kCols consecutive fp32 accumulator columns of one row
// (as raw bits in r[]) and writes them straight to global memory.

// ---- LayerNorm folded into the consumer GEMM (prepend-mode DiT blocks) --------------------------------------------
// The producer of the residual stream (EpiResidualLN below) stores x16 = 16-bit(h * gamma) next to h and accumulates the
// row sums s1 = sum h, s2 = sum h^2.  With c[n] = sum_k gamma_k W[n,k] and d[n] = sum_k beta_k W[n,k] (prepared once),
//   LayerNorm(h) W^T = rstd (h gamma) W^T - rstd mean c + d,   mean = s1 / D, rstd = rsqrt(s2 / D - mean^2 + eps)
// (models/transformer.py:188-206 followed by the Linear), so the consumer GEMM reads x16 and its epilogue applies one
// multiply-add per element: no LayerNorm pass over the residual stream, no extra kernel.
constexpr int kLnSlots = 12;   // partial sums per row: 6 column tiles of 256 x 2 epilogue warps (D = 1536); fixed
                               // slots summed in a fixed order keep the result bit-reproducible (no atomics)
struct LnFold {
  const float2* stats;   // [rows][n_slots] partial (s1, s2) of the residual row, or null: no LayerNorm in front
  const float* c;        // [N]
  const float* d;        // [N] or null (beta = 0)
  float inv_dim;         // 1 / D
  float eps;
  int n_slots;
};
struct LnRow {
  float rstd, mr;        // rstd, mean * rstd
};
__device__ __forceinline__ LnRow ln_row(const LnFold& f, int row) {
  const float4* sp = reinterpret_cast<const float4*>(f.stats + static_cast<size_t>(row) * kLnSlots);
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < kLnSlots / 2; ++i) {
    if (2 * i < f.n_slots) {
      const float4 v = __ldg(sp + i);
      s1 += v.x + v.z;
      s2 += v.y + v.w;
    }
  }
  const float mean = s1 * f.inv_dim;
  const float var = fmaxf(s2 * f.inv_dim - mean * mean, 0.f);
  LnRow r;
  r.rstd = rsqrtf(var + f.eps);
  r.mr = mean * r.rstd;
  return r;
}
// v[0..3] <- rstd * v - (mean rstd) * c[col..col+3] (+ d[col..col+3]); col % 4 == 0 (128-bit loads of c / d)
__device__ __forceinline__ void ln_apply4(const LnFold& f, const LnRow& r, float& v0, float& v1, float& v2, float& v3, int col) {
  const float4 cc = __ldg(reinterpret_cast<const float4*>(f.c + col));
  v0 = fmaf(v0, r.rstd, -r.mr * cc.x);
  v1 = fmaf(v1, r.rstd, -r.mr * cc.y);
  v2 = fmaf(v2, r.rstd, -r.mr * cc.z);
  v3 = fmaf(v3, r.rstd, -r.mr * cc.w);
  if (f.d) {
    const float4 dd = __ldg(reinterpret_cast<const float4*>(f.d + col));
    v0 += dd.x; v1 += dd.y; v2 += dd.z; v3 += dd.w;
  }
}

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

// out16[row, col] = act(acc + bias)   (act: 0 none, 1 SiLU)
template <bool BF16, bool LN = false>   // LN: a LayerNorm is folded into this GEMM (LnFold); separate instantiation so that
struct EpiStore16 {                      // the plain epilogue carries none of its code or registers
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  struct Params {
    void* out;
    int ld;
    const float* bias;  // may be null
    int act;
    LnFold ln = LnFold{nullptr, nullptr, nullptr, 0.f, 0.f, 0};
  };
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[32]) {
    if (!c.valid) return;
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
    if constexpr (LN) {
      const LnRow lr = ln_row(p.ln, c.row);
#pragma unroll
      for (int j = 0; j < 32; j += 4) ln_apply4(p.ln, lr, v[j], v[j + 1], v[j + 2], v[j + 3], c.col0 + j);
    }
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + c.col0 + j));
        v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
      }
    }
    uint32_t o[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float a = v[2 * j], b = v[2 * j + 1];
      if (p.act == 1) {
        a = silu_f(a);
        b = silu_f(b);
      }
      o[j] = Op16<BF16>::pack(a, b);
    }
    uint4* dst = reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + static_cast<size_t>(c.row) * p.ld + c.col0);
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
  }
};

// out32[row, col] = acc (+ bias)
struct EpiStore32 {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  struct Params {
    float* out;
    int ld;
    const float* bias;
  };
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[32]) {
    if (!c.valid) return;
    float4* dst = reinterpret_cast<float4*>(p.out + static_cast<size_t>(c.row) * p.ld + c.col0);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float4 v = make_float4(__uint_as_float(r[4 * j]), __uint_as_float(r[4 * j + 1]), __uint_as_float(r[4 * j + 2]),
                             __uint_as_float(r[4 * j + 3]));
      if (p.bias) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + c.col0) + j);
        v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
      }
      dst[j] = v;
    }
  }
};

// Residual stream update (models/transformer.py:692-700 and adaLN :670-689):
//   h[row, col] += (acc + bias[col]) * gate[row / rows_per_item, col]
struct EpiResidual {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  struct Params {
    float* h;
    int ld;
    const float* bias;  // may be null
    const float* gate;  // may be null; sigmoid(1 - gate) precomputed, row stride gate_ld
    int rows_per_item;
    int gate_ld;
    int n_items;        // item = (row / rows_per_item) % n_items (CFG halves share the conditioning)
  };
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[32]) {
    if (!c.valid) return;
    float4* dst = reinterpret_cast<float4*>(p.h + static_cast<size_t>(c.row) * p.ld + c.col0);
    const float4* g = p.gate ? reinterpret_cast<const float4*>(
                                   p.gate + static_cast<size_t>((c.row / p.rows_per_item) % p.n_items) * p.gate_ld + c.col0)
                             : nullptr;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float4 v = make_float4(__uint_as_float(r[4 * j]), __uint_as_float(r[4 * j + 1]), __uint_as_float(r[4 * j + 2]),
                             __uint_as_float(r[4 * j + 3]));
      if (p.bias) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + c.col0) + j);
        v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
      }
      if (g) {
        const float4 gg = __ldg(g + j);
        v.x *= gg.x; v.y *= gg.y; v.z *= gg.z; v.w *= gg.w;
      }
      // fire-and-forget fp32 vector reduction in L2: every element receives exactly one add
      // per GEMM (no split-K), so the result is deterministic and no load stalls the epilogue
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + j), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                   : "memory");
    }
  }
};

// Residual stream update that also prepares the NEXT LayerNorm (see LnFold): h = h + acc + bias is written back in
// fp32 (plain load / store: every element belongs to exactly one lane of one tile), x16 = 16-bit(h * gamma) is what
// the next GEMM reads, and the partial row sums of this tile go to a fixed slot of stats.  Rows below `split` are
// followed by one LayerNorm (gamma_lo, stats_lo: the cross-attention norm of the conditional rows), the others by
// another (gamma_hi, stats_hi: the feed-forward norm of rows without cross-attention).
template <bool BF16>
struct EpiResidualLN {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 32 * 36 * 4;   // per-warp [32 rows][32 + 4 pad] fp32 transpose tile
  struct Params {
    float* h;
    int ld;
    const float* bias;       // may be null
    void* x16;               // [rows, ld] 16-bit
    const float* gamma_lo;   // may be null (= 1)
    const float* gamma_hi;
    float2* stats_lo;        // may be null (no LayerNorm follows: last block)
    float2* stats_hi;
    int split;               // rows < split: *_lo, else *_hi
  };
  // Warp-cooperative like EpiConv: the accumulator chunk (thread = row, 32 columns) goes through the per-warp smem
  // tile so that every global access is a coalesced 128 B row segment (8 lanes x 16 B, 4 rows per instruction); the
  // old h values are requested BEFORE the transpose so the loads are in flight meanwhile.  Lane = (row offset
  // lane / 8 within groups of 4 rows, 4-column group lane % 8): it owns rows l0 + lane / 8 + 4 i, i < 8.
  struct State {
    float s1[8], s2[8];
  };
  __device__ static __forceinline__ void tile_begin(const Params&, const EpiCtx&, State& st) {
#pragma unroll
    for (int i = 0; i < 8; ++i) st.s1[i] = st.s2[i] = 0.f;
  }
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[32], State& st) {
    const int g = c.lane & 7, r0 = c.lane >> 3;
    const int col = c.col0 + 4 * g;
    float4 old[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int l = c.l0 + r0 + 4 * i;
      old[i] = l < c.L ? *reinterpret_cast<const float4*>(p.h + (static_cast<size_t>(c.batch) * c.L + l) * p.ld + col)
                       : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float* stg = c.stage;
    {
      float4* mine = reinterpret_cast<float4*>(stg + c.lane * 36);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        mine[j] = make_float4(__uint_as_float(r[4 * j]), __uint_as_float(r[4 * j + 1]), __uint_as_float(r[4 * j + 2]),
                              __uint_as_float(r[4 * j + 3]));
    }
    __syncwarp();
    float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f), glo = make_float4(1.f, 1.f, 1.f, 1.f), ghi = glo;
    if (p.bias) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
    if (p.gamma_lo) glo = __ldg(reinterpret_cast<const float4*>(p.gamma_lo + col));
    if (p.gamma_hi) ghi = __ldg(reinterpret_cast<const float4*>(p.gamma_hi + col));
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int l = c.l0 + r0 + 4 * i;
      if (l < c.L) {
        const size_t row = static_cast<size_t>(c.batch) * c.L + l;
        const float4 a = *reinterpret_cast<const float4*>(stg + (r0 + 4 * i) * 36 + 4 * g);
        float4 v;
        v.x = a.x + b4.x + old[i].x; v.y = a.y + b4.y + old[i].y; v.z = a.z + b4.z + old[i].z; v.w = a.w + b4.w + old[i].w;
        *reinterpret_cast<float4*>(p.h + row * p.ld + col) = v;
        st.s1[i] += (v.x + v.y) + (v.z + v.w);
        st.s2[i] = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, st.s2[i]))));
        const float4 gg = static_cast<int>(row) < p.split ? glo : ghi;
        *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.x16) + row * p.ld + col) =
            make_uint2(Op16<BF16>::pack(v.x * gg.x, v.y * gg.y), Op16<BF16>::pack(v.z * gg.z, v.w * gg.w));
      }
    }
    __syncwarp();
  }
  __device__ static __forceinline__ void tile_end(const Params& p, const EpiCtx& c, State& st) {
    const int g = c.lane & 7, r0 = c.lane >> 3;
    const int slot = c.n_tile * 2 + c.half;      // one writer per (row, slot): plain store, summed by ln_row in order
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a = st.s1[i], b = st.s2[i];
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {            // the 8 lanes of a row segment (same lane / 8)
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      const int l = c.l0 + r0 + 4 * i;
      if (g == 0 && l < c.L && slot < kLnSlots) {
        const size_t row = static_cast<size_t>(c.batch) * c.L + l;
        float2* sp = static_cast<int>(row) < p.split ? p.stats_lo : p.stats_hi;
        if (sp) sp[row * kLnSlots + slot] = make_float2(a, b);
      }
    }
  }
};

// Fused QKV projection epilogue: split is implicit (q | k | v are column ranges of
// one [M, 3D] buffer); partial rotary of every q and k head (models/transformer.py:158-183,
// 438-452), position = token index within the sequence (prepend token = position 0).  fp32
// math, then cast.  A head of width head_dim has nf = max(head_dim / 2, 32) / 2 rotary pairs
// (j, j + nf).  The q / k rows of to_qkv are permuted inside each head at load time (dit.cu,
// qkv_head_perm) so that the pairs sit at positions (i, i + 16) of the head's 32-column chunks:
// chunk ci = (col % head_dim) / 32 rotates its first clamp(nf - 16 ci, 0, 16) pairs with the
// table columns 16 ci + i, and the rest of the head passes through.  q and k share the
// permutation, so every q . k is unchanged.  Head dim 64: identity; chunk 0 rotates 16 pairs.
template <bool BF16, bool LN = false>
struct EpiQkvRope {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  struct Params {
    void* out;
    int ld;            // 3*D
    int rope_cols;     // 2*D : columns >= this (v) are never rotated
    int seq_len;       // tokens per item (position = row % seq_len)
    int head_dim;      // 32, 64, 96 or 128
    int nf;            // rotary frequencies per head (table row stride): 16, 16, 24, 32
    const float* cos_tab;  // [seq_len, nf]
    const float* sin_tab;  // [seq_len, nf]
    LnFold ln = LnFold{nullptr, nullptr, nullptr, 0.f, 0.f, 0};
  };
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[32]) {
    if (!c.valid) return;
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
    if constexpr (LN) {
      const LnRow lr = ln_row(p.ln, c.row);
#pragma unroll
      for (int j = 0; j < 32; j += 4) ln_apply4(p.ln, lr, v[j], v[j + 1], v[j + 2], v[j + 3], c.col0 + j);
    }
    // chunk of 32 columns aligned to 32 (head_dim is a multiple of 32): its rotary pairs (i, i + 16), i < n_rot
    const int ci = (c.col0 % p.head_dim) >> 5;
    const int n_rot = min(max(p.nf - 16 * ci, 0), 16);   // 16 or 8 (head dim 96, chunk 1) or 0
    if (c.col0 < p.rope_cols && n_rot > 0 && p.cos_tab) {
      const int pos = c.row % p.seq_len;
      const float4* ct = reinterpret_cast<const float4*>(p.cos_tab + pos * p.nf + 16 * ci);
      const float4* st = reinterpret_cast<const float4*>(p.sin_tab + pos * p.nf + 16 * ci);
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        if (4 * j4 >= n_rot) break;
        const float4 cs = __ldg(ct + j4), sn = __ldg(st + j4);
        const float cc[4] = {cs.x, cs.y, cs.z, cs.w}, ss[4] = {sn.x, sn.y, sn.z, sn.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = j4 * 4 + u;
          const float a = v[j], b = v[j + 16];
          v[j] = a * cc[u] - b * ss[u];       // t*cos + rotate_half(t)*sin, rotate_half = [-b, a]
          v[j + 16] = b * cc[u] + a * ss[u];
        }
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + static_cast<size_t>(c.row) * p.ld + c.col0);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      dst[j] = make_uint4(Op16<BF16>::pack(v[8 * j], v[8 * j + 1]), Op16<BF16>::pack(v[8 * j + 2], v[8 * j + 3]),
                          Op16<BF16>::pack(v[8 * j + 4], v[8 * j + 5]), Op16<BF16>::pack(v[8 * j + 6], v[8 * j + 7]));
  }
};

// 16-bit store of whole 64-wide heads with the optional cosine-similarity normalisation of q / k
// (attn_kwargs.qk_norm, models/transformer.py:433-436: F.normalize(., dim=-1), eps 1e-12) for columns
// below norm_cols, followed by the partial rotary of EpiQkvRope for columns below rope_cols.  Used for the
// fused QKV projection, the cross-attention q projection and the (step-invariant) k | v projection when
// the model is built with qk_norm; the thread owns one head (64 accumulator columns) of one row.
template <bool BF16>
struct EpiHeadNorm16 {
  static constexpr int kCols = 64;
  static constexpr int kStageBytes = 0;
  struct Params {
    void* out;
    int ld;
    int norm_cols;         // columns >= this are stored as they are (v)
    int rope_cols;         // 0: no rotary
    int seq_len;
    const float* cos_tab;  // [seq_len, 16]
    const float* sin_tab;
  };
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[64]) {
    if (!c.valid) return;
    float inv = 1.f;
    if (c.col0 < p.norm_cols) {
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < 64; ++j) ss = fmaf(__uint_as_float(r[j]), __uint_as_float(r[j]), ss);
      inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
    }
    uint4* dst = reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + static_cast<size_t>(c.row) * p.ld + c.col0);
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]) * inv;
    if (c.col0 < p.rope_cols && p.cos_tab) {
      const int pos = c.row % p.seq_len;
      const float4* ct = reinterpret_cast<const float4*>(p.cos_tab + pos * 16);
      const float4* st = reinterpret_cast<const float4*>(p.sin_tab + pos * 16);
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        const float4 cs = __ldg(ct + j4), sn = __ldg(st + j4);
        const float cc[4] = {cs.x, cs.y, cs.z, cs.w}, ss4[4] = {sn.x, sn.y, sn.z, sn.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = j4 * 4 + u;
          const float a = v[j], b = v[j + 16];
          v[j] = a * cc[u] - b * ss4[u];
          v[j + 16] = b * cc[u] + a * ss4[u];
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      dst[j] = make_uint4(Op16<BF16>::pack(v[8 * j], v[8 * j + 1]), Op16<BF16>::pack(v[8 * j + 2], v[8 * j + 3]),
                          Op16<BF16>::pack(v[8 * j + 4], v[8 * j + 5]), Op16<BF16>::pack(v[8 * j + 6], v[8 * j + 7]));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t* q = &r[32 + 8 * j];
      dst[4 + j] = make_uint4(Op16<BF16>::pack(__uint_as_float(q[0]) * inv, __uint_as_float(q[1]) * inv),
                              Op16<BF16>::pack(__uint_as_float(q[2]) * inv, __uint_as_float(q[3]) * inv),
                              Op16<BF16>::pack(__uint_as_float(q[4]) * inv, __uint_as_float(q[5]) * inv),
                              Op16<BF16>::pack(__uint_as_float(q[6]) * inv, __uint_as_float(q[7]) * inv));
    }
  }
};

// SwiGLU epilogue (models/transformer.py:232-235: value = first half, gate = second
// half of the projection).  The weight rows are interleaved at load time so every
// 64-column group holds 32 value columns followed by their 32 gate columns:
//   out[row, g*32 + j] = (acc[g*64 + j] + b) * silu(acc[g*64 + 32 + j] + b')
template <bool BF16, bool LN = false>
struct EpiSwiglu {
  static constexpr int kCols = 64;
  static constexpr int kStageBytes = 0;
  struct Params {
    void* out;
    int ld;             // inner dim (N/2)
    const float* bias;  // interleaved like the weight rows; may be null
    LnFold ln = LnFold{nullptr, nullptr, nullptr, 0.f, 0.f, 0};
  };
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[64]) {
    if (!c.valid) return;
    // four value columns and their four gate columns at a time, straight from the accumulator registers (a 64-float
    // working copy next to the two 64-register chunk buffers of the epilogue loop spills)
    uint32_t o[16];
    if constexpr (!LN) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float a0 = __uint_as_float(r[2 * j]), a1 = __uint_as_float(r[2 * j + 1]);
        float g0 = __uint_as_float(r[32 + 2 * j]), g1 = __uint_as_float(r[33 + 2 * j]);
        if (p.bias) {
          a0 += __ldg(p.bias + c.col0 + 2 * j);
          a1 += __ldg(p.bias + c.col0 + 2 * j + 1);
          g0 += __ldg(p.bias + c.col0 + 32 + 2 * j);
          g1 += __ldg(p.bias + c.col0 + 33 + 2 * j);
        }
        o[j] = Op16<BF16>::pack(a0 * silu_f(g0), a1 * silu_f(g1));
      }
      uint4* dst0 =
          reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + static_cast<size_t>(c.row) * p.ld + (c.col0 >> 1));
#pragma unroll
      for (int j = 0; j < 4; ++j) dst0[j] = make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
      return;
    }
    LnRow lr{1.f, 0.f};
    if constexpr (LN) lr = ln_row(p.ln, c.row);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a0 = __uint_as_float(r[4 * j]), a1 = __uint_as_float(r[4 * j + 1]), a2 = __uint_as_float(r[4 * j + 2]),
            a3 = __uint_as_float(r[4 * j + 3]);
      float g0 = __uint_as_float(r[32 + 4 * j]), g1 = __uint_as_float(r[33 + 4 * j]), g2 = __uint_as_float(r[34 + 4 * j]),
            g3 = __uint_as_float(r[35 + 4 * j]);
      if constexpr (LN) {
        ln_apply4(p.ln, lr, a0, a1, a2, a3, c.col0 + 4 * j);
        ln_apply4(p.ln, lr, g0, g1, g2, g3, c.col0 + 32 + 4 * j);
      }
      if (p.bias) {
        const float4 ba = __ldg(reinterpret_cast<const float4*>(p.bias + c.col0 + 4 * j));
        const float4 bg = __ldg(reinterpret_cast<const float4*>(p.bias + c.col0 + 32 + 4 * j));
        a0 += ba.x; a1 += ba.y; a2 += ba.z; a3 += ba.w;
        g0 += bg.x; g1 += bg.y; g2 += bg.z; g3 += bg.w;
      }
      o[2 * j] = Op16<BF16>::pack(a0 * silu_f(g0), a1 * silu_f(g1));
      o[2 * j + 1] = Op16<BF16>::pack(a2 * silu_f(g2), a3 * silu_f(g3));
    }
    uint4* dst =
        reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + static_cast<size_t>(c.row) * p.ld + (c.col0 >> 1));
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
  }
};

// ------------------------------------------------------- convolution epilogues
// SnakeBeta (models/blocks.py:318-319) with precomputed a = e^alpha, ib = 1/(e^beta + 1e-9):
// v + ib * sin^2(a v) with the SFU sine (sin.approx = multiply by 1/2pi + MUFU.SIN, which is periodic
// in its argument).  Its absolute error is 2^-21.4 + ~|a v| * 2^-23 -- the second term is the rounding
// of the argument itself -- i.e. < 2e-5 for |a v| < 100, far below the 16-bit rounding (2^-11 relative)
// applied to the result right after.  Five instructions per element instead of ten for an explicit
// Cody-Waite reduction, and one SFU operation instead of two.
__device__ __forceinline__ float snake_fast(float v, float a, float ib) {
  const float sn = __sinf(v * a);
  return fmaf(ib, sn * sn, v);
}

// fp32 pairs in one 64-bit register (two lanes of a 4-element segment) for the convolution epilogues.
__device__ __forceinline__ uint64_t f2_pack(float lo, float hi) {
  uint64_t d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(lo), "f"(hi));
  return d;
}
__device__ __forceinline__ void f2_unpack(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t f2_add(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  return f2_pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f2_mul(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  return f2_pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  f2_unpack(c, c0, c1);
  return f2_pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
// snake_fast on two values at once: same operations and roundings as the scalar version.
__device__ __forceinline__ uint64_t snake_fast2(uint64_t v, uint64_t a, uint64_t ib) {
  float t0, t1;
  f2_unpack(f2_mul(v, a), t0, t1);
  const uint64_t sn = f2_pack(__sinf(t0), __sinf(t1));
  return f2_fma(ib, f2_mul(sn, sn), v);
}

// Epilogue of every tensor-core convolution of the Oobleck VAE (models/autoencoders.py:45-116):
//   y = acc + bias[co] (+ resid[pos, co])            ResidualUnit skip :66-68
//   raw_out[pos, co] = y (fp32, optional)            kept only where a later skip needs it
//   s16_out[pos, co] = 16-bit( snake_next(y) )       the NEXT layer's activation, fused here
// Transposed convolutions (:102-105) run as a 2-tap GEMM over N = up*cout columns
// (column = phase*cout + co): output position = l*up + phase - pad.
struct EpiConvParams {
  const float* bias;    // [cout] or null
  const void* resid;    // raw skip stream [B*L_out, cout] (fp32, or 16-bit when raw16) or null
  void* raw_out;        // raw stream out, same type, or null
  void* s16_out;        // 16-bit [B*L_out, cout] or null
  const float* sn_a;    // [cout] e^alpha of the consumer's Snake, or null (plain cast)
  const float* sn_ib;   // [cout] 1/(e^beta + 1e-9)
  int cout;
  int L_out;            // output positions per batch item
  int up;               // transposed-conv stride (1 = ordinary conv)
  int pad;              // transposed-conv padding
  void* s16_lo_out;     // split-operand mode: 16-bit(y' - 16-bit(y')) next to s16_out (y' = the Snake-activated value), or null
  int raw16;            // 1: the raw (un-activated) stream is stored in the 16-bit operand type instead of fp32:
                        // 8 instead of 12 bytes per element and channel through a fused ResidualUnit (the sums
                        // are still formed in fp32; only the value carried to the next unit's skip is rounded)
};
// MASKED = true: the kernel carries ONLY the lean path (one index per chunk, per-segment validity as a bit mask, Snake and
// 16-bit raw streams unconditional) - for launches whose Params satisfy fast_flags(); the host picks the instantiation
// (oobleck.cu run_conv_gemm).  Compiled next to the general path in one kernel the lean path pays ~200 bytes of spills
// in the persistent GEMM kernels (long-scoreboard stalls on the reloads, profiles/r02_ncu_convT_s2.txt).
template <bool BF16, bool MASKED = false>
struct EpiConv {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 32 * 36 * 4;   // per-warp [32 rows][32 + 4 pad] fp32 transpose tile
  typedef EpiConvParams Params;
  // Snake-activated 16-bit output, raw streams (if any) in the 16-bit type, no lo copy: what the default fp16 decode runs
  __host__ __device__ static bool fast_flags(const Params& p) {
    return p.s16_out != nullptr && p.sn_a != nullptr && p.s16_lo_out == nullptr &&
           (p.raw16 != 0 || (p.resid == nullptr && p.raw_out == nullptr));
  }
  // Warp-cooperative: the accumulator chunk (thread = row, 32 columns) is transposed through the
  // per-warp smem tile so that every global access is coalesced (8 lanes x 16 B = one 128 B row
  // segment, 4 rows per instruction) and each lane needs the per-channel parameters of only 4 channels.
  // Column decomposition of a chunk, computed once: transposed convolutions put (phase, channel) on N.
  struct Seg {
    int phase, co;
  };
  __device__ static __forceinline__ Seg seg_of(const Params& p, const EpiCtx& c) {
    Seg sg{0, c.col0};
    if (p.up > 1) {
      sg.phase = c.col0 / p.cout;
      sg.co = c.col0 - sg.phase * p.cout;
    }
    sg.co += 4 * (c.lane & 7);
    return sg;
  }
  // Output address of row segment i (rows r0 + 4i of this warp's 32, channels co .. co+3);
  // false when the row / output position does not exist.
  __device__ static __forceinline__ bool seg_index(const Params& p, const EpiCtx& c, const Seg& sg, int i, size_t* idx) {
    const int l = c.l0 + (c.lane >> 3) + 4 * i;
    const int lo = l * p.up + sg.phase - p.pad;
    const bool ok = l < c.L && lo >= 0 && lo < p.L_out;
    *idx = (static_cast<size_t>(c.batch) * p.L_out + (ok ? lo : 0)) * p.cout + sg.co;
    return ok;
  }
  // ---- fast path.  The general code below costs ~120 instructions per 4-element segment, of which ~55 % are index
  // arithmetic, bounds tests and branches on the (launch-uniform) Params flags (ncu source page of the stride-2
  // transposed convolution, profiles/r02_ncu_convT_s2.txt: 30 instructions per element; the 128-channel layers are
  // bound by exactly this epilogue).  For a chunk whose 32 rows all exist - every chunk but the ragged ends of an item -
  // the 8 segments of a lane are idx0 + i * stride, so one index, one bounds test and one branch per chunk do;
  // the flags become template parameters.  Conditions: 16-bit raw streams (or none), a 16-bit output, no lo copy.
  struct Plan {
    size_t idx0;      // element index of segment 0
    int stride;       // elements between consecutive segments (4 rows)
    bool fast;        // warp-uniform
    int co;
  };
  __device__ static __forceinline__ Plan plan_of(const Params& p, const EpiCtx& c) {
    const Seg sg = seg_of(p, c);
    const int l_first = c.l0 + (c.lane >> 3), l_last = l_first + 28;
    const int lo_first = l_first * p.up + sg.phase - p.pad, lo_last = l_last * p.up + sg.phase - p.pad;
    const bool ok = l_last < c.L && lo_first >= 0 && lo_last < p.L_out;
    // (Moving the general path out of line instead - __noinline__ - made the decode 40-90 % SLOWER: the call sites
    // force the chunk registers through local memory.)
    const bool flags = fast_flags(p);
    Plan pl;
    pl.fast = flags && __all_sync(0xffffffffu, ok);
    pl.idx0 = (static_cast<size_t>(c.batch) * p.L_out + (ok ? lo_first : 0)) * p.cout + sg.co;
    pl.stride = 4 * p.up * p.cout;
    pl.co = sg.co;
    return pl;
  }
  template <bool RESID, bool RAWOUT, bool SNAKE>
  __device__ static __forceinline__ void finish_fast(const Params& p, const EpiCtx& c, const Plan& pl, const uint32_t (&r)[32],
                                                     const float4 (&rs)[8]) {
    const uint32_t st = smem_u32(c.stage);
    const int g = c.lane & 7, r0 = c.lane >> 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) sts128(st + (c.lane * 36 + 4 * j) * 4, r[4 * j], r[4 * j + 1], r[4 * j + 2], r[4 * j + 3]);
    __syncwarp();
    ulonglong2 b2 = make_ulonglong2(0ull, 0ull), a2 = b2, ib2 = b2;   // (x,y) and (z,w) pairs; 0 bits = 0.f
    if (p.bias) b2 = __ldg(reinterpret_cast<const ulonglong2*>(p.bias + pl.co));
    if (SNAKE) {
      a2 = __ldg(reinterpret_cast<const ulonglong2*>(p.sn_a + pl.co));
      ib2 = __ldg(reinterpret_cast<const ulonglong2*>(p.sn_ib + pl.co));
    }
    uint16_t* raw_o = static_cast<uint16_t*>(p.raw_out) + pl.idx0;
    uint16_t* s_o = static_cast<uint16_t*>(p.s16_out) + pl.idx0;
    uint32_t ld_addr = st + (r0 * 36 + 4 * g) * 4;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const ulonglong2 acc = lds128_b64x2(ld_addr);   // (reading all eight segments back first was not faster)
      ld_addr += 4 * 36 * 4;
      uint64_t v01 = f2_add(acc.x, b2.x), v23 = f2_add(acc.y, b2.y);
      if (RESID) {
        const float2 lo = Op16<BF16>::unpack(__float_as_uint(rs[i].x)), hi = Op16<BF16>::unpack(__float_as_uint(rs[i].y));
        v01 = f2_add(v01, f2_pack(lo.x, lo.y));
        v23 = f2_add(v23, f2_pack(hi.x, hi.y));
      }
      if (RAWOUT) {
        float y0, y1, y2, y3;
        f2_unpack(v01, y0, y1);
        f2_unpack(v23, y2, y3);
        *reinterpret_cast<uint2*>(raw_o) = make_uint2(Op16<BF16>::pack(y0, y1), Op16<BF16>::pack(y2, y3));
        raw_o += pl.stride;
      }
      if (SNAKE) {
        v01 = snake_fast2(v01, a2.x, ib2.x);
        v23 = snake_fast2(v23, a2.y, ib2.y);
      }
      float x0, x1, x2, x3;
      f2_unpack(v01, x0, x1);
      f2_unpack(v23, x2, x3);
      *reinterpret_cast<uint2*>(s_o) = make_uint2(Op16<BF16>::pack(x0, x1), Op16<BF16>::pack(x2, x3));
      s_o += pl.stride;
    }
    __syncwarp();
  }
  // ---- MASKED kernels: the same arithmetic for every chunk, ragged ones included (bit i of the mask = segment i exists)
  struct MPlan {
    long long idx0;   // element index of segment 0 (may point before the buffer when that segment does not exist)
    int stride;
    uint32_t mask;
    int co;
  };
  __device__ static __forceinline__ MPlan mplan_of(const Params& p, const EpiCtx& c) {
    const Seg sg = seg_of(p, c);
    const int l0 = c.l0 + (c.lane >> 3);
    const int lo0 = l0 * p.up + sg.phase - p.pad;
    MPlan pl;
    pl.mask = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int l = l0 + 4 * i, lo = lo0 + 4 * i * p.up;
      if (l < c.L && lo >= 0 && lo < p.L_out) pl.mask |= 1u << i;
    }
    pl.idx0 = (static_cast<long long>(c.batch) * p.L_out + lo0) * p.cout + sg.co;
    pl.stride = 4 * p.up * p.cout;
    pl.co = sg.co;
    return pl;
  }
  __device__ static __forceinline__ void prefetch_masked(const Params& p, const EpiCtx& c, float4 (&rs)[8]) {
    if (p.resid) {
      const MPlan pl = mplan_of(p, c);
      const uint16_t* rp = static_cast<const uint16_t*>(p.resid) + pl.idx0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        uint2 u = make_uint2(0u, 0u);
        if ((pl.mask >> i) & 1u) u = *reinterpret_cast<const uint2*>(rp);     // the loaded BITS (converted in finish)
        rp += pl.stride;
        rs[i] = make_float4(__uint_as_float(u.x), __uint_as_float(u.y), 0.f, 0.f);
      }
    }
  }
  template <bool RESID, bool RAWOUT>
  __device__ static __forceinline__ void finish_masked_t(const Params& p, const EpiCtx& c, const uint32_t (&r)[32],
                                                         const float4 (&rs)[8]) {
    const MPlan pl = mplan_of(p, c);
    const uint32_t st = smem_u32(c.stage);
    const int g = c.lane & 7, r0 = c.lane >> 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) sts128(st + (c.lane * 36 + 4 * j) * 4, r[4 * j], r[4 * j + 1], r[4 * j + 2], r[4 * j + 3]);
    __syncwarp();
    ulonglong2 b2 = make_ulonglong2(0ull, 0ull);
    if (p.bias) b2 = __ldg(reinterpret_cast<const ulonglong2*>(p.bias + pl.co));
    const ulonglong2 a2 = __ldg(reinterpret_cast<const ulonglong2*>(p.sn_a + pl.co));
    const ulonglong2 ib2 = __ldg(reinterpret_cast<const ulonglong2*>(p.sn_ib + pl.co));
    uint16_t* raw_o = static_cast<uint16_t*>(p.raw_out) + pl.idx0;
    uint16_t* s_o = static_cast<uint16_t*>(p.s16_out) + pl.idx0;
    uint32_t ld_addr = st + (r0 * 36 + 4 * g) * 4;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const ulonglong2 acc = lds128_b64x2(ld_addr);
      ld_addr += 4 * 36 * 4;
      const bool ok = (pl.mask >> i) & 1u;
      uint64_t v01 = f2_add(acc.x, b2.x), v23 = f2_add(acc.y, b2.y);
      if (RESID) {
        const float2 lo = Op16<BF16>::unpack(__float_as_uint(rs[i].x)), hi = Op16<BF16>::unpack(__float_as_uint(rs[i].y));
        v01 = f2_add(v01, f2_pack(lo.x, lo.y));
        v23 = f2_add(v23, f2_pack(hi.x, hi.y));
      }
      if (RAWOUT) {
        float y0, y1, y2, y3;
        f2_unpack(v01, y0, y1);
        f2_unpack(v23, y2, y3);
        if (ok) *reinterpret_cast<uint2*>(raw_o) = make_uint2(Op16<BF16>::pack(y0, y1), Op16<BF16>::pack(y2, y3));
        raw_o += pl.stride;
      }
      v01 = snake_fast2(v01, a2.x, ib2.x);
      v23 = snake_fast2(v23, a2.y, ib2.y);
      float x0, x1, x2, x3;
      f2_unpack(v01, x0, x1);
      f2_unpack(v23, x2, x3);
      if (ok) *reinterpret_cast<uint2*>(s_o) = make_uint2(Op16<BF16>::pack(x0, x1), Op16<BF16>::pack(x2, x3));
      s_o += pl.stride;
    }
    __syncwarp();
  }
  __device__ static __forceinline__ void finish_masked(const Params& p, const EpiCtx& c, const uint32_t (&r)[32],
                                                       const float4 (&rs)[8]) {
    if (p.resid) {
      if (p.raw_out) finish_masked_t<true, true>(p, c, r, rs);
      else finish_masked_t<true, false>(p, c, r, rs);
    } else {
      if (p.raw_out) finish_masked_t<false, true>(p, c, r, rs);
      else finish_masked_t<false, false>(p, c, r, rs);
    }
  }
  // Issue the residual (skip) loads of a chunk; they can be left in flight across other work.
  __device__ static __forceinline__ void prefetch(const Params& p, const EpiCtx& c, float4 (&rs)[8]) {
    if constexpr (MASKED) {
      prefetch_masked(p, c, rs);
      return;
    }
    {
      const Plan pl = plan_of(p, c);
      if (pl.fast) {
        if (p.resid) {
          const uint16_t* rp = static_cast<const uint16_t*>(p.resid) + pl.idx0;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const uint2 u = *reinterpret_cast<const uint2*>(rp);     // the loaded BITS (converted in finish())
            rp += pl.stride;
            rs[i] = make_float4(__uint_as_float(u.x), __uint_as_float(u.y), 0.f, 0.f);
          }
        }
        return;
      }
    }
    const Seg sg = seg_of(p, c);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      size_t idx;
      const bool ok = seg_index(p, c, sg, i, &idx);
      rs[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok && p.resid) {
        if (p.raw16) {
          // keep the loaded BITS (converted in finish()): touching the value here would wait for the load and
          // defeat the point of requesting the skip rows early
          const uint2 u = *reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(p.resid) + idx);
          rs[i] = make_float4(__uint_as_float(u.x), __uint_as_float(u.y), 0.f, 0.f);
        } else {
          rs[i] = *reinterpret_cast<const float4*>(static_cast<const float*>(p.resid) + idx);
        }
      }
    }
  }
  __device__ static __forceinline__ void finish(const Params& p, const EpiCtx& c, const uint32_t (&r)[32],
                                                const float4 (&rs)[8]) {
    if constexpr (MASKED) {
      finish_masked(p, c, r, rs);
      return;
    }
    {
      const Plan pl = plan_of(p, c);
      if (pl.fast) {
        if (p.resid) {
          if (p.raw_out) finish_fast<true, true, true>(p, c, pl, r, rs);
          else finish_fast<true, false, true>(p, c, pl, r, rs);    // last unit of a block: nobody reads its raw output
        } else {
          if (p.raw_out) finish_fast<false, true, true>(p, c, pl, r, rs);
          else finish_fast<false, false, true>(p, c, pl, r, rs);
        }
        return;
      }
    }
    float* st = c.stage;
    const int g = c.lane & 7, r0 = c.lane >> 3;
    {
      float4* mine = reinterpret_cast<float4*>(st + c.lane * 36);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        mine[j] = make_float4(__uint_as_float(r[4 * j]), __uint_as_float(r[4 * j + 1]), __uint_as_float(r[4 * j + 2]),
                              __uint_as_float(r[4 * j + 3]));
    }
    __syncwarp();
    const Seg sg = seg_of(p, c);
    const int co = sg.co;
    ulonglong2 b2 = make_ulonglong2(0ull, 0ull), a2 = b2, ib2 = b2;   // (x,y) and (z,w) pairs; 0 bits = 0.f
    if (p.bias) b2 = __ldg(reinterpret_cast<const ulonglong2*>(p.bias + co));
    const bool snake = p.s16_out != nullptr && p.sn_a != nullptr;
    if (snake) {
      a2 = __ldg(reinterpret_cast<const ulonglong2*>(p.sn_a + co));
      ib2 = __ldg(reinterpret_cast<const ulonglong2*>(p.sn_ib + co));
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      size_t idx;
      if (seg_index(p, c, sg, i, &idx)) {
        const ulonglong2 acc = *reinterpret_cast<const ulonglong2*>(st + (r0 + 4 * i) * 36 + 4 * g);
        uint64_t r01, r23;
        if (p.raw16 && p.resid) {
          const float2 lo = Op16<BF16>::unpack(__float_as_uint(rs[i].x)), hi = Op16<BF16>::unpack(__float_as_uint(rs[i].y));
          r01 = f2_pack(lo.x, lo.y);
          r23 = f2_pack(hi.x, hi.y);
        } else {
          r01 = f2_pack(rs[i].x, rs[i].y);
          r23 = f2_pack(rs[i].z, rs[i].w);
        }
        uint64_t v01 = f2_add(acc.x, f2_add(b2.x, r01));
        uint64_t v23 = f2_add(acc.y, f2_add(b2.y, r23));
        if (p.raw_out) {
          if (p.raw16) {
            float y0, y1, y2, y3;
            f2_unpack(v01, y0, y1);
            f2_unpack(v23, y2, y3);
            *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.raw_out) + idx) =
                make_uint2(Op16<BF16>::pack(y0, y1), Op16<BF16>::pack(y2, y3));
          } else {
            *reinterpret_cast<ulonglong2*>(static_cast<float*>(p.raw_out) + idx) = make_ulonglong2(v01, v23);
          }
        }
        if (p.s16_out) {
          if (snake) {
            v01 = snake_fast2(v01, a2.x, ib2.x);
            v23 = snake_fast2(v23, a2.y, ib2.y);
          }
          float x0, x1, x2, x3;
          f2_unpack(v01, x0, x1);
          f2_unpack(v23, x2, x3);
          const uint32_t h01 = Op16<BF16>::pack(x0, x1), h23 = Op16<BF16>::pack(x2, x3);
          *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.s16_out) + idx) = make_uint2(h01, h23);
          if (p.s16_lo_out) {
            const float2 a = Op16<BF16>::unpack(h01), b = Op16<BF16>::unpack(h23);
            *reinterpret_cast<uint2*>(static_cast<uint16_t*>(p.s16_lo_out) + idx) =
                make_uint2(Op16<BF16>::pack(x0 - a.x, x1 - a.y), Op16<BF16>::pack(x2 - b.x, x3 - b.y));
          }
        }
      }
    }
    __syncwarp();
  }
  // residual values of this lane's 8 row segments are requested first so that the loads are in
  // flight during the smem transpose
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[32]) {
    float4 rs[8];
    prefetch(p, c, rs);
    finish(p, c, r, rs);
  }
};

// out[b, n, l] (NCL fp32) = acc + bias[n]; consecutive lanes hold consecutive l, so every
// per-column store is a coalesced 128 B line.
struct EpiStoreNCL {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  struct Params {
    float* out;
    const float* bias;
    int N;
    int L;
    int do_tanh;
  };
  __device__ static __forceinline__ void apply(const Params& p, const EpiCtx& c, const uint32_t (&r)[32]) {
    if (!c.valid) return;
    float* o = p.out + (static_cast<size_t>(c.batch) * p.N + c.col0) * p.L + c.l;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (c.col0 + j < p.N) {
        const float v = __uint_as_float(r[j]) + (p.bias ? __ldg(p.bias + c.col0 + j) : 0.f);
        o[static_cast<size_t>(j) * p.L] = p.do_tanh ? tanhf(v) : v;
      }
    }
  }
};

// ------------------------------------------------------------------ host side
int make_tmap_a(CUtensorMap* m, const void* ptr, int K, int L, int batches, int64_t row_stride_elems,
                int64_t batch_stride_elems, int stride = 1, int box_rows = kBlockM);
int make_tmap_b(CUtensorMap* m, const void* ptr, int K, int rows, int64_t row_stride_elems, int box_rows);

template <class Epi, int BN, bool BF16>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& s, const typename Epi::Params& ep,
                cudaStream_t stream, const CUtensorMap* tmA2 = nullptr) {
  using Cfg = GemmCfg<BN, Epi::kCols, Epi::kStageBytes>;
  auto kern = gemm_wgmma_kernel<Epi, BN, BF16>;
  static PerDeviceOnce attr;
  if (attr.first()) SATB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  const int m_tiles = ceil_div(s.L, kBlockM), n_tiles = ceil_div(s.N, BN);
  const int total = m_tiles * s.batches * n_tiles;
  if (total <= 0) return 0;
  int grid = device_sm_count();
  if (grid > total) grid = total;
  SATB_REQUIRE(s.n_parts == 1 || tmA2 != nullptr, "split-operand GEMM needs the second A tensor map");
  SATB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, tmA, tmB, tmA2 ? *tmA2 : tmA, s, ep));
  count_launch();
  return 0;
}

}  // namespace satb
