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
//                                      fused epilogue (the DiT linears: fused op on the fragment -> global; EpiHeadNorm16
//                                      and the convolutions: accumulator -> smem -> one row per thread -> fused op -> global)
// The producer runs ahead into the next tile's k-blocks while the epilogue of the current one runs.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "fp8.cuh"
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
// kCols: columns per accumulator staging chunk, 0 for an epilogue that works on the accumulator fragment (no staging).
// kEpiStage: bytes of epilogue staging smem per epilogue warp.
template <int BN, int kCols, int kEpiStage = 0>
struct GemmCfg {
  static constexpr int kStageA = kBlockM * kBlockK * 2;
  static constexpr int kStageB = BN * kBlockK * 2;
  static constexpr int kStage = kStageA + kStageB;
  static constexpr int kAccLd = kCols + 4;              // fp32 row pitch of the accumulator staging tile
  static constexpr int kAccStage = kCols ? 2 * 64 * kAccLd * 4 : 0;   // per MMA warpgroup: two column chunks of its 64 rows
  static constexpr int kFixed = 1024 /*align slack*/ + 256 /*barriers*/ + 2 * kAccStage + kEpiWarps * kEpiStage;
  static constexpr int kStages = (kSmemBudget - kFixed) / kStage > 8 ? 8 : (kSmemBudget - kFixed) / kStage;
  static constexpr int kSmemBytes = kStages * kStage + kFixed;
  static_assert(BN == 64 || BN == 128 || BN == 256, "BN must be 64/128/256");
  static_assert(kStages >= 2, "shared memory too small for a two-stage ring");
};

// An epilogue with `static constexpr bool kFragment = true` receives the MMA warpgroup's accumulator fragment itself
// (Epi::apply_fragment) instead of row chunks staged through shared memory (Epi::apply).
template <class Epi, class = void>
struct EpiFragment : std::false_type {};
template <class Epi>
struct EpiFragment<Epi, std::void_t<decltype(Epi::kFragment)>> : std::bool_constant<Epi::kFragment> {};
template <class Epi>
constexpr int kStagedCols = EpiFragment<Epi>::value ? 0 : Epi::kCols;

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
};

// Epilogue of one 128 x BN tile, run by MMA warpgroup cw (rows [64 cw, 64 cw + 64)) on its accumulator fragment.
// The accumulator goes through shared memory (acc_st: 2 x 64 x (kCols + 4) fp32 per warpgroup) two column chunks at a
// time, so that every epilogue thread receives kCols consecutive columns of ONE row (thread = row, as the epilogues
// expect).  epi_st: the epilogue's own per-warp staging (Epi::kStageBytes), or null.
template <class Epi, int BN>
__device__ __forceinline__ void gemm_tile_epilogue(const float (&acc)[BN / 2], float* acc_st, float* epi_st,
                                                   const typename Epi::Params& ep, int L, int N, int m0, int n0, int batch,
                                                   int cw, int warp, int lane) {
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
  c.stage = epi_st;
  int n_valid = (N - n0 + Epi::kCols - 1) / Epi::kCols;   // chunks that hold real columns (warp-uniform)
  if (n_valid > kChunks) n_valid = kChunks;
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
      Epi::apply(ep, c, r);
    }
  }
}
// FP8 operand mode (FP8 = true): A and B hold e4m3 bytes, one power-of-two scale per A row and per B row.  A k-block
// is then 128 elements (the same 128 B per row, so the ring, its boxes and its barriers are unchanged) and takes four
// m64nBNk32 e4m3 MMAs; the accumulator is dequantised, acc *= a_scale[row] * w_scale[col], before the epilogue runs
// (exact: a product of powers of two).  K must be a multiple of 128.  Unused by the 16-bit instances.
struct Fp8Scales {
  const float* a = nullptr;   // [rows of A]
  const float* w = nullptr;   // [rows of B] = [N]
};
constexpr int kBlockKFp8 = 128;   // 128 x 8-bit = 128 B

// Block-scaled A (the FP8 FF-out option): an FP8 instance whose epilogue type is BlockScaledA<Epi> reads A with one
// power-of-two scale per (row, k-block of 128), sc.a [rows of A, K / 128], instead of one per row.  Each k-block's four
// e4m3 MMAs go into a temporary accumulator, which is retired (wgmma.wait_group 0) and promoted into the accumulator,
// acc += tmp * a_scale[row, kb] (exact: the scale is a power of two); w_scale[col] is applied once before the epilogue.
// The flag rides on the epilogue type so that the existing instances keep their template arguments.  BN 128 only: the
// two accumulators take 64 + 64 registers.
template <class Epi>
struct BlockScaledA : Epi {
  static constexpr bool kBlockScaledA = true;
};
template <class Epi, class = void>
struct EpiBlockScaledA : std::false_type {};
template <class Epi>
struct EpiBlockScaledA<Epi, std::void_t<decltype(Epi::kBlockScaledA)>> : std::bool_constant<Epi::kBlockScaledA> {};

template <class Epi, int BN, bool BF16, bool FP8 = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmA2, const GemmShape s, const typename Epi::Params ep,
                  const Fp8Scales sc) {
  static_assert(!(FP8 && BF16), "the FP8 mode keeps fp16 as its 16-bit type");
  constexpr bool kBlockA = EpiBlockScaledA<Epi>::value;
  static_assert(!kBlockA || (FP8 && BN == 128), "block-scaled A: FP8 operands, BN 128");
  constexpr int kKElems = FP8 ? kBlockKFp8 : kBlockK;   // elements of one k-block
  using Cfg = GemmCfg<BN, kStagedCols<Epi>, Epi::kStageBytes>;
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
  const int kb_per_tap = (s.K + kKElems - 1) / kKElems;
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
          const int k0 = (kbp - tap * kb_per_tap) * kKElems;
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
          const int k0 = (kbp - tap * kb_per_tap) * kKElems;
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
      if constexpr (kBlockA) {
        // block-scaled mainloop (BlockScaledA): rows r0, r0 + 8 of the fragment; the next k-block's scales are
        // requested while this one's MMAs run
        const int r0 = m0 + 64 * cw + 16 * (warp & 3) + (lane >> 2);
        const bool ok0 = r0 < s.L, ok1 = r0 + 8 < s.L;
        const float* sa0 = sc.a + (static_cast<size_t>(batch) * s.L + (ok0 ? r0 : 0)) * num_kb;
        const float* sa1 = sc.a + (static_cast<size_t>(batch) * s.L + (ok1 ? r0 + 8 : 0)) * num_kb;
        float s0 = ok0 ? __ldg(sa0) : 0.f, s1 = ok1 ? __ldg(sa1) : 0.f;
        float tmp[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t a_addr = smem_u32(smem + stage * Cfg::kStage) + cw * 64 * kBlockK * 2;
          const uint32_t b_addr = smem_u32(smem + stage * Cfg::kStage) + Cfg::kStageA;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBlockK / kWgmmaK; ++k)
            wgmma_ss_e4m3<BN>(tmp, make_desc_kmajor_sw128(a_addr + k * kWgmmaK * 2),
                              make_desc_kmajor_sw128(b_addr + k * kWgmmaK * 2), k != 0 ? 1u : 0u);
          wgmma_commit();
          float s0_next = 0.f, s1_next = 0.f;
          if (kb + 1 < num_kb) {
            if (ok0) s0_next = __ldg(sa0 + kb + 1);
            if (ok1) s1_next = __ldg(sa1 + kb + 1);
          }
          wgmma_wait<0>(tmp);
          if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            acc[4 * j] = fmaf(tmp[4 * j], s0, acc[4 * j]);
            acc[4 * j + 1] = fmaf(tmp[4 * j + 1], s0, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(tmp[4 * j + 2], s1, acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(tmp[4 * j + 3], s1, acc[4 * j + 3]);
          }
          s0 = s0_next;
          s1 = s1_next;
          if (++stage == Cfg::kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        const int fc = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + fc;
          const float2 sw = col < s.N ? __ldg(reinterpret_cast<const float2*>(sc.w + col)) : make_float2(0.f, 0.f);
          acc[4 * j] *= sw.x;
          acc[4 * j + 1] *= sw.y;
          acc[4 * j + 2] *= sw.x;
          acc[4 * j + 3] *= sw.y;
        }
        Epi::template apply_fragment<BN>(ep, acc, s.L, s.N, r0, n0, batch, lane);
        continue;
      }
      // mainloop: one wgmma group per k-block; the smem slot of k-block kb - 1 is released once group kb is issued
      // and group kb - 1 has retired
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * Cfg::kStage) + cw * 64 * kBlockK * 2;
        const uint32_t b_addr = smem_u32(smem + stage * Cfg::kStage) + Cfg::kStageA;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {   // 4 x 32 B of every row: k16 (16-bit) or k32 (e4m3) steps
          if constexpr (FP8)
            wgmma_ss_e4m3<BN>(acc, make_desc_kmajor_sw128(a_addr + k * kWgmmaK * 2),
                              make_desc_kmajor_sw128(b_addr + k * kWgmmaK * 2), (kb | k) != 0 ? 1u : 0u);
          else
            wgmma_ss<BN, BF16>(acc, make_desc_kmajor_sw128(a_addr + k * kWgmmaK * 2),
                               make_desc_kmajor_sw128(b_addr + k * kWgmmaK * 2), (kb | k) != 0 ? 1u : 0u);
        }
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
      if constexpr (FP8) {
        // dequantise the fragment (ptx.cuh wgmma_ss layout): rows r0, r0 + 8, column pairs 8 j + fc, + 1
        const int r0 = m0 + 64 * cw + 16 * (warp & 3) + (lane >> 2);
        const int fc = 2 * (lane & 3);
        const float* sa_row = sc.a + static_cast<size_t>(batch) * s.L;
        const float sa0 = r0 < s.L ? __ldg(sa_row + r0) : 0.f;
        const float sa1 = r0 + 8 < s.L ? __ldg(sa_row + r0 + 8) : 0.f;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + fc;
          const float2 sw = col < s.N ? __ldg(reinterpret_cast<const float2*>(sc.w + col)) : make_float2(0.f, 0.f);
          acc[4 * j] *= sa0 * sw.x;
          acc[4 * j + 1] *= sa0 * sw.y;
          acc[4 * j + 2] *= sa1 * sw.x;
          acc[4 * j + 3] *= sa1 * sw.y;
        }
      }

      if constexpr (EpiFragment<Epi>::value)
        Epi::template apply_fragment<BN>(ep, acc, s.L, s.N, m0 + 64 * cw + 16 * (warp & 3) + (lane >> 2), n0, batch, lane);
      else
        gemm_tile_epilogue<Epi, BN>(acc, acc_st, epi_st, ep, s.L, s.N, m0, n0, batch, cw, warp, lane);
    }
  }
}

// ------------------------------------------------------------------ epilogues
// A staged epilogue (Epi::apply) receives kCols consecutive fp32 accumulator columns of one row (as raw bits in r[]);
// a fragment epilogue (Epi::apply_fragment<BN>) receives the wgmma fragment of its warpgroup's 64 rows x BN columns
// (ptx.cuh wgmma_ss): row0 is the thread's first fragment row (the second is row0 + 8), and in every 8-column group j
// it holds columns 8 j + 2 (lane & 3), + 1 at acc[4 j], acc[4 j + 1] (row0) and acc[4 j + 2], acc[4 j + 3] (row0 + 8).
// Both write straight to global memory.  kCols of a fragment epilogue is the column multiple N must have.

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

// Stores one fragment row's 16-bit pairs of two neighbouring 8-column groups starting at column c0: w0 holds columns
// c0 + fc, + 1 and w1 holds c0 + 8 + fc, + 1 (fc = 2 (lane & 3)).  The lanes with fc = 0 and 2, and those with fc = 4
// and 6, swap one word, so that the even lane stores columns c0 + fc .. + 3 and the odd one c0 + 8 + fc - 2 .. + 3 as
// 8 bytes each: the four lanes of a row write one whole 32-byte sector per store instead of four 4-byte pieces of two
// sectors.  Every lane of the warp must take part (the swap is a warp shuffle); `ok` only gates the store.
__device__ __forceinline__ void store16_group_pair(uint16_t* row, int c0, uint32_t w0, uint32_t w1, int lane, bool ok) {
  const bool odd = lane & 1;
  const uint32_t got = __shfl_xor_sync(0xffffffffu, odd ? w0 : w1, 1);
  const int fc = 2 * (lane & 3);
  if (ok) *reinterpret_cast<uint2*>(row + c0 + (odd ? 6 + fc : fc)) = odd ? make_uint2(got, w1) : make_uint2(w0, got);
}

// out16[row, col] = act(acc + bias)   (act: 0 none, 1 SiLU); stored by store16_group_pair, two 8-column groups at a
// time (N is a multiple of 32, so a pair of groups is either wholly inside N or wholly past it).
template <bool BF16>
struct EpiStore16 {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    void* out;
    int ld;
    const float* bias;  // may be null
    int act;
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; j += 2) {
      if (n0 + 8 * j >= N) break;
      float2 b[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
      if (p.bias) {
        b[0] = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + fc));
        b[1] = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + 8 + fc));
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        uint32_t w[2];
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          float x0 = acc[4 * (j + g) + 2 * rr], x1 = acc[4 * (j + g) + 2 * rr + 1];
          if (p.bias) {
            x0 += b[g].x;
            x1 += b[g].y;
          }
          if (p.act == 1) {
            x0 = silu_f(x0);
            x1 = silu_f(x1);
          }
          w[g] = Op16<BF16>::pack(x0, x1);
        }
        store16_group_pair(static_cast<uint16_t*>(p.out) + static_cast<size_t>(batch * L + l) * p.ld, n0 + 8 * j, w[0],
                           w[1], lane, l < L);
      }
    }
  }
};

// out32[row, col] = acc (+ bias); each thread stores its fp32 pairs (c, c + 1).
struct EpiStore32 {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    float* out;
    int ld;
    const float* bias;
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      if (n0 + 8 * j >= N) break;
      const int col = n0 + 8 * j + fc;
      float2 b = make_float2(0.f, 0.f);
      if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        if (l >= L) continue;
        float2 v = make_float2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
        if (p.bias) {
          v.x += b.x;
          v.y += b.y;
        }
        *reinterpret_cast<float2*>(p.out + static_cast<size_t>(batch * L + l) * p.ld + col) = v;
      }
    }
  }
};

// EpiStore32 plus one row of a position table: out32[row, col] = acc (+ bias) + pos[row % n_seq, col], pos [n_seq, N]
// fp32.  The DiT's project_in runs it to add the positional embedding (transformer.py:784-785) to every item's n_seq
// rows.  A type of its own, so that the plain EpiStore32 instances stay as they are.
struct EpiStore32Pos {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    float* out;
    int ld;
    const float* bias;  // may be null
    const float* pos;
    int n_seq;
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
    const float* prow[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
      prow[rr] = p.pos + static_cast<size_t>((batch * L + row0 + 8 * rr) % p.n_seq) * N;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      if (n0 + 8 * j >= N) break;
      const int col = n0 + 8 * j + fc;
      float2 b = make_float2(0.f, 0.f);
      if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        if (l >= L) continue;
        const float2 e = __ldg(reinterpret_cast<const float2*>(prow[rr] + col));
        float2 v = make_float2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
        if (p.bias) {
          v.x += b.x;
          v.y += b.y;
        }
        v.x += e.x;
        v.y += e.y;
        *reinterpret_cast<float2*>(p.out + static_cast<size_t>(batch * L + l) * p.ld + col) = v;
      }
    }
  }
};

// Residual stream update (models/transformer.py:692-700 and adaLN :670-689):
//   h[row, col] += (acc + bias[col]) * gate[row / rows_per_item, col]
// Runs on the accumulator fragment: each thread adds its column pairs (c, c + 1) of rows row0 and row0 + 8 with one
// fire-and-forget fp32 vector reduction in L2 each, so every warp-wide reduction covers whole 32-byte sectors.  Every
// element receives exactly one add per GEMM (no split-K), so the result is deterministic.
struct EpiResidual {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    float* h;
    int ld;
    const float* bias;  // may be null
    const float* gate;  // may be null; sigmoid(1 - gate) precomputed, row stride gate_ld
    int rows_per_item;
    int gate_ld;
    int n_items;        // item = (row / rows_per_item) % n_items (CFG halves share the conditioning)
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
    const float* grow[2] = {nullptr, nullptr};
    float* hrow[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int row = batch * L + row0 + 8 * rr;
      hrow[rr] = p.h + static_cast<size_t>(row) * p.ld + n0 + fc;
      if (p.gate) grow[rr] = p.gate + static_cast<size_t>((row / p.rows_per_item) % p.n_items) * p.gate_ld + n0 + fc;
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      if (n0 + 8 * j >= N) break;
      float2 b = make_float2(0.f, 0.f);
      if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + fc + 8 * j));
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (row0 + 8 * rr >= L) continue;
        float2 v = make_float2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
        if (p.bias) {
          v.x += b.x; v.y += b.y;
        }
        if (p.gate) {
          const float2 gg = __ldg(reinterpret_cast<const float2*>(grow[rr] + 8 * j));
          v.x *= gg.x; v.y *= gg.y;
        }
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(hrow[rr] + 8 * j), "f"(v.x), "f"(v.y) : "memory");
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
// Runs on the accumulator fragment: pair (i, i + 16) of a chunk lies in the same thread, in fragment groups jj and
// jj + 2 of the chunk (i = 8 jj + 2 (lane & 3) + e, jj < 2), so the thread rotates its own pairs of rows row0 and
// row0 + 8 with the table entries of its own columns; the 16-bit results go straight to global memory through
// store16_group_pair.
template <bool BF16>
struct EpiQkvRope {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    void* out;
    int ld;            // 3*D
    int rope_cols;     // 2*D : columns >= this (v) are never rotated
    int seq_len;       // tokens per item (position = row % seq_len)
    int head_dim;      // 32, 64, 96 or 128
    int nf;            // rotary frequencies per head (table row stride): 16, 16, 24, 32
    const float* cos_tab;  // [seq_len, nf]
    const float* sin_tab;  // [seq_len, nf]
  };
  // t*cos + rotate_half(t)*sin with rotate_half = [-b, a]: a' = a c - b s, b' = b c + a s.  The contraction is spelled
  // out (b s and b c rounded, then one fused multiply-add with a) so the bits do not depend on how the compiler would
  // contract the plain expressions; this is the contraction the expressions a * c - b * s and b * c + a * s compile to.
  __device__ static __forceinline__ void rotate(float& a, float& b, float c, float s) {
    const float ra = __fmaf_rn(a, c, -__fmul_rn(b, s));
    const float rb = __fmaf_rn(a, s, __fmul_rn(b, c));
    a = ra;
    b = rb;
  }
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
    // Only chunks 0 and 1 of a head rotate (nf <= 32), and every rotating chunk with the same ci uses the same table
    // entries: (cos, sin) of columns 16 ci + 8 jj + fc, + 1 at the positions of rows row0 and row0 + 8.  They are
    // loaded once, up front, so that the loads are in flight together instead of one round trip per group.
    float2 tc[2][2][2], ts[2][2][2];   // [ci][jj][rr]
    const bool tile_rot = n0 < p.rope_cols && p.cos_tab;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int pos = (batch * L + row0 + 8 * rr) % p.seq_len;   // a row past L still has a position in the table
#pragma unroll
      for (int ci = 0; ci < 2; ++ci) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          tc[ci][jj][rr] = ts[ci][jj][rr] = make_float2(0.f, 0.f);
          if (tile_rot && 8 * jj + fc < p.nf - 16 * ci) {
            const int t = pos * p.nf + 16 * ci + 8 * jj + fc;
            tc[ci][jj][rr] = __ldg(reinterpret_cast<const float2*>(p.cos_tab + t));
            ts[ci][jj][rr] = __ldg(reinterpret_cast<const float2*>(p.sin_tab + t));
          }
        }
      }
    }
#pragma unroll
    for (int ch = 0; ch < BN / 32; ++ch) {
      const int col0 = n0 + 32 * ch;
      if (col0 >= N) break;
      // chunk of 32 columns aligned to 32 (head_dim is a multiple of 32): its rotary pairs (i, i + 16), i < n_rot
      const int ci = (col0 % p.head_dim) >> 5;
      const int n_rot = col0 < p.rope_cols && p.cos_tab ? min(max(p.nf - 16 * ci, 0), 16) : 0;   // 16, 8 or 0
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        uint32_t w[4];                              // 16-bit pairs of groups 0..3 of the chunk, this row
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int i = 8 * jj + fc;               // pair index of this thread's first column in the group
          const int ia = 4 * (4 * ch + jj) + 2 * rr, ib = ia + 8;   // groups jj and jj + 2 of the chunk
          float a0 = acc[ia], a1 = acc[ia + 1], b0 = acc[ib], b1 = acc[ib + 1];
          if (i < n_rot) {                         // n_rot is even, so pair i + 1 is rotated with pair i; ci is 0 or 1
            const float2 cs = ci ? tc[1][jj][rr] : tc[0][jj][rr], sn = ci ? ts[1][jj][rr] : ts[0][jj][rr];
            rotate(a0, b0, cs.x, sn.x);
            rotate(a1, b1, cs.y, sn.y);
          }
          w[jj] = Op16<BF16>::pack(a0, a1);
          w[jj + 2] = Op16<BF16>::pack(b0, b1);
        }
        uint16_t* row = static_cast<uint16_t*>(p.out) + static_cast<size_t>(batch * L + l) * p.ld;
        store16_group_pair(row, col0, w[0], w[1], lane, l < L);
        store16_group_pair(row, col0 + 16, w[2], w[3], lane, l < L);
      }
    }
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

// Where the e4m3 QKV epilogues below put q and k (FP8 self-attention, attention_fp8.cu): columns [0, 64 H) are q and
// [64 H, 128 H) k, stored as e4m3 [rows, 64 H] in q8 / k8 with one power-of-two scale per (row, head) (fp8_row_exp of
// the head's 16-bit values) at s[(item H + head) * scale_ld + token], item = row / seq_len, token = row % seq_len.
struct QkE4m3Out {
  uint8_t *q8, *k8;
  float *sq, *sk;
  int heads;
  int scale_ld;
};
// e4m3 bytes and scale of the (row, head) a value belongs to; `which` 0 = q, 1 = k
__device__ __forceinline__ uint8_t* qk8_row(const QkE4m3Out& o, int which, int row, int head) {
  return (which ? o.k8 : o.q8) + static_cast<size_t>(row) * (64 * o.heads) + 64 * head;
}
__device__ __forceinline__ float* qk8_scale(const QkE4m3Out& o, int which, int row, int head, int seq_len) {
  return (which ? o.sk : o.sq) + static_cast<size_t>(row / seq_len * o.heads + head) * o.scale_ld + row % seq_len;
}

// EpiQkvRope at head dim 64 (nf 16) with q and k stored as e4m3 (QkE4m3Out): the 16-bit values it computes - the same
// row permutation, rotary arithmetic and rounding, so the same bits - are quantised instead of stored.  A head's 64
// columns of a fragment row lie in one quad (8 groups of 8 columns, 2 per lane), so its amax takes two shfl_xor.  v
// columns (>= 128 H) are stored in 16 bits as by EpiQkvRope.  N must be a multiple of 64.
template <bool BF16>
struct EpiQkvRopeE4m3 {
  static constexpr int kCols = 64;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    typename EpiQkvRope<BF16>::Params base;   // head_dim 64, nf 16
    QkE4m3Out o;
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& pp, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const typename EpiQkvRope<BF16>::Params& p = pp.base;
    const int fc = 2 * (lane & 3);
    const int qk_cols = 128 * pp.o.heads;
    float2 tc[2][2], ts[2][2];   // [jj][rr]: (cos, sin) of pair columns 8 jj + fc, + 1 (chunk 0 of every head)
    const bool tile_rot = n0 < p.rope_cols && p.cos_tab;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int pos = (batch * L + row0 + 8 * rr) % p.seq_len;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        tc[jj][rr] = ts[jj][rr] = make_float2(0.f, 0.f);
        if (tile_rot) {
          const int t = pos * p.nf + 8 * jj + fc;
          tc[jj][rr] = __ldg(reinterpret_cast<const float2*>(p.cos_tab + t));
          ts[jj][rr] = __ldg(reinterpret_cast<const float2*>(p.sin_tab + t));
        }
      }
    }
#pragma unroll
    for (int hd = 0; hd < BN / 64; ++hd) {
      const int col0 = n0 + 64 * hd;
      if (col0 >= N) break;
      const bool rot = col0 < p.rope_cols && p.cos_tab;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        const int row = batch * L + l;
        uint32_t w[8];   // 16-bit pairs of the head's 8 column groups, this row
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {   // chunk 0: pairs (i, i + 16), i = 8 jj + fc, + 1, all rotated
          const int ia = 4 * (8 * hd + jj) + 2 * rr, ib = ia + 8;
          float a0 = acc[ia], a1 = acc[ia + 1], b0 = acc[ib], b1 = acc[ib + 1];
          if (rot) {
            EpiQkvRope<BF16>::rotate(a0, b0, tc[jj][rr].x, ts[jj][rr].x);
            EpiQkvRope<BF16>::rotate(a1, b1, tc[jj][rr].y, ts[jj][rr].y);
          }
          w[jj] = Op16<BF16>::pack(a0, a1);
          w[jj + 2] = Op16<BF16>::pack(b0, b1);
        }
#pragma unroll
        for (int g = 4; g < 8; ++g) {      // chunk 1: passes through
          const int ia = 4 * (8 * hd + g) + 2 * rr;
          w[g] = Op16<BF16>::pack(acc[ia], acc[ia + 1]);
        }
        if (col0 < qk_cols) {              // warp-uniform
          float v[16], amax = 0.f;
#pragma unroll
          for (int g = 0; g < 8; ++g) {
            const float2 f = Op16<BF16>::unpack(w[g]);
            v[2 * g] = f.x;
            v[2 * g + 1] = f.y;
            amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
          }
          amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
          amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
          const int e = fp8_row_exp(amax);
          const float inv = pow2f(-e);
          if (l < L) {
            const int which = col0 >= 64 * pp.o.heads, head = (col0 >> 6) - which * pp.o.heads;
            uint8_t* dst = qk8_row(pp.o, which, row, head) + fc;
#pragma unroll
            for (int g = 0; g < 8; ++g)
              *reinterpret_cast<uint16_t*>(dst + 8 * g) = static_cast<uint16_t>(
                  __nv_cvt_float2_to_fp8x2(make_float2(v[2 * g] * inv, v[2 * g + 1] * inv), __NV_SATFINITE, __NV_E4M3));
            if (fc == 0) *qk8_scale(pp.o, which, row, head, p.seq_len) = pow2f(e);
          }
        } else {
          uint16_t* out = static_cast<uint16_t*>(p.out) + static_cast<size_t>(row) * p.ld;
#pragma unroll
          for (int q = 0; q < 4; ++q) store16_group_pair(out, col0 + 16 * q, w[2 * q], w[2 * q + 1], lane, l < L);
        }
      }
    }
  }
};

// EpiHeadNorm16 with q and k stored as e4m3 (QkE4m3Out; norm_cols must be 128 H): the same normalised and rotated
// 16-bit values, quantised per (row, head) instead of stored; v columns are stored in 16 bits as by EpiHeadNorm16.
template <bool BF16>
struct EpiHeadNormE4m3 {
  static constexpr int kCols = 64;
  static constexpr int kStageBytes = 0;
  struct Params {
    typename EpiHeadNorm16<BF16>::Params base;
    QkE4m3Out o;
  };
  __device__ static __forceinline__ void apply(const Params& pp, const EpiCtx& c, const uint32_t (&r)[64]) {
    const typename EpiHeadNorm16<BF16>::Params& p = pp.base;
    if (c.col0 >= p.norm_cols) {
      EpiHeadNorm16<BF16>::apply(p, c, r);
      return;
    }
    if (!c.valid) return;
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 64; ++j) ss = fmaf(__uint_as_float(r[j]), __uint_as_float(r[j]), ss);
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
    float v[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) v[j] = __uint_as_float(r[j]) * inv;
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
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 64; j += 2) {   // the values EpiHeadNorm16 stores
      const float2 f = Op16<BF16>::unpack(Op16<BF16>::pack(v[j], v[j + 1]));
      v[j] = f.x;
      v[j + 1] = f.y;
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
    const int e = fp8_row_exp(amax);
    const float s = pow2f(-e);
    const int which = c.col0 >= 64 * pp.o.heads, head = (c.col0 >> 6) - which * pp.o.heads;
    uint4* dst = reinterpret_cast<uint4*>(qk8_row(pp.o, which, c.row, head));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* x = v + 16 * j;
      dst[j] = make_uint4(e4m3x4(x[0] * s, x[1] * s, x[2] * s, x[3] * s), e4m3x4(x[4] * s, x[5] * s, x[6] * s, x[7] * s),
                          e4m3x4(x[8] * s, x[9] * s, x[10] * s, x[11] * s),
                          e4m3x4(x[12] * s, x[13] * s, x[14] * s, x[15] * s));
    }
    *qk8_scale(pp.o, which, c.row, head, p.seq_len) = pow2f(e);
  }
};

// SwiGLU epilogue (models/transformer.py:232-235: value = first half, gate = second
// half of the projection).  The weight rows are interleaved at load time so every
// 64-column group holds 32 value columns followed by their 32 gate columns:
//   out[row, g*32 + j] = (acc[g*64 + j] + b) * silu(acc[g*64 + 32 + j] + b')
// Value column c and gate column c + 32 of a group sit in the same thread's accumulator fragment (8-column groups j
// and j + 4), so the epilogue runs on the fragment: no staging through shared memory, no barrier, and the 16-bit
// results go straight to global memory through store16_group_pair, two 8-column output groups at a time.
template <bool BF16>
struct EpiSwiglu {
  static constexpr int kCols = 64;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    void* out;
    int ld;             // inner dim (N/2)
    const float* bias;  // interleaved like the weight rows; may be null
  };
  // acc: the wgmma fragment of 64 rows x BN columns (ptx.cuh wgmma_ss); row0: this thread's first fragment row (the
  // second is row0 + 8), lane & 3 selects its column pair in every 8-column group.
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
#pragma unroll
    for (int g = 0; g < BN / 64; ++g) {
      const int col0 = n0 + 64 * g;
      if (col0 >= N) break;
#pragma unroll
      for (int jp = 0; jp < 4; jp += 2) {   // output groups jp, jp + 1 of this 32-column output chunk
        float2 bv[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)}, bg[2] = {bv[0], bv[0]};
        if (p.bias) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c = 8 * (jp + h) + fc;   // value columns c, c + 1; gate columns c + 32, c + 33
            bv[h] = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + c));
            bg[h] = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 32 + c));
          }
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int l = row0 + 8 * rr;
          uint32_t w[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int av = 4 * (8 * g + jp + h) + 2 * rr, ag = av + 16;
            float a0 = acc[av], a1 = acc[av + 1], g0 = acc[ag], g1 = acc[ag + 1];
            if (p.bias) {
              a0 += bv[h].x;
              a1 += bv[h].y;
              g0 += bg[h].x;
              g1 += bg[h].y;
            }
            w[h] = Op16<BF16>::pack(a0 * silu_f(g0), a1 * silu_f(g1));
          }
          store16_group_pair(static_cast<uint16_t*>(p.out) + static_cast<size_t>(batch * L + l) * p.ld,
                             (col0 >> 1) + 8 * jp, w[0], w[1], lane, l < L);
        }
      }
    }
  }
};

// The FF intermediate of the FP8 FF-out option in e4m3 with one power-of-two scale per (row, 128-column block): q [rows,
// ld] e4m3, scale [rows, ld / 128] fp32, by the rule of fp8_row_exp applied to the block's fp32 amax.  One block is one
// k-block of the FF-out GEMM that reads it (BlockScaledA).
struct BlockE4m3Out {
  uint8_t* q;
  float* scale;
  int ld;   // a multiple of 128
};

// Quantises and stores one fragment row's 128-column block starting at column c0: v[2 g], v[2 g + 1] hold columns
// c0 + 8 g + fc, + 1 (g < 16, fc = 2 (lane & 3)), so the quad's four lanes hold the whole block and its amax takes two
// shfl_xor.  Per four groups g0 .. g0 + 3, two exchanges inside the quad (as in store16_group_pair, then between lanes
// q and q ^ 2) leave lane q with all 8 bytes of group g0 + q, so the quad stores one whole 32-byte sector.  Every lane
// of the warp must take part; `ok` gates the stores.
__device__ __forceinline__ void store_e4m3_block(const BlockE4m3Out& o, int row, int c0, const float (&v)[32], int lane,
                                                 bool ok) {
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) amax = fmaxf(amax, fabsf(v[i]));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
  const int e = fp8_row_exp(amax);
  const float inv = pow2f(-e);
  const bool odd = lane & 1, hi = lane & 2;
  uint8_t* dst = o.q + static_cast<size_t>(row) * o.ld + c0 + 8 * (lane & 3);
#pragma unroll
  for (int g0 = 0; g0 < 16; g0 += 4) {
    uint32_t w[4];   // this lane's byte pair of groups g0 .. g0 + 3
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int g = g0 + i;
      w[i] = __nv_cvt_float2_to_fp8x2(make_float2(v[2 * g] * inv, v[2 * g + 1] * inv), __NV_SATFINITE, __NV_E4M3);
    }
    // after the first exchange, lane q holds 4 bytes: of group g0 + (q & 1) in u01, of g0 + 2 + (q & 1) in u23, bytes
    // 0-3 for q < 2 and 4-7 for q >= 2
    const uint32_t got01 = __shfl_xor_sync(0xffffffffu, odd ? w[0] : w[1], 1);
    const uint32_t got23 = __shfl_xor_sync(0xffffffffu, odd ? w[2] : w[3], 1);
    const uint32_t u01 = odd ? got01 | (w[1] << 16) : w[0] | (got01 << 16);
    const uint32_t u23 = odd ? got23 | (w[3] << 16) : w[2] | (got23 << 16);
    const uint32_t got = __shfl_xor_sync(0xffffffffu, hi ? u01 : u23, 2);
    if (ok) *reinterpret_cast<uint2*>(dst + 8 * g0) = hi ? make_uint2(got, u23) : make_uint2(u01, got);
  }
  if (ok && (lane & 3) == 0) o.scale[static_cast<size_t>(row) * (o.ld / 128) + c0 / 128] = pow2f(e);
}

// EpiSwiglu with the output stored as e4m3 blocks (BlockE4m3Out) instead of 16 bits: the same fp32 values, quantised.
// BN 256: a tile's 128 output columns are one block.  N a multiple of 256.
struct EpiSwigluE4m3 {
  static constexpr int kCols = 256;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    BlockE4m3Out o;     // ld: inner dim (N / 2)
    const float* bias;  // interleaved like the weight rows; may be null
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    static_assert(BN == 256, "one tile = one 128-column output block");
    const int fc = 2 * (lane & 3);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int l = row0 + 8 * rr;
      float v[32];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {   // value columns c, c + 1 and gate columns c + 32, c + 33 of group g
          const int c = n0 + 64 * g + 8 * jj + fc;
          const int av = 4 * (8 * g + jj) + 2 * rr, ag = av + 16;
          float a0 = acc[av], a1 = acc[av + 1], g0 = acc[ag], g1 = acc[ag + 1];
          if (p.bias) {
            const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + c));
            const float2 bg = __ldg(reinterpret_cast<const float2*>(p.bias + c + 32));
            a0 += bv.x;
            a1 += bv.y;
            g0 += bg.x;
            g1 += bg.y;
          }
          v[2 * (4 * g + jj)] = a0 * silu_f(g0);
          v[2 * (4 * g + jj) + 1] = a1 * silu_f(g1);
        }
      }
      store_e4m3_block(p.o, batch * L + l, n0 >> 1, v, lane, l < L);
    }
  }
};

// The plain-SiLU FF-in (EpiStore16 with act 1) with the output stored as e4m3 blocks (BlockE4m3Out): silu(acc + bias).
// N a multiple of 128.
struct EpiSiluE4m3 {
  static constexpr int kCols = 128;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    BlockE4m3Out o;     // ld: N
    const float* bias;  // may be null
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
#pragma unroll
    for (int blk = 0; blk < BN / 128; ++blk) {
      const int c0 = n0 + 128 * blk;
      if (c0 >= N) break;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        float v[32];
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          const int a = 4 * (16 * blk + g) + 2 * rr;
          float x0 = acc[a], x1 = acc[a + 1];
          if (p.bias) {
            const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + c0 + 8 * g + fc));
            x0 += b.x;
            x1 += b.y;
          }
          v[2 * g] = silu_f(x0);
          v[2 * g + 1] = silu_f(x1);
        }
        store_e4m3_block(p.o, batch * L + l, c0, v, lane, l < L);
      }
    }
  }
};

// ------------------------------------------------------- T5 feed-forward epilogues (t5.cu)
// Two 16-bit pairs of the T5 encoder's FF-in activations.  In fp16 the values saturate to +-65504 instead of rounding
// to infinity (cvt .satfinite; a NaN stays NaN): the encoder's overflow behaviour, where the reference's fp16 model
// clamps its infinities afterwards (modeling_t5.py:451-456).  bf16 has the range of fp32 and is stored as is.
template <bool BF16>
__device__ __forceinline__ uint32_t pack16_satfinite(float a, float b) {
  if constexpr (BF16) {
    return Op16<true>::pack(a, b);
  } else {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
  }
}

// T5 FF-in with the ReLU of T5DenseActDense (modeling_t5.py:84-103): out16[row, col] = max(acc, 0), saturating.  A type
// of its own so that EpiStore16 keeps no runtime activation branch for it.  N a multiple of 32.
template <bool BF16>
struct EpiRelu16 {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    void* out;
    int ld;
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
#pragma unroll
    for (int j = 0; j < BN / 8; j += 2) {
      if (n0 + 8 * j >= N) break;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        uint32_t w[2];
#pragma unroll
        for (int g = 0; g < 2; ++g)
          w[g] = pack16_satfinite<BF16>(fmaxf(acc[4 * (j + g) + 2 * rr], 0.f), fmaxf(acc[4 * (j + g) + 2 * rr + 1], 0.f));
        store16_group_pair(static_cast<uint16_t*>(p.out) + static_cast<size_t>(batch * L + l) * p.ld, n0 + 8 * j, w[0],
                           w[1], lane, l < L);
      }
    }
  }
};

// gelu_new (the tanh form, transformers activations.NewGELUActivation): 0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3)))
__device__ __forceinline__ float gelu_tanh_f(float x) {
  return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * fmaf(0.044715f * x, x * x, x)));
}

// T5 FF-in of T5DenseGatedActDense (modeling_t5.py:106-130): out16[row, c] = gelu_new(x wi_0[c]) * (x wi_1[c]),
// saturating.  The weight is [wi_1; wi_0] interleaved at load time as swiglu_perm does (every 64 rows: 32 rows of wi_1,
// then the same 32 rows of wi_0), so value column c and gate column c + 32 sit in one thread's fragment as in EpiSwiglu.
// N (= 2 d_ff) a multiple of 64; out [M, N / 2].
template <bool BF16>
struct EpiGeglu16 {
  static constexpr int kCols = 64;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    void* out;
    int ld;   // d_ff (N / 2)
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
#pragma unroll
    for (int g = 0; g < BN / 64; ++g) {
      const int col0 = n0 + 64 * g;
      if (col0 >= N) break;
#pragma unroll
      for (int jp = 0; jp < 4; jp += 2) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int l = row0 + 8 * rr;
          uint32_t w[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int av = 4 * (8 * g + jp + h) + 2 * rr, ag = av + 16;
            w[h] = pack16_satfinite<BF16>(acc[av] * gelu_tanh_f(acc[ag]), acc[av + 1] * gelu_tanh_f(acc[ag + 1]));
          }
          store16_group_pair(static_cast<uint16_t*>(p.out) + static_cast<size_t>(batch * L + l) * p.ld,
                             (col0 >> 1) + 8 * jp, w[0], w[1], lane, l < L);
        }
      }
    }
  }
};

// ------------------------------------------------------- RoBERTa feed-forward epilogue (roberta.cu)
// The exact erf GELU of transformers' ACT2FN["gelu"] (GELUActivation, torch.nn.functional.gelu), not gelu_new.
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// RoBERTa FF-in (RobertaIntermediate): out16[row, col] = gelu(acc + bias[col]), saturating in fp16 like EpiRelu16.
// N a multiple of 32.
template <bool BF16>
struct EpiBiasGelu16 {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 0;
  static constexpr bool kFragment = true;
  struct Params {
    void* out;
    int ld;
    const float* bias;
  };
  template <int BN>
  __device__ static __forceinline__ void apply_fragment(const Params& p, const float (&acc)[BN / 2], int L, int N,
                                                        int row0, int n0, int batch, int lane) {
    const int fc = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; j += 2) {
      if (n0 + 8 * j >= N) break;
      const float2 b[2] = {__ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + fc)),
                           __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + 8 + fc))};
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int l = row0 + 8 * rr;
        uint32_t w[2];
#pragma unroll
        for (int g = 0; g < 2; ++g)
          w[g] = pack16_satfinite<BF16>(gelu_erf_f(acc[4 * (j + g) + 2 * rr] + b[g].x),
                                        gelu_erf_f(acc[4 * (j + g) + 2 * rr + 1] + b[g].y));
        store16_group_pair(static_cast<uint16_t*>(p.out) + static_cast<size_t>(batch * L + l) * p.ld, n0 + 8 * j, w[0],
                           w[1], lane, l < L);
      }
    }
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

// The activation a convolution epilogue applies to the 16-bit copy it writes (the consuming layer's activation,
// models/autoencoders.py:29-42): a template parameter of every kernel that applies one.
constexpr int kActSnake = 0;   // SnakeBeta (use_snake=True), per-channel a = e^alpha, ib = 1/(e^beta + 1e-9)
constexpr int kActElu = 1;     // nn.ELU() (use_snake=False), alpha 1, no parameters

// ELU: v > 0 ? v : e^v - 1.  e^v - 1 through the SFU exponential (ex2.approx) carries an absolute error of up to
// ~2^-21.8, which near 0 exceeds the value's own 16-bit rounding (below |v| ~ 2^-12).  For -2^-6 < v <= 0 the cubic
// Taylor polynomial is used instead: its truncation is < v^4 / 24, i.e. < 2^-22.6 |v| there.  Below -2^-6 the SFU
// value's 2^-21.8 is < 2^-15.8 |e^v - 1|.  Same formulation in every instance (scalar and pair).  The exponential
// flushes subnormal results (e^v < 2^-126, where e^v - 1 is -1 either way), which saves __expf's subnormal fix-up.
__device__ __forceinline__ float elu_fast(float v) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * 1.4426950409f));
  e -= 1.0f;
  const float p = v * fmaf(v, fmaf(v, 0.16666667f, 0.5f), 1.0f);
  return v > 0.0f ? v : (v > -0.015625f ? p : e);
}
template <int ACT>
__device__ __forceinline__ float act_fast(float v, float a, float ib) {
  if constexpr (ACT == kActElu) return elu_fast(v);
  else return snake_fast(v, a, ib);
}
template <int ACT>
__device__ __forceinline__ uint64_t act_fast2(uint64_t v, uint64_t a, uint64_t ib) {
  if constexpr (ACT == kActElu) {
    float x0, x1;
    f2_unpack(v, x0, x1);
    return f2_pack(elu_fast(x0), elu_fast(x1));
  } else {
    return snake_fast2(v, a, ib);
  }
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
  const float* sn_a;    // [cout] e^alpha of the consumer's Snake, or null (plain cast); ELU instances ignore sn_a /
                        // sn_ib and always apply ELU to s16_out
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
// MASKED = true: the kernel carries ONLY the lean path - for launches whose Params satisfy fast_flags(); the host picks
// the instantiation (oobleck.cu run_conv_gemm).  The general path costs ~120 instructions per 4-element segment, ~55 %
// of them index arithmetic, bounds tests and branches on the launch-uniform Params flags, and the 128-channel layers
// are bound by exactly this epilogue.  The lean path computes one index per chunk (the 8 segments of a lane are
// idx0 + i * stride), keeps per-segment validity as a bit mask and makes Snake and the 16-bit raw streams
// unconditional.  Compiled next to the general path in one kernel it pays ~200 bytes of spills in the persistent GEMM
// kernels (long-scoreboard stalls on the reloads, profiles/r02_ncu_convT_s2.txt).
//
// ACT: the activation of the 16-bit output (kActSnake / kActElu).  The body is EpiConvT; the instances are the two
// derived names below, so the Snake instances keep the kernel symbols they had before ACT existed.
template <bool BF16, bool MASKED, int ACT>
struct EpiConvT {
  static constexpr int kCols = 32;
  static constexpr int kStageBytes = 32 * 36 * 4;   // per-warp [32 rows][32 + 4 pad] fp32 transpose tile
  static constexpr int kAct = ACT;
  static constexpr bool kMasked = MASKED;
  typedef EpiConvParams Params;
  // activated 16-bit output, raw streams (if any) in the 16-bit type, no lo copy: what the default fp16 decode runs
  __host__ __device__ static bool fast_flags(const Params& p) {
    return p.s16_out != nullptr && (ACT == kActElu || p.sn_a != nullptr) && p.s16_lo_out == nullptr &&
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
  // ---- lean path (MASKED): the same arithmetic for every chunk, ragged ones included (mask bit i: segment i exists)
  struct Plan {
    long long idx0;   // element index of segment 0 (may point before the buffer when that segment does not exist)
    int stride;
    uint32_t mask;
    int co;
  };
  __device__ static __forceinline__ Plan chunk_plan(const Params& p, const EpiCtx& c) {
    const Seg sg = seg_of(p, c);
    const int l0 = c.l0 + (c.lane >> 3);
    const int lo0 = l0 * p.up + sg.phase - p.pad;
    Plan pl;
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
      const Plan pl = chunk_plan(p, c);
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
    const Plan pl = chunk_plan(p, c);
    const uint32_t st = smem_u32(c.stage);
    const int g = c.lane & 7, r0 = c.lane >> 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) sts128(st + (c.lane * 36 + 4 * j) * 4, r[4 * j], r[4 * j + 1], r[4 * j + 2], r[4 * j + 3]);
    __syncwarp();
    ulonglong2 b2 = make_ulonglong2(0ull, 0ull);
    if (p.bias) b2 = __ldg(reinterpret_cast<const ulonglong2*>(p.bias + pl.co));
    const ulonglong2 a2 = ACT == kActSnake ? __ldg(reinterpret_cast<const ulonglong2*>(p.sn_a + pl.co)) : b2;
    const ulonglong2 ib2 = ACT == kActSnake ? __ldg(reinterpret_cast<const ulonglong2*>(p.sn_ib + pl.co)) : b2;
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
      v01 = act_fast2<ACT>(v01, a2.x, ib2.x);
      v23 = act_fast2<ACT>(v23, a2.y, ib2.y);
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
      else finish_masked_t<true, false>(p, c, r, rs);    // last unit of a block: nobody reads its raw output
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
    const bool act = p.s16_out != nullptr && (ACT == kActElu || p.sn_a != nullptr);
    if (ACT == kActSnake && act) {
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
          if (act) {
            v01 = act_fast2<ACT>(v01, a2.x, ib2.x);
            v23 = act_fast2<ACT>(v23, a2.y, ib2.y);
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
template <bool BF16, bool MASKED = false>
struct EpiConv : EpiConvT<BF16, MASKED, kActSnake> {};
template <bool BF16, bool MASKED = false>
struct EpiConvElu : EpiConvT<BF16, MASKED, kActElu> {};
template <bool BF16, bool MASKED, int ACT>
using EpiConvFor = typename std::conditional<ACT == kActElu, EpiConvElu<BF16, MASKED>, EpiConv<BF16, MASKED>>::type;

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
// elem_bytes: 2 (16-bit operands) or 1 (e4m3); the box is 128 B of every row either way.
int make_tmap_a(CUtensorMap* m, const void* ptr, int K, int L, int batches, int64_t row_stride_elems,
                int64_t batch_stride_elems, int stride = 1, int box_rows = kBlockM, int elem_bytes = 2);
int make_tmap_b(CUtensorMap* m, const void* ptr, int K, int rows, int64_t row_stride_elems, int box_rows,
                int elem_bytes = 2);

template <class Epi, int BN, bool BF16, bool FP8 = false>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& s, const typename Epi::Params& ep,
                cudaStream_t stream, const CUtensorMap* tmA2 = nullptr, const Fp8Scales& sc = Fp8Scales{}) {
  using Cfg = GemmCfg<BN, kStagedCols<Epi>, Epi::kStageBytes>;
  auto kern = gemm_wgmma_kernel<Epi, BN, BF16, FP8>;
  if (FP8)
    SATB_REQUIRE(s.K % kBlockKFp8 == 0 && s.n_taps == 1 && s.n_parts == 1 && s.stride == 1 && sc.a && sc.w,
                 "FP8 GEMM: K must be a multiple of 128, one tap, one part, and both scale vectors given");
  static PerDeviceOnce attr;
  if (attr.first()) SATB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  const int m_tiles = ceil_div(s.L, kBlockM), n_tiles = ceil_div(s.N, BN);
  const int total = m_tiles * s.batches * n_tiles;
  if (total <= 0) return 0;
  int grid = device_sm_count();
  if (grid > total) grid = total;
  SATB_REQUIRE(s.n_parts == 1 || tmA2 != nullptr, "split-operand GEMM needs the second A tensor map");
  SATB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, tmA, tmB, tmA2 ? *tmA2 : tmA, s, ep,
                             sc));
  count_launch();
  return 0;
}

}  // namespace satb
