// k-tap (dilated) convolutions that load every activation row ONCE per tile, as a wgmma implicit GEMM.
//
//   conv[b, l, n] = sum_{t, k} A[b, l + (t - taps/2) * dil, k] * W[t * N + n, k]
//
// TMA brings the 128 + (taps - 1) * dil activation rows of a 64-channel k-block into one 128B-swizzled smem slot, and
// tap t reads it through a matrix descriptor shifted by t * dil rows (make_desc_kmajor_sw128); only the tap
// weights stream through the ring.  The generic GEMM reloads the A tile once per tap (7x the L2 -> SM traffic).
//
// FUSE = false: the decoder's final convolution (128 -> 2 channels, k = 7, models/autoencoders.py:190); the epilogue
// (EpiStoreNCL) ignores the columns >= N of the 64-wide tile.
// FUSE = true: a whole Oobleck ResidualUnit (models/autoencoders.py:45-68), y = x + conv1x1(snake2(conv7(snake1(x)))):
// the conv7 accumulator never leaves the SM - bias + snake2 + 16-bit rounding, written to smem in the swizzled K-major
// layout, feeds a second wgmma chain with the 1x1 weights (streamed through the same ring), whose accumulator goes to
// EpiConv (+ bias + skip, raw stream, the consumer's Snake).  N = channels = 128 or 256.
//
// Same warp roles as gemm_wgmma_kernel: warpgroup 0 one TMA producer thread, warpgroups 1, 2 MMA + epilogue on 64 rows
// each; one persistent CTA per SM over 128-position tiles.
#pragma once
#include "gemm.cuh"

namespace satb {

struct HaloShape {
  int L;         // positions per batch item
  int batches;
  int K;         // input channels (multiple of 64)
  int n_taps;    // odd
  int dil;       // (n_taps - 1) * dil <= kHaloMax
  int N;         // output channels (rows of W per tap)
};

struct ResUnitPre {      // FUSE: the inner conv7 -> snake2 step (ELU instead when Epi::kAct is kActElu)
  const float* bias7;    // [N] or null
  const float* sn2_a;    // e^alpha of snake2 (unused by ELU)
  const float* sn2_ib;   // 1/(e^beta + 1e-9) of snake2 (unused by ELU)
};

constexpr int kHaloMax = 54;   // halo rows beyond the tile: 6 taps x dilation 9

template <int BN, int kCols, int kEpiStage, bool FUSE>
struct HaloCfg {
  static constexpr int kSlotA = ((kBlockM + kHaloMax) * 128 + 1023) / 1024 * 1024;   // 24 KB halo slot
  static constexpr int kStagesA = 2;
  static constexpr int kStageB = BN * kBlockK * 2;
  static constexpr int kA2 = FUSE ? kBlockM * BN * 2 : 0;                // snake2(conv7) tile, BN / 64 swizzled atoms
  static constexpr int kAccStage = 2 * 64 * (kCols + 4) * 4;             // per MMA warpgroup (gemm_tile_epilogue)
  static constexpr int kShared = kA2 > 2 * kAccStage ? kA2 : 2 * kAccStage;   // the A2 tile and the accumulator
                                                                          // staging take turns in one region
  static constexpr int kFixed = 1024 + kStagesA * kSlotA + kShared + 256 + kEpiWarps * kEpiStage;
  static constexpr int kStagesB = (kSmemBudget - kFixed) / kStageB > 8 ? 8 : (kSmemBudget - kFixed) / kStageB;
  static constexpr int kSmemBytes = kFixed + kStagesB * kStageB;
  static_assert(kStagesB >= 2, "shared memory too small for a two-stage weight ring");
};

template <class Epi, int BN, bool BF16, bool FUSE>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv_halo_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmB1, const HaloShape s, const ResUnitPre pre,
                       const typename Epi::Params ep) {
  using Cfg = HaloCfg<BN, Epi::kCols, Epi::kStageBytes, FUSE>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* slot_a = smem;
  uint8_t* shared = slot_a + Cfg::kStagesA * Cfg::kSlotA;
  uint8_t* ring_b = shared + Cfg::kShared;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring_b + Cfg::kStagesB * Cfg::kStageB);
  uint64_t* full_a = bars;
  uint64_t* empty_a = bars + Cfg::kStagesA;
  uint64_t* full_b = bars + 2 * Cfg::kStagesA;
  uint64_t* empty_b = full_b + Cfg::kStagesB;
  uint8_t* epi_smem = reinterpret_cast<uint8_t*>(bars) + 256;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int m_tiles = (s.L + kBlockM - 1) / kBlockM;
  const int total_tiles = m_tiles * s.batches;
  const int n_kb = s.K / kBlockK;
  const int halo_rows = kBlockM + (s.n_taps - 1) * s.dil;
  const int halo0 = -(s.n_taps / 2) * s.dil;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < Cfg::kStagesA; ++i) {
      mbar_init(&full_a[i], 1);
      mbar_init(&empty_a[i], 2);
    }
    for (int i = 0; i < Cfg::kStagesB; ++i) {
      mbar_init(&full_b[i], 1);
      mbar_init(&empty_b[i], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ------------------------------------------------------------ TMA producer
      pdl_wait();
      int ia = 0, ib = 0;
      uint32_t pa = 0, pb = 0;
      auto load_b = [&](const CUtensorMap* m, int k0, int row) {
        mbar_wait(&empty_b[ib], pb ^ 1);
        mbar_expect_tx(&full_b[ib], Cfg::kStageB);
        tma_load_2d(ring_b + ib * Cfg::kStageB, m, &full_b[ib], k0, row);
        if (++ib == Cfg::kStagesB) {
          ib = 0;
          pb ^= 1;
        }
      };
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int batch = tile / m_tiles;
        const int m0 = (tile - batch * m_tiles) * kBlockM;
        for (int kb = 0; kb < n_kb; ++kb) {
          mbar_wait(&empty_a[ia], pa ^ 1);
          mbar_expect_tx(&full_a[ia], halo_rows * 128);
          tma_load_4d(slot_a + ia * Cfg::kSlotA, &tmA, &full_a[ia], kb * kBlockK, 0, m0 + halo0, batch);
          if (++ia == Cfg::kStagesA) {
            ia = 0;
            pa ^= 1;
          }
          for (int tap = 0; tap < s.n_taps; ++tap) load_b(&tmB, kb * kBlockK, tap * s.N);
        }
        if constexpr (FUSE)
          for (int kb = 0; kb < BN / kBlockK; ++kb) load_b(&tmB1, kb * kBlockK, 0);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    pdl_wait();
    // ------------------------------------------------------------ MMA + epilogue warpgroups
    const int cw = wg - 1;
    const uint32_t tid = threadIdx.x & 127;
    float acc[BN / 2];
    int ia = 0, ib = 0;
    uint32_t pa = 0, pb = 0;
    // one wgmma group per weight stage; a stage is released once the next group is issued and the previous retired
    auto mma_stage = [&](uint32_t a_addr, bool first) {
      mbar_wait(&full_b[ib], pb);
      const uint32_t b_addr = smem_u32(ring_b + ib * Cfg::kStageB);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
        const uint32_t a = a_addr + k * kWgmmaK * 2;
        wgmma_ss<BN, BF16>(acc, make_desc_kmajor_sw128(a),
                           make_desc_kmajor_sw128(b_addr + k * kWgmmaK * 2), (!first || k != 0) ? 1u : 0u);
      }
      wgmma_commit();
    };
    auto retire = [&](int& prev) {   // after mma_stage: retire the previous group and free its stage
      wgmma_wait<1>(acc);
      if (prev >= 0 && tid == 0) mbar_arrive(&empty_b[prev]);
      prev = ib;
      if (++ib == Cfg::kStagesB) {
        ib = 0;
        pb ^= 1;
      }
    };
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int batch = tile / m_tiles;
      const int m0 = (tile - batch * m_tiles) * kBlockM;
      // conv (k taps) over the halo slots
      for (int kb = 0; kb < n_kb; ++kb) {
        mbar_wait(&full_a[ia], pa);
        const uint32_t a_base = smem_u32(slot_a + ia * Cfg::kSlotA) + cw * 64 * 128;
        int prev = -1;
        for (int tap = 0; tap < s.n_taps; ++tap) {
          mma_stage(a_base + tap * s.dil * 128, kb == 0 && tap == 0);
          retire(prev);
        }
        wgmma_wait<0>(acc);
        if (tid == 0) {
          mbar_arrive(&empty_b[prev]);
          mbar_arrive(&empty_a[ia]);
        }
        if (++ia == Cfg::kStagesA) {
          ia = 0;
          pa ^= 1;
        }
      }
      if constexpr (FUSE) {
        named_bar_sync(3, 256);   // both warpgroups have read the previous tile's accumulator staging (same region)
        // acc -> + bias7 -> snake2 (or ELU: Epi::kAct) -> 16-bit -> rows [64 cw, 64 cw + 64) of the A2 tile (K-major,
        // 128B-swizzled atoms)
        constexpr int ACT = Epi::kAct;
        const int fr = 64 * cw + 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = 8 * j + fc;
          const float b0 = pre.bias7 ? __ldg(pre.bias7 + col) : 0.f, b1 = pre.bias7 ? __ldg(pre.bias7 + col + 1) : 0.f;
          const float a0 = ACT == kActSnake ? __ldg(pre.sn2_a + col) : 0.f;
          const float a1 = ACT == kActSnake ? __ldg(pre.sn2_a + col + 1) : 0.f;
          const float i0 = ACT == kActSnake ? __ldg(pre.sn2_ib + col) : 0.f;
          const float i1 = ACT == kActSnake ? __ldg(pre.sn2_ib + col + 1) : 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = fr + 8 * h;
            const uint32_t v = Op16<BF16>::pack(act_fast<ACT>(acc[4 * j + 2 * h] + b0, a0, i0),
                                                act_fast<ACT>(acc[4 * j + 2 * h + 1] + b1, a1, i1));
            const int chunk = (col & 63) >> 3;
            *reinterpret_cast<uint32_t*>(shared + (col >> 6) * (kBlockM * 128) + r * 128 + ((chunk ^ (r & 7)) << 4) +
                                         (col & 7) * 2) = v;
          }
        }
        fence_proxy_async_smem();   // generic-proxy stores -> visible to the tensor core's reads
        named_bar_sync(1 + cw, 128);
        // 1x1 convolution: K = BN channels, A2 rows of this warpgroup, weights through the ring
        int prev = -1;
        const uint32_t a2 = smem_u32(shared) + cw * 64 * 128;
        for (int kb = 0; kb < BN / kBlockK; ++kb) {
          mma_stage(a2 + kb * kBlockM * 128, kb == 0);
          retire(prev);
        }
        wgmma_wait<0>(acc);
        if (tid == 0) mbar_arrive(&empty_b[prev]);
        named_bar_sync(3, 256);   // both warpgroups' second chains have read A2: the region becomes the staging
      }
      float* epi_st = Epi::kStageBytes > 0
                          ? reinterpret_cast<float*>(epi_smem + (warp - 4) * Epi::kStageBytes)
                          : nullptr;
      gemm_tile_epilogue<Epi, BN>(acc, reinterpret_cast<float*>(shared + cw * Cfg::kAccStage), epi_st, ep, s.L, s.N,
                                  m0, 0, batch, cw, warp, lane);
    }
  }
}

template <class Epi, int BN, bool BF16, bool FUSE>
int launch_conv_halo(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap* tmB1, const HaloShape& s,
                     const ResUnitPre& pre, const typename Epi::Params& ep, cudaStream_t stream) {
  using Cfg = HaloCfg<BN, Epi::kCols, Epi::kStageBytes, FUSE>;
  SATB_REQUIRE(s.K % kBlockK == 0 && s.n_taps % 2 == 1 && (s.n_taps - 1) * s.dil <= kHaloMax && s.N <= BN,
               "halo convolution: unsupported shape");
  if constexpr (FUSE) {
    SATB_REQUIRE(tmB1 != nullptr && s.N == BN && s.K == BN && (Epi::kAct == kActElu || (pre.sn2_a && pre.sn2_ib)),
                 "fused ResidualUnit: needs the 1x1 weights, channels = tile width, and snake2");
  }
  auto kern = conv_halo_wgmma_kernel<Epi, BN, BF16, FUSE>;
  static PerDeviceOnce attr;
  if (attr.first()) SATB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  const int total = ceil_div(s.L, kBlockM) * s.batches;
  if (total <= 0) return 0;
  int grid = device_sm_count();
  if (grid > total) grid = total;
  SATB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, tmA, tmB, tmB1 ? *tmB1 : tmB,
                             s, pre, ep));
  count_launch();
  return 0;
}

}  // namespace satb
