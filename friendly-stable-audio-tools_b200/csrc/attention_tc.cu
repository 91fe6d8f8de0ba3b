// Tensor-core attention forward, head dim D in {32, 64, 96, 128}, no mask, non-causal, optional GQA:
//   O = softmax(Q K^T / sqrt(D)) V      (reference models/transformer.py:496-536)
//
// Head dim 64 (every shipped model) runs attn_wgmma_kernel, described at the kernel below.  The other head dims run
// attn_kernel<D>: one CTA of four warps per 64 query rows of one (batch item, head), the mma.sync flash-attention core
// of mma_tile.cuh (mma_attention) with the 1 / sqrt(D) scale in log2 units; head h reads kv head h / group.
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.h"
#include "mma_tile.cuh"
#include "ptx.cuh"
#include <cmath>
#include <type_traits>

namespace satb {

namespace {

struct AttnArgs {
  const uint16_t *q, *k, *v;
  uint16_t* o;
  int64_t ldq, ldk, ldv, ldo, q_bs, k_bs, v_bs, o_bs;
  int q_col, k_col, v_col;   // column offsets (elements) of head 0 inside the q / k / v tensors
  int Nq, Nk, group;
  float scale_log2;
};

template <int D, bool BF16>
__global__ void __launch_bounds__(kMmaAttnThreads) attn_kernel(const AttnArgs p) {
  extern __shared__ __align__(128) uint16_t smem_attn[];
  // the item's rows and the head's columns come from the arguments alone: worked out while the previous kernel drains
  const int h = blockIdx.y, b = blockIdx.z;
  const int hk = h / p.group;
  const uint16_t *q = p.q + b * p.q_bs, *k = p.k + b * p.k_bs, *v = p.v + b * p.v_bs;
  const int qc = p.q_col + h * D, kc = p.k_col + hk * D, vc = p.v_col + hk * D;
  pdl_launch_dependents();
  pdl_wait();   // q / k / v are written by the previous kernels
  mma_attention<D, BF16>(smem_attn, q, p.ldq, qc, k, p.ldk, kc, v, p.ldv, vc, p.o + b * p.o_bs, p.ldo, h * D,
                         blockIdx.x * 64, p.Nq, p.Nk, ScaleScore{p.scale_log2});
}

// ------------------------------------------------------------------------------------------------ head dim 64, wgmma
// One CTA of three warpgroups per 128 query rows of one (batch item, head), FA3-shaped:
//   warpgroup 0      producer: one thread loads Q once and streams 128-key K / V tiles by TMA into a ring of
//                    kWgStages stages (full / empty mbarriers).  The tensor maps are 3-D (columns, rows of the item,
//                    item), so rows past Nq / Nk of an item arrive zero-filled; the head is a column coordinate.
//   warpgroups 1, 2  consumers, 64 query rows each.  Per key tile: S = Q K^T by wgmma from shared memory (64 x 128,
//                    fp32 in registers), online softmax (exp2), P packed to 16-bit A fragments in registers, then
//                    O += P V by wgmma with A from registers and V read MN-major (transposed) from shared memory.
// The two consumers ping-pong on the tensor cores through named barriers kBarTurn + cw: a consumer waits for its turn,
// issues S_j = Q K_j^T together with O += P_{j-1} V_{j-1}, and passes the turn on; its softmax of S_j then runs while the
// other consumer's MMAs do.  Consumer 0 goes first (consumer 1 arrives once at the start), every consumer takes
// n_tiles + 1 turns (the last one only O += P V of the last tile), and consumer 1 skips the hand-over after its last
// turn, so that each barrier sees exactly as many arrivals as waits.
// A consumer whose 64 rows all lie past Nq (the second one of a CTA with at most 64 valid rows) issues no MMAs and does
// no softmax, but takes every turn and arrives on every empty barrier like an active one: both the named-barrier and
// the mbarrier counts are the same for every Nq and Nk by construction.
// The last key tile is issued at the smallest width w = 16 .. 128 (a multiple of 16) that covers the remaining keys:
// S_j and the exponentials cover w columns, O += P V takes w / 16 k-steps.
constexpr int kWgQ = 128;                    // query rows per CTA
constexpr int kWgK = 128;                    // keys per tile
constexpr int kWgStages = 4;                 // K / V ring depth
constexpr int kWgThreads = 384;
constexpr int kWgTile = 128 * 64 * 2;        // 128 rows x 64 columns, 16-bit, 128B-swizzled: 16 KB
constexpr int kWgSmem = 1024 /*align slack*/ + kWgTile * (1 + 2 * kWgStages) + 256 /*barriers*/;
constexpr int kBarTurn = 1;                  // named barriers 1, 2: "consumer 0 / 1 may issue its MMAs"

struct AttnWgArgs {
  uint16_t* o;
  int64_t ldo, o_bs;
  int q_col, k_col, v_col;   // column offsets (elements) of head 0 inside the q / k / v tensors
  int Nq, Nk, group;
  float scale_log2;
};

// S (64 x W) = Q K^T over the 4 k16-steps of the head dim; K-major operands in 128B-swizzled tiles
template <int W, bool BF16>
__device__ __forceinline__ void issue_qk(float (&s)[64], uint32_t q_addr, uint32_t k_addr) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_ss<W, BF16>(*reinterpret_cast<float(*)[W / 2]>(&s[0]), make_desc_kmajor_sw128(q_addr + 32 * k),
                      make_desc_kmajor_sw128(k_addr + 32 * k), k != 0 ? 1u : 0u);
}

// Online softmax on the S fragment of one key tile (scaled log2 units): s becomes the unnormalised P, m the new row
// maximum, l the rescaled row sum (this thread's columns only, reduced at the end), alpha the factor for O.  LAST: the
// tile holds w columns (a multiple of 16) of which those at keys >= Nk are masked; the 8-column groups >= w are skipped.
template <bool LAST>
__device__ __forceinline__ void softmax_tile(float (&s)[64], float (&m)[2], float (&l)[2], float (&alpha)[2], float scale,
                                             int w, int key0, int Nk) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    if (LAST && 8 * g >= w) break;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (LAST && key0 + 8 * g + (e & 1) >= Nk) s[4 * g + e] = -INFINITY;
      mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * g + e]);
    }
  }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
    const float mn = fmaxf(m[i], mx[i] * scale);   // every row has a valid key in every tile: mx is finite
    alpha[i] = exp2f(m[i] - mn);
    m[i] = mn;
  }
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    if (LAST && 8 * g >= w) break;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      s[4 * g + e] = exp2f(fmaf(s[4 * g + e], scale, -m[e >> 1]));
      sum[e >> 1] += s[4 * g + e];
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) l[i] = fmaf(l[i], alpha[i], sum[i]);
}

template <bool BF16>
__global__ void __launch_bounds__(kWgThreads, 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmq, const __grid_constant__ CUtensorMap tmk,
                  const __grid_constant__ CUtensorMap tmv, const AttnWgArgs p) {
  extern __shared__ uint8_t smem_wg[];
  uint8_t* sQ = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_wg) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = sQ + kWgTile;                   // [kWgStages][128 keys x 64]
  uint8_t* sV = sK + kWgStages * kWgTile;       // [kWgStages][128 keys x 64]
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(sV + kWgStages * kWgTile);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kWgStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // broadcast from lane 0 so that the compiler knows the warpgroup index is warp-uniform: wgmma under a branch it
  // cannot prove uniform gets serialized
  const int wg = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);
  const int q0 = blockIdx.x * kWgQ, h = blockIdx.y, b = blockIdx.z;
  const int n_tiles = (p.Nk + kWgK - 1) / kWgK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmq);
    tma_prefetch_desc(&tmk);
    tma_prefetch_desc(&tmv);
    mbar_init(q_bar, 1);
    for (int i = 0; i < kWgStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrival per consumer warpgroup, active or not
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      pdl_wait();   // q / k / v are written by the previous kernels
      const int hk = h / p.group;
      mbar_expect_tx(q_bar, kWgTile);
      tma_load_4d(sQ, &tmq, q_bar, p.q_col + h * 64, 0, q0, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % kWgStages;
        mbar_wait(&empty_bar[st], ((j / kWgStages) & 1) ^ 1);
        mbar_expect_tx(&full_bar[st], 2 * kWgTile);   // out-of-range rows are zero-filled and counted
        tma_load_4d(sK + st * kWgTile, &tmk, &full_bar[st], p.k_col + hk * 64, 0, j * kWgK, b);
        tma_load_4d(sV + st * kWgTile, &tmv, &full_bar[st], p.v_col + hk * 64, 0, j * kWgK, b);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    pdl_wait();
    const int cw = wg - 1;                        // query rows [q0 + 64 cw, q0 + 64 cw + 64)
    const bool active = q0 + 64 * cw < p.Nq;      // warpgroup-uniform
    const uint32_t q_addr = smem_u32(sQ) + cw * 64 * 128;
    const int rem = p.Nk - (n_tiles - 1) * kWgK;  // keys in the last tile, 1 .. 128
    const int w_last = (rem + 15) & ~15;
    const int key_lane = 2 * (lane & 3);

    if (!active) {
      // the same turns and releases as an active consumer, nothing else (only consumer 1 can be inactive: a CTA has
      // q0 < Nq)
      if (cw == 1) named_bar_arrive(kBarTurn, 256);
      for (int j = 0; j <= n_tiles; ++j) {
        named_bar_sync(kBarTurn + cw, 256);
        if (cw == 0 || j < n_tiles) named_bar_arrive(kBarTurn + (cw ^ 1), 256);
        if (j > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(j - 1) % kWgStages]);
      }
      return;
    }

    float s[64], o[32];
    uint32_t pf[8][4];   // P of the previous tile: A fragments of its 8 k16-steps
    float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f}, alpha[2];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;

    auto issue_pv = [&](int j, int w) {   // O += P_j V_j over the first w keys of tile j
      const uint32_t v_addr = smem_u32(sV + (j % kWgStages) * kWgTile);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        if (16 * kk < w) wgmma_rs_tb<64, BF16>(o, pf[kk], make_desc_mnmajor_sw128(v_addr + 2048 * kk), 1u);
    };
    auto retire_pv = [&](int j) {   // wait for O += P_j V_j; P and K / V of tile j are free again
      wgmma_wait<0>(o);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_fence_regs(pf[kk]);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[j % kWgStages]);
    };
    auto rescale_and_pack = [&](int w) {   // P of the first w columns (the others are not read)
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        o[4 * g] *= alpha[0];
        o[4 * g + 1] *= alpha[0];
        o[4 * g + 2] *= alpha[1];
        o[4 * g + 3] *= alpha[1];
      }
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if (16 * kk >= w) break;
        pf[kk][0] = Op16<BF16>::pack(s[8 * kk], s[8 * kk + 1]);
        pf[kk][1] = Op16<BF16>::pack(s[8 * kk + 2], s[8 * kk + 3]);
        pf[kk][2] = Op16<BF16>::pack(s[8 * kk + 4], s[8 * kk + 5]);
        pf[kk][3] = Op16<BF16>::pack(s[8 * kk + 6], s[8 * kk + 7]);
      }
    };
    // Turn j of a full tile (j < n_tiles - 1): S_j, with O += P_{j-1} V_{j-1} (a full tile too) when PREV (j > 0).
    auto full_turn = [&](int j, auto prevc) {
      constexpr bool PREV = decltype(prevc)::value;
      mbar_wait(&full_bar[j % kWgStages], (j / kWgStages) & 1);
      named_bar_sync(kBarTurn + cw, 256);
      wgmma_fence();
      issue_qk<kWgK, BF16>(s, q_addr, smem_u32(sK + (j % kWgStages) * kWgTile));
      wgmma_commit();
      if constexpr (PREV) {
        issue_pv(j - 1, kWgK);
        wgmma_commit();
      }
      named_bar_arrive(kBarTurn + (cw ^ 1), 256);
      if constexpr (PREV) wgmma_wait<1>(s);
      else wgmma_wait<0>(s);
      softmax_tile<false>(s, m, l, alpha, p.scale_log2, kWgK, j * kWgK + key_lane, p.Nk);
      if constexpr (PREV) retire_pv(j - 1);
      rescale_and_pack(kWgK);
    };
    // Turns n_tiles - 1 and n_tiles: S of the last tile at its width W, with O += P V of the tile before it if there
    // is one (PREV), then O += P V of the last tile over W / 16 k-steps.
    // W and PREV (here and in full_turn) are compile-time constants, so that no merge of differently-issued
    // accumulators falls between a wgmma and its wait: ptxas would serialize every wgmma of the kernel.
    auto last_turns = [&](auto wc, auto prevc) {
      constexpr int W = decltype(wc)::value;
      constexpr bool PREV = decltype(prevc)::value;
      const int j = n_tiles - 1;
      mbar_wait(&full_bar[j % kWgStages], (j / kWgStages) & 1);
      named_bar_sync(kBarTurn + cw, 256);
      wgmma_fence();
      issue_qk<W, BF16>(s, q_addr, smem_u32(sK + (j % kWgStages) * kWgTile));
      wgmma_commit();
      if constexpr (PREV) {
        issue_pv(j - 1, kWgK);
        wgmma_commit();
      }
      named_bar_arrive(kBarTurn + (cw ^ 1), 256);
      if constexpr (PREV) wgmma_wait<1>(s);
      else wgmma_wait<0>(s);
      softmax_tile<true>(s, m, l, alpha, p.scale_log2, W, j * kWgK + key_lane, p.Nk);
      if constexpr (PREV) retire_pv(j - 1);
      rescale_and_pack(W);
      named_bar_sync(kBarTurn + cw, 256);
      wgmma_fence();
      issue_pv(j, W);
      wgmma_commit();
      if (cw == 0) named_bar_arrive(kBarTurn + 1, 256);   // consumer 1 hands over no further turn
      retire_pv(j);
    };
    auto last_turns_w = [&](auto prevc) {
      switch (w_last) {
        case 16: last_turns(std::integral_constant<int, 16>{}, prevc); break;
        case 32: last_turns(std::integral_constant<int, 32>{}, prevc); break;
        case 48: last_turns(std::integral_constant<int, 48>{}, prevc); break;
        case 64: last_turns(std::integral_constant<int, 64>{}, prevc); break;
        case 80: last_turns(std::integral_constant<int, 80>{}, prevc); break;
        case 96: last_turns(std::integral_constant<int, 96>{}, prevc); break;
        case 112: last_turns(std::integral_constant<int, 112>{}, prevc); break;
        default: last_turns(std::integral_constant<int, 128>{}, prevc); break;
      }
    };

    mbar_wait(q_bar, 0);
    if (cw == 1) named_bar_arrive(kBarTurn, 256);   // consumer 0 takes the first turn
    if (n_tiles == 1) {
      last_turns_w(std::false_type{});
    } else {
      full_turn(0, std::false_type{});
      for (int j = 1; j < n_tiles - 1; ++j) full_turn(j, std::true_type{});
      last_turns_w(std::true_type{});
    }

    // normalise; stage the warp's 16 rows in its own rows of this consumer's (no longer read) Q tile, then 16-byte
    // stores of the rows < Nq
    float inv[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
      inv[i] = 1.f / l[i];
    }
    uint16_t* so = reinterpret_cast<uint16_t*>(sQ + cw * 64 * 128);
    const int wq = warp & 3;
    const int rr = 16 * wq + (lane >> 2);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      *reinterpret_cast<uint32_t*>(so + swz<64>(rr, g) + key_lane) = Op16<BF16>::pack(o[4 * g] * inv[0], o[4 * g + 1] * inv[0]);
      *reinterpret_cast<uint32_t*>(so + swz<64>(rr + 8, g) + key_lane) =
          Op16<BF16>::pack(o[4 * g + 2] * inv[1], o[4 * g + 3] * inv[1]);
    }
    __syncwarp();
    uint16_t* ob = p.o + b * p.o_bs + h * 64;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = lane + 32 * i;
      const int r = 16 * wq + (idx >> 3), c = idx & 7;
      const int row = q0 + 64 * cw + r;
      if (row < p.Nq)
        *reinterpret_cast<uint4*>(ob + static_cast<int64_t>(row) * p.ldo + c * 8) =
            *reinterpret_cast<const uint4*>(so + swz<64>(r, c));
    }
  }
}

}  // namespace

// q / k / v are 16-bit row-major buffers [batch, rows, cols] with row strides ld* and batch strides
// *_bs (elements); head h of q lives at columns q_col + h*head_dim (k, v likewise with the kv head).
// For the fused QKV buffer pass the same pointer three times with different column offsets.
int launch_attention_tc(const void* q, const void* k, const void* v, void* o, int64_t ldq, int64_t ldk, int64_t ldv,
                        int64_t ldo, int64_t q_bs, int64_t k_bs, int64_t v_bs, int64_t o_bs, int q_cols, int k_cols,
                        int v_cols, int q_col, int k_col, int v_col, int batch, int H, int H_kv, int Nq, int Nk,
                        int head_dim, bool bf16, cudaStream_t stream, const CUtensorMap* tmq, const CUtensorMap* tmk,
                        const CUtensorMap* tmv) {
  SATB_REQUIRE(head_dim == 32 || head_dim == 64 || head_dim == 96 || head_dim == 128,
               "attention head dim must be 32, 64, 96 or 128");
  SATB_REQUIRE(H >= 1 && H_kv >= 1, "attention needs at least one head");
  SATB_REQUIRE(H % H_kv == 0, "num_heads must be a multiple of kv heads");
  SATB_REQUIRE(Nk >= 1 && Nq >= 1, "empty attention problem");
  SATB_REQUIRE(ldo % 8 == 0 && o_bs % 8 == 0 && (reinterpret_cast<uintptr_t>(o) & 15) == 0,
               "attention output must be 16B aligned");
  SATB_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && q_col % 8 == 0 && k_col % 8 == 0 && v_col % 8 == 0 &&
                   q_bs % 8 == 0 && k_bs % 8 == 0 && v_bs % 8 == 0,
               "attention operand strides / column offsets must be 16B aligned");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(k) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(v) & 15) == 0,
               "attention operands must be 16B aligned");
  const int64_t dh = head_dim;
  SATB_REQUIRE(q_col + H * dh <= q_cols && k_col + H_kv * dh <= k_cols && v_col + H_kv * dh <= v_cols,
               "attention heads exceed the operand columns");
  AttnArgs a;
  a.q = static_cast<const uint16_t*>(q); a.k = static_cast<const uint16_t*>(k); a.v = static_cast<const uint16_t*>(v);
  a.o = static_cast<uint16_t*>(o);
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo;
  a.q_bs = q_bs; a.k_bs = k_bs; a.v_bs = v_bs; a.o_bs = o_bs;
  a.q_col = q_col; a.k_col = k_col; a.v_col = v_col;
  a.Nq = Nq; a.Nk = Nk; a.group = H / H_kv;
  a.scale_log2 = (1.0f / sqrtf(static_cast<float>(head_dim))) * 1.4426950408889634f;
  if (head_dim == 64) {
    CUtensorMap mq, mk, mv;
    if (!tmq) SATB_PROPAGATE(make_tmap_a(&mq, q, q_cols, Nq, batch, ldq, q_bs));
    if (!tmk) SATB_PROPAGATE(make_tmap_a(&mk, k, k_cols, Nk, batch, ldk, k_bs));
    if (!tmv) SATB_PROPAGATE(make_tmap_a(&mv, v, v_cols, Nk, batch, ldv, v_bs));
    AttnWgArgs w;
    w.o = a.o; w.ldo = ldo; w.o_bs = o_bs;
    w.q_col = q_col; w.k_col = k_col; w.v_col = v_col;
    w.Nq = Nq; w.Nk = Nk; w.group = a.group;
    w.scale_log2 = a.scale_log2;
    const dim3 grid(ceil_div(Nq, kWgQ), H, batch);
    SATB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "attention grid too large");
    auto kern = bf16 ? attn_wgmma_kernel<true> : attn_wgmma_kernel<false>;
    static PerDeviceOnce once_wg[2];
    if (once_wg[bf16 ? 1 : 0].first())
      SATB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem));
    SATB_CHECK_CUDA(launch_pdl(kern, grid, dim3(kWgThreads), kWgSmem, stream, tmq ? *tmq : mq, tmk ? *tmk : mk,
                               tmv ? *tmv : mv, w));
    count_launch();
    SATB_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  const dim3 grid(ceil_div(Nq, 64), H, batch);
  SATB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "attention grid too large");
  switch (head_dim) {
    case 32:
      SATB_PROPAGATE((bf16 ? launch_mma_attention<attn_kernel<32, true>, 32>(grid, stream, a)
                          : launch_mma_attention<attn_kernel<32, false>, 32>(grid, stream, a)));
      break;
    case 96:
      SATB_PROPAGATE((bf16 ? launch_mma_attention<attn_kernel<96, true>, 96>(grid, stream, a)
                          : launch_mma_attention<attn_kernel<96, false>, 96>(grid, stream, a)));
      break;
    default:
      SATB_PROPAGATE((bf16 ? launch_mma_attention<attn_kernel<128, true>, 128>(grid, stream, a)
                          : launch_mma_attention<attn_kernel<128, false>, 128>(grid, stream, a)));
      break;
  }
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace satb
