// FP8 self-attention, head dim 64 (the DiT's attention_dtype "fp8"; DESIGN.md sections 3-5):
//   O = softmax(Q K^T / 8) V  with Q, K, V and the probabilities P as e4m3 tensor-core operands.
//
// q and k come as e4m3 with one power-of-two scale per (token, head) from the QKV GEMM's e4m3 epilogues (gemm.cuh
// EpiQkvRopeE4m3, EpiHeadNormE4m3); v in 16 bits.  Two launches per block:
//   attn_fp8_vt_kernel     one CTA per (batch item, head): v -> e4m3 with one power-of-two scale per (item, head,
//                          channel), taken over the item's N tokens, stored transposed (V^T, keys contiguous)
//                          because FP8 wgmma takes B K-major only.  Within each 32-key group the keys are stored in the order of the S accumulator's
//                          column ownership (fp8_key_of below), so that P goes from the S registers into the e4m3 A
//                          fragment of O += P V without shuffles.  Keys past N are zero.
//   attn_wgmma_fp8_kernel  the structure of attn_wgmma_kernel (attention_tc.cu): a producer warpgroup with a TMA ring
//                          for K, V^T and the key scales, two consumer warpgroups of 64 query rows that take turns on
//                          the tensor cores.  S = Q K^T by wgmma m64nWk32 e4m3 (64-byte rows, 64B swizzle), the key
//                          scales multiply S's columns, the row's q scale folds into its softmax scale; P = e4m3 of
//                          exp2(s - m) against the running maximum m, in [0, 1], no scale; O += P V^T by wgmma with A
//                          from registers; the channel scales multiply O's columns in the epilogue.  The row sum l
//                          adds the fp32 P (before its e4m3 rounding).
#include "common.cuh"
#include "fp8.cuh"
#include "kernels.h"
#include "ptx.cuh"
#include <type_traits>

namespace satb {

namespace {

constexpr int kF8Q = 128;                    // query rows per CTA
constexpr int kF8K = 128;                    // keys per tile
constexpr int kF8Stages = 4;                 // K / V^T / key-scale ring depth
constexpr int kF8Threads = 384;
constexpr int kF8QTile = 128 * 64;           // 128 query rows x 64 e4m3, 64B-swizzled: 8 KB
constexpr int kF8KTile = 128 * 64;           // 128 keys x 64 e4m3, 64B-swizzled: 8 KB
constexpr int kF8VTile = 64 * 128;           // 64 channels x 128 keys e4m3, 128B-swizzled: 8 KB
constexpr int kF8OTile = 128 * 64 * 2;       // output staging, 128 rows x 64 16-bit: 16 KB
constexpr int kF8STile = 128 * 4;            // 128 key scales
constexpr int kF8Smem = 1024 /*align slack*/ + kF8QTile + kF8Stages * (kF8KTile + kF8VTile) + kF8OTile +
                        kF8Stages * kF8STile + 256 /*barriers*/;
constexpr int kBarTurn = 1;                  // named barriers 1, 2: "consumer 0 / 1 may issue its MMAs"
constexpr int kQuantThreads = 256;
constexpr int kVtPitch = 65;                 // staged v tile row pitch (16-bit elements): odd, to spread banks

// Key stored at position j (0 .. 31) of a 32-key group.  The e4m3 A fragment of thread t holds k indices
// 4 (t % 4) + {0..3} (and + 16); the S accumulator gives it columns 2 (t % 4) + {0, 1} of each 8-column group.  So k
// index j = 16 hi + 4 q + i holds key 16 hi + 8 (i / 2) + 2 q + i % 2.
__host__ __device__ __forceinline__ int fp8_key_of(int j) {
  return 16 * (j >> 4) + 8 * ((j & 3) >> 1) + 2 * ((j >> 2) & 3) + (j & 1);
}

template <bool BF16>
__device__ __forceinline__ float bits16_to_float(uint32_t u) {
  if constexpr (BF16) return __uint_as_float(u << 16);
  else return __half2float(__ushort_as_half(static_cast<unsigned short>(u)));
}

template <bool BF16>
__device__ __forceinline__ void unpack8(const uint4& raw, float (&x)[8]) {
  const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[2 * i] = bits16_to_float<BF16>(w[i] & 0xFFFFu);
    x[2 * i + 1] = bits16_to_float<BF16>(w[i] >> 16);
  }
}

template <bool BF16>
__global__ void __launch_bounds__(kQuantThreads) attn_fp8_vt_kernel(const uint16_t* __restrict__ v, int64_t ld,
                                                                    int64_t bs, const AttnFp8Bufs o, int H, int N) {
  __shared__ float red[32][65];                  // partial channel maxima of v, one row per 8-lane row slot
  __shared__ float vinv[64];                     // 2^-e of each channel
  __shared__ uint16_t vt[kF8K * kVtPitch];       // one 128-key tile of v, [key][channel]
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int bh = b * H + h, Np = attn_fp8_pad(N);
  pdl_launch_dependents();
  pdl_wait();   // v is written by the QKV GEMM

  // v channel maxima over the item's N tokens: thread = (8 channels, row slot r0 of 32)
  {
    const int c8 = tid & 7, r0 = tid >> 3;
    float am[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int r = r0; r < N; r += 32) {
      float x[8];
      unpack8<BF16>(*reinterpret_cast<const uint4*>(v + b * bs + r * ld + h * 64 + c8 * 8), x);
#pragma unroll
      for (int i = 0; i < 8; ++i) am[i] = fmaxf(am[i], fabsf(x[i]));
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) red[r0][c8 * 8 + i] = am[i];
  }
  __syncthreads();
  if (tid < 64) {
    float a = 0.f;
    for (int j = 0; j < 32; ++j) a = fmaxf(a, red[j][tid]);
    const int e = fp8_row_exp(a);
    vinv[tid] = pow2f(-e);
    o.sv[static_cast<int64_t>(bh) * 64 + tid] = pow2f(e);
  }
  __syncthreads();

  // V^T, one 128-key tile at a time: stage [key][channel] (zeros past N), then 16 stored keys per thread and chunk
  uint8_t* vt_out = o.vt8 + static_cast<int64_t>(bh) * 64 * Np;
  for (int t0 = 0; t0 < Np; t0 += kF8K) {
    for (int idx = tid; idx < kF8K * 8; idx += kQuantThreads) {
      const int kr = idx >> 3, c8 = idx & 7, key = t0 + kr;
      const uint4 raw = key < N ? *reinterpret_cast<const uint4*>(v + b * bs + key * ld + h * 64 + c8 * 8)
                                : make_uint4(0, 0, 0, 0);
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        vt[kr * kVtPitch + c8 * 8 + 2 * i] = static_cast<uint16_t>(w[i] & 0xFFFFu);
        vt[kr * kVtPitch + c8 * 8 + 2 * i + 1] = static_cast<uint16_t>(w[i] >> 16);
      }
    }
    __syncthreads();
    for (int idx = tid; idx < 64 * 8; idx += kQuantThreads) {
      const int c = idx >> 3, k16 = idx & 7;
      const float inv = vinv[c];
      uint32_t w[4];
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4) {
        float x[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int pos = 16 * k16 + 4 * j4 + i;   // stored position in the tile
          const int key = (pos & ~31) + fp8_key_of(pos & 31);
          x[i] = bits16_to_float<BF16>(vt[key * kVtPitch + c]) * inv;
        }
        w[j4] = e4m3x4(x[0], x[1], x[2], x[3]);
      }
      *reinterpret_cast<uint4*>(vt_out + static_cast<int64_t>(c) * Np + t0 + 16 * k16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    __syncthreads();
  }
}

struct AttnF8Args {
  const float* sq;   // [B * H, pad(Nq)]
  const float* sv;   // [B * H, 64]
  uint16_t* o;
  int64_t ldo, o_bs;
  int H, Nq, Nk;
  float scale_log2;
};

// S (64 x W) = Q K^T over the 2 k32-steps of the head dim; K-major e4m3 operands in 64B-swizzled tiles
template <int W>
__device__ __forceinline__ void issue_qk8(float (&s)[64], uint32_t q_addr, uint32_t k_addr) {
#pragma unroll
  for (int k = 0; k < 2; ++k)
    wgmma_ss_e4m3<W>(*reinterpret_cast<float(*)[W / 2]>(&s[0]), make_desc_kmajor_sw64(q_addr + 32 * k),
                     make_desc_kmajor_sw64(k_addr + 32 * k), k != 0 ? 1u : 0u);
}

// Online softmax on the S fragment of one key tile: s (q8 . k8) times the key scales ks, in log2 units with the row
// scales rs (1/8 log2(e) times the row's q scale); s becomes the unnormalised fp32 P, m the new row maximum, l the
// rescaled row sum of the fp32 P (this thread's columns only, reduced at the end), alpha the factor for O.  LAST: the
// tile holds w columns (a multiple of 32) of which those at keys >= Nk are masked; the 8-column groups >= w are skipped.
template <bool LAST>
__device__ __forceinline__ void softmax_tile8(float (&s)[64], float (&m)[2], float (&l)[2], float (&alpha)[2],
                                              const float (&rs)[2], uint32_t ks, int w, int key0, int Nk) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    if (LAST && 8 * g >= w) break;
    float kx, ky;   // volatile: loaded where used (hoisted, the 32 loads would starve the pending wgmma's registers)
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(kx), "=f"(ky) : "r"(ks + 32 * g));
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      s[4 * g + e] *= (e & 1) ? ky : kx;
      if (LAST && key0 + 8 * g + (e & 1) >= Nk) s[4 * g + e] = -INFINITY;
      mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * g + e]);
    }
  }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
    const float mn = fmaxf(m[i], mx[i] * rs[i]);   // every row has a valid key in every tile: mx is finite
    alpha[i] = exp2f(m[i] - mn);
    m[i] = mn;
  }
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    if (LAST && 8 * g >= w) break;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      s[4 * g + e] = exp2f(fmaf(s[4 * g + e], rs[e >> 1], -m[e >> 1]));
      sum[e >> 1] += s[4 * g + e];
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) l[i] = fmaf(l[i], alpha[i], sum[i]);
}

// The turn protocol, barrier counts and inactive-consumer handling are those of attn_wgmma_kernel (attention_tc.cu);
// only the operand types, the scales and the 32-key granularity of the last tile differ.
template <bool BF16>
__global__ void __launch_bounds__(kF8Threads, 1)
attn_wgmma_fp8_kernel(const __grid_constant__ CUtensorMap tmq, const __grid_constant__ CUtensorMap tmk,
                      const __grid_constant__ CUtensorMap tmv, const __grid_constant__ CUtensorMap tms,
                      const AttnF8Args p) {
  extern __shared__ uint8_t smem_f8[];
  uint8_t* sQ = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_f8) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = sQ + kF8QTile;                     // [kF8Stages][128 keys x 64]
  uint8_t* sV = sK + kF8Stages * kF8KTile;         // [kF8Stages][64 channels x 128 keys]
  uint8_t* sO = sV + kF8Stages * kF8VTile;         // [128 rows x 64] 16-bit output staging
  float* sS = reinterpret_cast<float*>(sO + kF8OTile);   // [kF8Stages][128] key scales
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(sS + kF8Stages * 128);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kF8Stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);
  const int q0 = blockIdx.x * kF8Q, h = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.H + h;
  const int n_tiles = (p.Nk + kF8K - 1) / kF8K;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmq);
    tma_prefetch_desc(&tmk);
    tma_prefetch_desc(&tmv);
    tma_prefetch_desc(&tms);
    mbar_init(q_bar, 1);
    for (int i = 0; i < kF8Stages; ++i) {
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
      pdl_wait();   // the operands are written by the quantiser
      mbar_expect_tx(q_bar, kF8QTile);
      tma_load_3d(sQ, &tmq, q_bar, h * 64, q0, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % kF8Stages;
        mbar_wait(&empty_bar[st], ((j / kF8Stages) & 1) ^ 1);
        mbar_expect_tx(&full_bar[st], kF8KTile + kF8VTile + kF8STile);   // out-of-range boxes are zero-filled and counted
        tma_load_3d(sK + st * kF8KTile, &tmk, &full_bar[st], h * 64, j * kF8K, b);
        tma_load_3d(sV + st * kF8VTile, &tmv, &full_bar[st], j * kF8K, 0, bh);
        tma_load_2d(sS + st * 128, &tms, &full_bar[st], j * kF8K, bh);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    pdl_wait();
    const int cw = wg - 1;                        // query rows [q0 + 64 cw, q0 + 64 cw + 64)
    const bool active = q0 + 64 * cw < p.Nq;      // warpgroup-uniform
    const uint32_t q_addr = smem_u32(sQ) + cw * 64 * 64;
    const int rem = p.Nk - (n_tiles - 1) * kF8K;  // keys in the last tile, 1 .. 128
    const int w_last = (rem + 31) & ~31;
    const int key_lane = 2 * (lane & 3);
    const int wq = warp & 3;

    if (!active) {
      if (cw == 1) named_bar_arrive(kBarTurn, 256);
      for (int j = 0; j <= n_tiles; ++j) {
        named_bar_sync(kBarTurn + cw, 256);
        if (cw == 0 || j < n_tiles) named_bar_arrive(kBarTurn + (cw ^ 1), 256);
        if (j > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(j - 1) % kF8Stages]);
      }
      return;
    }

    const int Npq = attn_fp8_pad(p.Nq);
    float rs[2];   // the rows' softmax scales in log2 units
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = q0 + 64 * cw + 16 * wq + (lane >> 2) + 8 * i;
      // rows past Nq (never stored) keep a finite positive scale, so that their masked columns stay -inf, not NaN
      rs[i] = p.scale_log2 * (row < p.Nq ? __ldg(p.sq + static_cast<int64_t>(bh) * Npq + row) : 1.f);
    }
    float s[64], o[32];
    uint32_t pf[4][4];   // P of the previous tile: e4m3 A fragments of its 4 k32-steps
    float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f}, alpha[2];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;

    auto issue_pv = [&](int j, int w) {   // O += P_j V_j over the first w keys of tile j
      const uint32_t v_addr = smem_u32(sV + (j % kF8Stages) * kF8VTile);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        if (32 * kk < w) wgmma_rs_e4m3_n64(o, pf[kk], make_desc_kmajor_sw128(v_addr + 32 * kk), 1u);
    };
    auto retire_pv = [&](int j) {   // wait for O += P_j V_j; P and the stage of tile j are free again
      wgmma_wait<0>(o);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_fence_regs(pf[kk]);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[j % kF8Stages]);
    };
    auto rescale_and_pack = [&](int w) {   // P of the first w columns, in the stored key order of fp8_key_of
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        o[4 * g] *= alpha[0];
        o[4 * g + 1] *= alpha[0];
        o[4 * g + 2] *= alpha[1];
        o[4 * g + 3] *= alpha[1];
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if (32 * kk >= w) break;
        const float* t = s + 16 * kk;   // column groups 4 kk .. 4 kk + 3
        pf[kk][0] = e4m3x4(t[0], t[1], t[4], t[5]);
        pf[kk][1] = e4m3x4(t[2], t[3], t[6], t[7]);
        pf[kk][2] = e4m3x4(t[8], t[9], t[12], t[13]);
        pf[kk][3] = e4m3x4(t[10], t[11], t[14], t[15]);
      }
    };
    auto key_scales = [&](int j) { return smem_u32(sS + (j % kF8Stages) * 128 + key_lane); };
    auto full_turn = [&](int j, auto prevc) {
      constexpr bool PREV = decltype(prevc)::value;
      mbar_wait(&full_bar[j % kF8Stages], (j / kF8Stages) & 1);
      named_bar_sync(kBarTurn + cw, 256);
      wgmma_fence();
      issue_qk8<kF8K>(s, q_addr, smem_u32(sK + (j % kF8Stages) * kF8KTile));
      wgmma_commit();
      if constexpr (PREV) {
        issue_pv(j - 1, kF8K);
        wgmma_commit();
      }
      named_bar_arrive(kBarTurn + (cw ^ 1), 256);
      if constexpr (PREV) wgmma_wait<1>(s);
      else wgmma_wait<0>(s);
      softmax_tile8<false>(s, m, l, alpha, rs, key_scales(j), kF8K, j * kF8K + key_lane, p.Nk);
      if constexpr (PREV) retire_pv(j - 1);
      rescale_and_pack(kF8K);
    };
    auto last_turns = [&](auto wc, auto prevc) {
      constexpr int W = decltype(wc)::value;
      constexpr bool PREV = decltype(prevc)::value;
      const int j = n_tiles - 1;
      mbar_wait(&full_bar[j % kF8Stages], (j / kF8Stages) & 1);
      named_bar_sync(kBarTurn + cw, 256);
      wgmma_fence();
      issue_qk8<W>(s, q_addr, smem_u32(sK + (j % kF8Stages) * kF8KTile));
      wgmma_commit();
      if constexpr (PREV) {
        issue_pv(j - 1, kF8K);
        wgmma_commit();
      }
      named_bar_arrive(kBarTurn + (cw ^ 1), 256);
      if constexpr (PREV) wgmma_wait<1>(s);
      else wgmma_wait<0>(s);
      softmax_tile8<true>(s, m, l, alpha, rs, key_scales(j), W, j * kF8K + key_lane, p.Nk);
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
        case 32: last_turns(std::integral_constant<int, 32>{}, prevc); break;
        case 64: last_turns(std::integral_constant<int, 64>{}, prevc); break;
        case 96: last_turns(std::integral_constant<int, 96>{}, prevc); break;
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

    // normalise, multiply by the channel scales; stage the warp's 16 rows, then 16-byte stores of the rows < Nq
    float inv[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
      inv[i] = 1.f / l[i];
    }
    uint16_t* so = reinterpret_cast<uint16_t*>(sO) + cw * 64 * 64;
    const float* svp = p.sv + static_cast<int64_t>(bh) * 64 + key_lane;
    const int rr = 16 * wq + (lane >> 2);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const float2 c = __ldg(reinterpret_cast<const float2*>(svp + 8 * g));
      const int off0 = rr * 64 + ((g ^ (rr & 7)) << 3) + key_lane;
      const int off1 = (rr + 8) * 64 + ((g ^ ((rr + 8) & 7)) << 3) + key_lane;
      *reinterpret_cast<uint32_t*>(so + off0) = Op16<BF16>::pack(o[4 * g] * inv[0] * c.x, o[4 * g + 1] * inv[0] * c.y);
      *reinterpret_cast<uint32_t*>(so + off1) = Op16<BF16>::pack(o[4 * g + 2] * inv[1] * c.x, o[4 * g + 3] * inv[1] * c.y);
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
            *reinterpret_cast<const uint4*>(so + r * 64 + ((c ^ (r & 7)) << 3));
    }
  }
}

}  // namespace

size_t attn_fp8_workspace_bytes(int B, int H, int Nq, int Nk) {
  const size_t D = static_cast<size_t>(H) * 64, BH = static_cast<size_t>(B) * H;
  const size_t npq = attn_fp8_pad(Nq), npk = attn_fp8_pad(Nk);
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  return al(B * static_cast<size_t>(Nq) * D) + al(B * static_cast<size_t>(Nk) * D) + al(BH * npq * 4) + al(BH * npk * 4) +
         al(BH * 64 * npk) + al(BH * 64 * 4);
}

AttnFp8Bufs attn_fp8_bufs(void* ws, int B, int H, int Nq, int Nk) {
  const size_t D = static_cast<size_t>(H) * 64, BH = static_cast<size_t>(B) * H;
  const size_t npq = attn_fp8_pad(Nq), npk = attn_fp8_pad(Nk);
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  uint8_t* p = static_cast<uint8_t*>(ws);
  AttnFp8Bufs r;
  r.q8 = p; p += al(B * static_cast<size_t>(Nq) * D);
  r.k8 = p; p += al(B * static_cast<size_t>(Nk) * D);
  r.sq = reinterpret_cast<float*>(p); p += al(BH * npq * 4);
  r.sk = reinterpret_cast<float*>(p); p += al(BH * npk * 4);
  r.vt8 = p; p += al(BH * 64 * npk);
  r.sv = reinterpret_cast<float*>(p);
  return r;
}

int launch_attention_fp8_vt(const void* v, int64_t ld, int64_t bs, const AttnFp8Bufs& o, int B, int H, int N, bool bf16,
                            cudaStream_t stream) {
  SATB_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && H <= 65535 && N >= 1,
               "FP8 attention V quantiser: need B, H in 1 .. 65535 and N >= 1");
  SATB_REQUIRE(ld % 8 == 0 && bs % 8 == 0 && ld >= static_cast<int64_t>(H) * 64 && bs >= 0,
               "FP8 attention V quantiser: row pitch and item stride must be multiples of 8 elements, ld >= H * 64");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(v) & 15) == 0 && (reinterpret_cast<uintptr_t>(o.vt8) & 15) == 0,
               "FP8 attention V quantiser: v and vt8 must be 16B aligned");
  auto kern = bf16 ? attn_fp8_vt_kernel<true> : attn_fp8_vt_kernel<false>;
  SATB_CHECK_CUDA(launch_pdl(kern, dim3(H, B), dim3(kQuantThreads), 0, stream, static_cast<const uint16_t*>(v), ld, bs,
                             o, H, N));
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int make_attention_fp8_maps(AttnFp8Maps* m, const AttnFp8Bufs& bufs, int B, int H, int Nq, int Nk) {
  SATB_REQUIRE(B >= 1 && H >= 1 && Nq >= 1 && Nk >= 1, "FP8 attention: empty problem");
  const uint64_t D = static_cast<uint64_t>(H) * 64, npk = attn_fp8_pad(Nk);
  {
    const uint64_t dims[3] = {D, static_cast<uint64_t>(Nq), static_cast<uint64_t>(B)};
    const uint64_t strides[2] = {D, D * Nq};
    const uint32_t box[3] = {64, kF8Q, 1};
    SATB_PROPAGATE(make_tmap_nd(&m->q, bufs.q8, 3, CU_TENSOR_MAP_DATA_TYPE_UINT8, dims, strides, box,
                                CU_TENSOR_MAP_SWIZZLE_64B));
  }
  {
    const uint64_t dims[3] = {D, static_cast<uint64_t>(Nk), static_cast<uint64_t>(B)};
    const uint64_t strides[2] = {D, D * Nk};
    const uint32_t box[3] = {64, kF8K, 1};
    SATB_PROPAGATE(make_tmap_nd(&m->k, bufs.k8, 3, CU_TENSOR_MAP_DATA_TYPE_UINT8, dims, strides, box,
                                CU_TENSOR_MAP_SWIZZLE_64B));
  }
  {
    const uint64_t dims[3] = {npk, 64, static_cast<uint64_t>(B) * H};
    const uint64_t strides[2] = {npk, 64 * npk};
    const uint32_t box[3] = {kF8K, 64, 1};
    SATB_PROPAGATE(make_tmap_nd(&m->vt, bufs.vt8, 3, CU_TENSOR_MAP_DATA_TYPE_UINT8, dims, strides, box,
                                CU_TENSOR_MAP_SWIZZLE_128B));
  }
  {
    const uint64_t dims[2] = {npk, static_cast<uint64_t>(B) * H};
    const uint64_t strides[1] = {npk * 4};
    const uint32_t box[2] = {kF8K, 1};
    SATB_PROPAGATE(make_tmap_nd(&m->sk, bufs.sk, 2, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dims, strides, box,
                                CU_TENSOR_MAP_SWIZZLE_NONE));
  }
  return 0;
}

int launch_attention_fp8(const AttnFp8Maps& maps, const AttnFp8Bufs& bufs, void* o, int64_t ldo, int64_t o_bs, int B,
                         int H, int Nq, int Nk, bool bf16, cudaStream_t stream) {
  SATB_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && H <= 65535 && Nq >= 1 && Nk >= 1, "FP8 attention: bad shape");
  SATB_REQUIRE(ldo % 8 == 0 && o_bs % 8 == 0 && (reinterpret_cast<uintptr_t>(o) & 15) == 0,
               "FP8 attention output must be 16B aligned");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(bufs.sv) & 7) == 0, "FP8 attention channel scales must be 8B aligned");
  AttnF8Args a;
  a.sq = bufs.sq; a.sv = bufs.sv;
  a.o = static_cast<uint16_t*>(o); a.ldo = ldo; a.o_bs = o_bs;
  a.H = H; a.Nq = Nq; a.Nk = Nk;
  a.scale_log2 = 0.125f * 1.4426950408889634f;
  auto kern = bf16 ? attn_wgmma_fp8_kernel<true> : attn_wgmma_fp8_kernel<false>;
  static PerDeviceOnce once[2];
  if (once[bf16 ? 1 : 0].first())
    SATB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kF8Smem));
  SATB_CHECK_CUDA(launch_pdl(kern, dim3(ceil_div(Nq, kF8Q), H, B), dim3(kF8Threads), kF8Smem, stream, maps.q, maps.k,
                             maps.vt, maps.sk, a));
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace satb
