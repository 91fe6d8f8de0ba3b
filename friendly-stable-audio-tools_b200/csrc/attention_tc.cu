// Tensor-core attention forward, head dim D in {32, 64, 96, 128}, no mask, non-causal, optional GQA:
//   O = softmax(Q K^T / sqrt(D)) V      (reference models/transformer.py:496-536)
//
// One CTA of four warps per 64 query rows of one (batch item, head); each warp owns 16 query rows.  Keys are
// processed in tiles of 64, double-buffered in shared memory by cp.async (rows past the end are zero-filled, their
// scores masked).  Per tile and warp: S = Q K^T with mma.sync m16n8k16 (Q fragments stay in registers for the whole
// row block, K fragments by ldmatrix), online softmax in fp32 on the S fragments (exp2, row max / sum reduced over the
// four lanes of a row), then O += P V with P repacked from the S fragments into 16-bit A fragments and V fragments
// by ldmatrix.trans.  The normalised output goes through shared memory so that it leaves as 16-byte row segments.
// The kernel is a template on D: D / 16 k-slices of Q K^T, D / 8 output fragments, 64 x D tiles.
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.h"
#include "ptx.cuh"
#include <cmath>

namespace satb {

namespace {

constexpr int kQ = 64;          // query rows per CTA
constexpr int kK = 64;          // keys per tile
constexpr int kAttnThreads = 128;
template <int D>
constexpr int tile_elems() { return 64 * D; }                    // one 64 x D 16-bit tile: 4, 8, 12 or 16 KB
template <int D>
constexpr int attn_smem() { return (1 + 2 * 2) * tile_elems<D>() * 2; }   // Q, two K and two V buffers: 20 .. 80 KB

struct AttnArgs {
  const uint16_t *q, *k, *v;
  uint16_t* o;
  int64_t ldq, ldk, ldv, ldo, q_bs, k_bs, v_bs, o_bs;
  int q_col, k_col, v_col;   // column offsets (elements) of head 0 inside the q / k / v tensors
  int Nq, Nk, group;
  float scale_log2;
};

// Element offset of 16-byte chunk `c` (0 .. D/8 - 1) of row `r` in a 64 x D tile: chunks are XOR-swizzled with the
// row so that the eight rows an ldmatrix phase reads (same c, rows 8i .. 8i + 7) fall into different banks.  A bank
// line is 8 chunks.  With 8 or 16 chunks per row, c ^ (r & 7) permutes the row's chunks and moves the eight rows to
// eight different chunk columns.  With 4 or 12 chunks per row (D = 32, 96) consecutive rows start half a bank line
// apart, so row parity already picks the half; c ^ ((r >> 1) & 3) stays inside the aligned group of 4 chunks (inside
// the row) and spreads the four rows of equal parity over that half's four chunk columns.
template <int D>
__device__ __forceinline__ int swz(int r, int c) {
  if constexpr ((D / 8) % 8 == 0) return r * D + ((c ^ (r & 7)) << 3);
  else return r * D + ((c ^ ((r >> 1) & 3)) << 3);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// row and chunk of the flat chunk index idx >= 0 of a tile with kChunks 16-byte chunks per row (shift and mask when
// kChunks is a power of two)
template <int kChunks>
__device__ __forceinline__ int chunk_row(int idx) {
  if constexpr ((kChunks & (kChunks - 1)) == 0) return idx >> (kChunks == 4 ? 2 : kChunks == 8 ? 3 : 4);
  else return idx / kChunks;
}
template <int kChunks>
__device__ __forceinline__ int chunk_col(int idx) {
  if constexpr ((kChunks & (kChunks - 1)) == 0) return idx & (kChunks - 1);
  else return idx % kChunks;
}

// rows [r0, r0 + 64) of a [rows, ld] 16-bit matrix, columns [col, col + D), into a swizzled tile; rows >= n_rows
// are zero-filled
template <int D>
__device__ __forceinline__ void load_tile(uint16_t* tile, const uint16_t* base, int64_t ld, int r0, int n_rows, int col) {
  constexpr int kChunks = D / 8;   // 16-byte chunks per row
  const uint32_t s = smem_u32(tile);
#pragma unroll
  for (int i = 0; i < 64 * kChunks / kAttnThreads; ++i) {
    const int idx = threadIdx.x + i * kAttnThreads;
    const int r = chunk_row<kChunks>(idx), c = chunk_col<kChunks>(idx);
    const bool ok = r0 + r < n_rows;
    const uint16_t* src = base + static_cast<int64_t>(ok ? r0 + r : 0) * ld + col + c * 8;
    cp_async16(s + swz<D>(r, c) * 2, src, ok);
  }
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}

// d (16 x 8 fp32) += a (16 x 16) * b (16 x 8)
template <bool BF16>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (BF16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads) attn_kernel(const AttnArgs p) {
  constexpr int kTileElems = tile_elems<D>();
  constexpr int kChunks = D / 8;   // 16-byte chunks per tile row
  extern __shared__ __align__(128) uint16_t smem_attn[];
  uint16_t* sQ = smem_attn;
  uint16_t* sK = sQ + kTileElems;        // [2][64 x D]
  uint16_t* sV = sK + 2 * kTileElems;    // [2][64 x D]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kQ, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / p.group;
  const uint16_t* qb = p.q + b * p.q_bs;
  const uint16_t* kbase = p.k + b * p.k_bs;
  const uint16_t* vbase = p.v + b * p.v_bs;
  const int qc = p.q_col + h * D, kc = p.k_col + hk * D, vc = p.v_col + hk * D;
  const int n_tiles = (p.Nk + kK - 1) / kK;

  pdl_launch_dependents();
  pdl_wait();   // q / k / v are written by the previous kernels
  load_tile<D>(sQ, qb, p.ldq, q0, p.Nq, qc);
  load_tile<D>(sK, kbase, p.ldk, 0, p.Nk, kc);
  load_tile<D>(sV, vbase, p.ldv, 0, p.Nk, vc);
  cp_async_commit();

  uint32_t qf[D / 16][4];   // Q fragments of this warp's 16 rows, D / 16 16-wide slices of the head dim
  float o[D / 8][4];        // O: 16 rows x D columns as D / 8 8-column fragments
  float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f};   // rows lane / 4 and lane / 4 + 8 (scaled log2 units)
#pragma unroll
  for (int j = 0; j < D / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;

  for (int t = 0; t < n_tiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < n_tiles) {   // next tile into the other buffer (freed by the barrier at the end of tile t - 1)
      load_tile<D>(sK + (buf ^ 1) * kTileElems, kbase, p.ldk, (t + 1) * kK, p.Nk, kc);
      load_tile<D>(sV + (buf ^ 1) * kTileElems, vbase, p.ldv, (t + 1) * kK, p.Nk, vc);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (t == 0) {
      const uint32_t sq = smem_u32(sQ);
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const int r = warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1), c = 2 * kk + (lane >> 4);
        ldsm_x4(sq + swz<D>(r, c) * 2, qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
      }
    }
    // S = Q K^T: 16 rows x 64 keys
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
    const uint32_t sk = smem_u32(sK + buf * kTileElems);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int nb = 0; nb < 4; ++nb) {   // keys 16 nb .. 16 nb + 15
        const int r = 16 * nb + (lane & 7) + 8 * (lane >> 4), c = 2 * kk + ((lane >> 3) & 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(sk + swz<D>(r, c) * 2, b0, b1, b2, b3);
        mma16816<BF16>(s[2 * nb], qf[kk], b0, b1);
        mma16816<BF16>(s[2 * nb + 1], qf[kk], b2, b3);
      }
    }
    // online softmax
    const int key0 = t * kK + 2 * (lane & 3);
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool ok = key0 + 8 * j + (e & 1) < p.Nk;
        s[j][e] = ok ? s[j][e] * p.scale_log2 : -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[j][e]);
      }
    }
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
      alpha[i] = exp2f(m[i] - mx[i]);
      m[i] = mx[i];
      l[i] *= alpha[i];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        s[j][e] = exp2f(s[j][e] - m[e >> 1]);
        l[e >> 1] += s[j][e];
        if (j < D / 8) o[j][e] *= alpha[e >> 1];
      }
    }
#pragma unroll
    for (int j = 8; j < D / 8; ++j) {   // head dims 96, 128: the O fragments past the eighth
#pragma unroll
      for (int e = 0; e < 4; ++e) o[j][e] *= alpha[e >> 1];
    }
    // O += P V
    const uint32_t sv = smem_u32(sV + buf * kTileElems);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {   // keys 16 kk .. 16 kk + 15
      uint32_t a[4];
      a[0] = Op16<BF16>::pack(s[2 * kk][0], s[2 * kk][1]);
      a[1] = Op16<BF16>::pack(s[2 * kk][2], s[2 * kk][3]);
      a[2] = Op16<BF16>::pack(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = Op16<BF16>::pack(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int db = 0; db < D / 16; ++db) {   // head-dim columns 16 db .. 16 db + 15
        const int r = 16 * kk + (lane & 7) + 8 * ((lane >> 3) & 1), c = 2 * db + (lane >> 4);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(sv + swz<D>(r, c) * 2, b0, b1, b2, b3);
        mma16816<BF16>(o[2 * db], a, b0, b1);
        mma16816<BF16>(o[2 * db + 1], a, b2, b3);
      }
    }
    __syncthreads();   // this buffer may be refilled
  }

  // normalise; stage the warp's 16 rows in its own rows of the Q tile, then 16-byte stores
  float inv[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
    inv[i] = 1.f / l[i];
  }
  const int rr = warp * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < D / 8; ++j) {
    const int col = 8 * j + 2 * (lane & 3);
    *reinterpret_cast<uint32_t*>(sQ + swz<D>(rr, col >> 3) + (col & 7)) = Op16<BF16>::pack(o[j][0] * inv[0], o[j][1] * inv[0]);
    *reinterpret_cast<uint32_t*>(sQ + swz<D>(rr + 8, col >> 3) + (col & 7)) =
        Op16<BF16>::pack(o[j][2] * inv[1], o[j][3] * inv[1]);
  }
  __syncwarp();
  uint16_t* ob = p.o + b * p.o_bs + h * D;
#pragma unroll
  for (int i = 0; i < 16 * kChunks / 32; ++i) {
    const int idx = lane + 32 * i;
    const int r = warp * 16 + chunk_row<kChunks>(idx), c = chunk_col<kChunks>(idx);
    if (q0 + r < p.Nq)
      *reinterpret_cast<uint4*>(ob + static_cast<int64_t>(q0 + r) * p.ldo + c * 8) =
          *reinterpret_cast<const uint4*>(sQ + swz<D>(r, c));
  }
}

}  // namespace

// q / k / v are 16-bit row-major buffers [batch, rows, cols] with row strides ld* and batch strides
// *_bs (elements); head h of q lives at columns q_col + h*head_dim (k, v likewise with the kv head).
// For the fused QKV buffer pass the same pointer three times with different column offsets.
int launch_attention_tc(const void* q, const void* k, const void* v, void* o, int64_t ldq, int64_t ldk, int64_t ldv,
                        int64_t ldo, int64_t q_bs, int64_t k_bs, int64_t v_bs, int64_t o_bs, int q_cols, int k_cols,
                        int v_cols, int q_col, int k_col, int v_col, int batch, int H, int H_kv, int Nq, int Nk,
                        int head_dim, bool bf16, cudaStream_t stream) {
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
  const dim3 grid(ceil_div(Nq, kQ), H, batch);
  SATB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "attention grid too large");
  auto go = [&](auto kern, int smem, PerDeviceOnce& once) -> int {
    if (once.first()) SATB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    SATB_CHECK_CUDA(launch_pdl(kern, grid, dim3(kAttnThreads), smem, stream, a));
    return 0;
  };
  static PerDeviceOnce once[4][2];   // [head_dim / 32 - 1][bf16]
  PerDeviceOnce& on = once[head_dim / 32 - 1][bf16 ? 1 : 0];
  switch (head_dim) {
    case 32: SATB_PROPAGATE(bf16 ? go(attn_kernel<32, true>, attn_smem<32>(), on) : go(attn_kernel<32, false>, attn_smem<32>(), on)); break;
    case 64: SATB_PROPAGATE(bf16 ? go(attn_kernel<64, true>, attn_smem<64>(), on) : go(attn_kernel<64, false>, attn_smem<64>(), on)); break;
    case 96: SATB_PROPAGATE(bf16 ? go(attn_kernel<96, true>, attn_smem<96>(), on) : go(attn_kernel<96, false>, attn_smem<96>(), on)); break;
    default: SATB_PROPAGATE(bf16 ? go(attn_kernel<128, true>, attn_smem<128>(), on) : go(attn_kernel<128, false>, attn_smem<128>(), on)); break;
  }
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace satb
