// The mma.sync flash-attention core shared by attention_tc.cu attn_kernel, t5.cu t5_attn_kernel and roberta.cu
// rb_attn_kernel, and its building blocks: 64 x D 16-bit tiles in XOR-swizzled shared memory filled by cp.async,
// ldmatrix fragment loads and the m16n8k16 MMA.  Each kernel is a thin wrapper that finds its item's rows, sets up its
// score policy and runs mma_attention.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace satb {
namespace {

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
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
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
// by a CTA of kThreads threads
template <int D, int kThreads = 128>
__device__ __forceinline__ void load_tile(uint16_t* tile, const uint16_t* base, int64_t ld, int r0, int n_rows, int col) {
  constexpr int kChunks = D / 8;   // 16-byte chunks per row
  const uint32_t s = smem_u32(tile);
#pragma unroll
  for (int i = 0; i < 64 * kChunks / kThreads; ++i) {
    const int idx = threadIdx.x + i * kThreads;
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

constexpr int kMmaAttnThreads = 128;   // four warps, 16 query rows each
template <int D>
constexpr int mma_attn_smem() { return 5 * 64 * D * 2; }   // Q, two K and two V 64 x D tiles: 20 .. 80 KB

// Score policy: the score times a constant, 1 / sqrt(d) in log2 units
struct ScaleScore {
  float scale_log2;
  __device__ __forceinline__ float operator()(float s, int /*query*/, int /*key*/) const { return s * scale_log2; }
};

// O = softmax(score(Q K^T)) V for query rows [q0, q0 + 64) of one (item, head), by a CTA of kMmaAttnThreads threads.
// q / k / v / o point at the item's row 0 with row pitches ld* (elements); the head occupies columns [c, c + D) of
// each.  Queries [0, n_q) and keys [0, n_k) exist (n_k >= 1); query rows past n_q are computed on zero rows and not
// stored.  smem: mma_attn_smem<D>() bytes, 128-byte aligned.  score(s, query, key) maps the fp32 Q K^T element of a
// valid key to the log2 units of the softmax; keys >= n_k are masked.
// Each warp owns 16 query rows.  Keys are processed in tiles of 64, double-buffered by cp.async (rows past n_k are
// zero-filled).  Per tile: S = Q K^T by mma.sync (Q fragments stay in registers, K fragments by ldmatrix), online
// softmax in fp32 on the S fragments (exp2, -1e30 initial maximum, row max / sum reduced over the four lanes of a row),
// then O += P V with P repacked from the S fragments into 16-bit A fragments and V fragments by ldmatrix.trans.  The
// normalised output goes through the Q tile so that it leaves as 16-byte row segments.
// The caller has run pdl_wait(): every global read here may see the previous kernel's writes.  cp.async copies the
// caller issued and did not commit join the first tiles' group: they are visible to the whole CTA from the first tile on.
template <int D, bool BF16, class Score>
__device__ __forceinline__ void mma_attention(uint16_t* smem, const uint16_t* q, int64_t ldq, int qc, const uint16_t* k,
                                              int64_t ldk, int kc, const uint16_t* v, int64_t ldv, int vc, uint16_t* o,
                                              int64_t ldo, int oc, int q0, int n_q, int n_k, const Score& score) {
  constexpr int kTileElems = 64 * D;
  constexpr int kChunks = D / 8;   // 16-byte chunks per tile row
  uint16_t* sQ = smem;
  uint16_t* sK = sQ + kTileElems;        // [2][64 x D]
  uint16_t* sV = sK + 2 * kTileElems;    // [2][64 x D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (n_k + 63) / 64;

  load_tile<D, kMmaAttnThreads>(sQ, q, ldq, q0, n_q, qc);
  load_tile<D, kMmaAttnThreads>(sK, k, ldk, 0, n_k, kc);
  load_tile<D, kMmaAttnThreads>(sV, v, ldv, 0, n_k, vc);
  cp_async_commit();

  uint32_t qf[D / 16][4];   // Q fragments of this warp's 16 rows, D / 16 16-wide slices of the head dim
  float acc[D / 8][4];      // O: 16 rows x D columns as D / 8 8-column fragments
  float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f};   // rows qrow and qrow + 8 (log2 units)
#pragma unroll
  for (int j = 0; j < D / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  const int qrow = q0 + warp * 16 + (lane >> 2);

  for (int t = 0; t < n_tiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < n_tiles) {   // next tile into the other buffer (freed by the barrier at the end of tile t - 1)
      load_tile<D, kMmaAttnThreads>(sK + (buf ^ 1) * kTileElems, k, ldk, (t + 1) * 64, n_k, kc);
      load_tile<D, kMmaAttnThreads>(sV + (buf ^ 1) * kTileElems, v, ldv, (t + 1) * 64, n_k, vc);
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
    // score, mask, online softmax
    const int key0 = t * 64 + 2 * (lane & 3);
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = key0 + 8 * j + (e & 1);
        s[j][e] = key < n_k ? score(s[j][e], qrow + 8 * (e >> 1), key) : -INFINITY;
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
      }
    }
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[j][e] *= alpha[e >> 1];
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
        mma16816<BF16>(acc[2 * db], a, b0, b1);
        mma16816<BF16>(acc[2 * db + 1], a, b2, b3);
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
    *reinterpret_cast<uint32_t*>(sQ + swz<D>(rr, col >> 3) + (col & 7)) =
        Op16<BF16>::pack(acc[j][0] * inv[0], acc[j][1] * inv[0]);
    *reinterpret_cast<uint32_t*>(sQ + swz<D>(rr + 8, col >> 3) + (col & 7)) =
        Op16<BF16>::pack(acc[j][2] * inv[1], acc[j][3] * inv[1]);
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 16 * kChunks / 32; ++i) {
    const int idx = lane + 32 * i;
    const int r = warp * 16 + chunk_row<kChunks>(idx), c = chunk_col<kChunks>(idx);
    if (q0 + r < n_q)
      *reinterpret_cast<uint4*>(o + static_cast<int64_t>(q0 + r) * ldo + oc + c * 8) =
          *reinterpret_cast<const uint4*>(sQ + swz<D>(r, c));
  }
}

// Launches Kernel, an mma_attention wrapper at head dim D, with its dynamic shared memory; the instance's shared
// memory limit is raised once per device.
template <auto Kernel, int D, class... Args>
int launch_mma_attention(dim3 grid, cudaStream_t st, const Args&... args) {
  static PerDeviceOnce once;
  if (once.first())
    SATB_CHECK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mma_attn_smem<D>()));
  SATB_CHECK_CUDA(launch_pdl(Kernel, grid, dim3(kMmaAttnThreads), mma_attn_smem<D>(), st, args...));
  return 0;
}

}  // namespace
}  // namespace satb
