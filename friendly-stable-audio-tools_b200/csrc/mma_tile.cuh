// mma.sync building blocks of the tensor-core attention kernels (attention_tc.cu attn_kernel, t5.cu t5_attn_kernel):
// 64 x D 16-bit tiles in XOR-swizzled shared memory filled by cp.async, ldmatrix fragment loads and the m16n8k16 MMA.
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

}  // namespace
}  // namespace satb
