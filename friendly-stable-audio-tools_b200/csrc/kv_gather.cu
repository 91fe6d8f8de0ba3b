// K/V gather of the token-sharded DiT forward (satb_dit_group_forward): every rank holds a contiguous range of every
// item's tokens, and its self-attention needs the keys and values of all of them.  Once per layer each rank pulls the
// k | v columns of every rank's qkv into one full-sequence buffer, reading the other ranks' buffers through peer
// pointers.  A pure copy: one 16-byte load and one 16-byte store per 8 elements, so it runs at the bandwidth of the
// slowest link it reads over.
#include "../../include/satb200.h"
#include "common.cuh"
#include "kernels.h"

namespace satb {

namespace {

constexpr int kGatherThreads = 256;
constexpr int kGatherUnroll = 4;   // 16-byte loads in flight per thread before the first store

struct KvGatherArgs {
  const uint4* src[kKvGatherMaxRanks];   // rank s's qkv [R, n_s, 3D] 16-bit
  int begin[kKvGatherMaxRanks + 1];      // rank s holds tokens begin[s] .. begin[s + 1] - 1 of every item
  int world;
};

// kv[(r N + tok) 2D + c] = qkv_s[(r n_s + tok - begin[s]) 3D + D + c] for the rank s whose range holds tok.
// Work items are 16-byte chunks, cpr = 2D / 8 per token row; the rows of one chunk index never straddle a source.
__global__ void __launch_bounds__(kGatherThreads) kv_gather_kernel(KvGatherArgs a, uint4* __restrict__ kv, int N,
                                                                   int cpr, int64_t total) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kGatherThreads * kGatherUnroll;
  const int src_ld = cpr + cpr / 2;   // 3D in 16-byte chunks
  for (int64_t base = static_cast<int64_t>(blockIdx.x) * kGatherThreads * kGatherUnroll + threadIdx.x; base < total;
       base += stride) {
    uint4 v[kGatherUnroll];
#pragma unroll
    for (int u = 0; u < kGatherUnroll; ++u) {
      const int64_t i = base + static_cast<int64_t>(u) * kGatherThreads;
      if (i < total) {
        const int64_t row = i / cpr;
        const int c = static_cast<int>(i - row * cpr);
        const int r = static_cast<int>(row / N), tok = static_cast<int>(row - static_cast<int64_t>(r) * N);
        // the source rank by selects over the unrolled ranks (a dynamic index into the parameters would go to the stack)
        const uint4* src = a.src[0];
        int b0 = 0, b1 = a.begin[1];
#pragma unroll
        for (int q = 1; q < kKvGatherMaxRanks; ++q)
          if (q < a.world && tok >= a.begin[q]) {
            src = a.src[q];
            b0 = a.begin[q];
            b1 = a.begin[q + 1];
          }
        const uint4* p = src + (static_cast<int64_t>(r) * (b1 - b0) + (tok - b0)) * src_ld + cpr / 2 + c;
        v[u] = __ldcs(p);   // read once: streamed past the caches
      }
    }
#pragma unroll
    for (int u = 0; u < kGatherUnroll; ++u) {
      const int64_t i = base + static_cast<int64_t>(u) * kGatherThreads;
      if (i < total) kv[i] = v[u];
    }
  }
}

}  // namespace

int launch_kv_gather(const void* const* qkv, const int* token_begin, int world, void* kv, int R, int D,
                     cudaStream_t stream) {
  SATB_REQUIRE(world >= 1 && world <= kKvGatherMaxRanks, "kv gather: world must be 1 .. 8");
  SATB_REQUIRE(R >= 1 && D >= 8 && D % 8 == 0, "kv gather: need R >= 1 and D % 8 == 0");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(kv) & 15) == 0, "kv gather: kv must be 16-byte aligned");
  KvGatherArgs a = {};
  a.world = world;
  for (int s = 0; s < world; ++s) {
    SATB_REQUIRE(qkv[s] && (reinterpret_cast<uintptr_t>(qkv[s]) & 15) == 0, "kv gather: qkv must be 16-byte aligned");
    SATB_REQUIRE(token_begin[s + 1] > token_begin[s], "kv gather: every rank must hold at least one token");
    a.src[s] = static_cast<const uint4*>(qkv[s]);
    a.begin[s] = token_begin[s];
  }
  SATB_REQUIRE(token_begin[0] == 0, "kv gather: rank 0 must start at token 0");
  const int N = token_begin[world];
  for (int s = world; s <= kKvGatherMaxRanks; ++s) a.begin[s] = N;
  const int cpr = 2 * D / 8;
  const int64_t total = static_cast<int64_t>(R) * N * cpr;
  int64_t grid = ceil_div64(total, static_cast<int64_t>(kGatherThreads) * kGatherUnroll);
  const int64_t cap = 8LL * device_sm_count();
  if (grid > cap) grid = cap;
  kv_gather_kernel<<<static_cast<unsigned>(grid), kGatherThreads, 0, stream>>>(a, static_cast<uint4*>(kv), N, cpr,
                                                                                total);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace satb

extern "C" int satb_kv_gather(const void* const* qkv, const int* token_begin, int world, void* kv, int R, int D,
                              void* stream) {
  SATB_REQUIRE(qkv && token_begin && kv, "null argument");
  return satb::launch_kv_gather(qkv, token_begin, world, kv, R, D, static_cast<cudaStream_t>(stream));
}
