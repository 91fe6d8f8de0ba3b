// Output gather of the time-sharded Oobleck decode / encode (satb_oobleck_group_*): every rank holds the output of its
// extended slice [B, C, n_ext] (its own range plus the recompute margin on each interior side), and the home device
// copies each rank's kept range out of it, reading the other devices' buffers through peer pointers, into the final
// [B, C, T] tensor.  The crop of the margin is the source offset of the copy.  A pure copy: 16-byte loads and stores
// when every offset and row length is a multiple of 4 floats (the decoder's audio, at multiples of the upsampling
// ratio), 4-byte ones otherwise (the encoder's latents).
#include "../../include/satb200.h"
#include "common.cuh"
#include "kernels.h"

namespace satb {

namespace {

constexpr int kTimeGatherThreads = 256;
constexpr int kTimeGatherUnroll = 4;   // loads in flight per thread before the first store

// Lengths and offsets in units of V (float4 or float).
struct TimeGatherArgs {
  const void* src[kKvGatherMaxRanks];   // rank q's output [rows, src_ld[q]]
  int src_ld[kKvGatherMaxRanks];        // its row length
  int src_off[kKvGatherMaxRanks];       // the first kept position of a row (the margin it recomputed on the left)
  int begin[kKvGatherMaxRanks + 1];     // rank q writes out positions begin[q] .. begin[q + 1] - 1 of every row
  int world;
};

// out[row, t] = src_q[row, src_off[q] + t - begin[q]] for the rank q whose range holds t.  Rows by blockIdx.y, positions
// by blockIdx.x, both grid-strided: no division per element.
template <class V>
__global__ void __launch_bounds__(kTimeGatherThreads) time_gather_kernel(TimeGatherArgs a, V* __restrict__ out, int T,
                                                                         int rows) {
  const int stride = gridDim.x * kTimeGatherThreads * kTimeGatherUnroll;
  for (int row = blockIdx.y; row < rows; row += gridDim.y) {
    V* o = out + static_cast<int64_t>(row) * T;
    for (int base = blockIdx.x * kTimeGatherThreads * kTimeGatherUnroll + threadIdx.x; base < T; base += stride) {
      V v[kTimeGatherUnroll];
#pragma unroll
      for (int u = 0; u < kTimeGatherUnroll; ++u) {
        const int t = base + u * kTimeGatherThreads;
        if (t < T) {
          // the source rank by selects over the unrolled ranks (a dynamic index into the parameters would go to the stack)
          const void* src = a.src[0];
          int ld = a.src_ld[0], off = a.src_off[0], b0 = 0;
#pragma unroll
          for (int q = 1; q < kKvGatherMaxRanks; ++q)
            if (q < a.world && t >= a.begin[q]) {
              src = a.src[q];
              ld = a.src_ld[q];
              off = a.src_off[q];
              b0 = a.begin[q];
            }
          v[u] = __ldcs(static_cast<const V*>(src) + static_cast<int64_t>(row) * ld + off + (t - b0));   // read once
        }
      }
#pragma unroll
      for (int u = 0; u < kTimeGatherUnroll; ++u) {
        const int t = base + u * kTimeGatherThreads;
        if (t < T) o[t] = v[u];
      }
    }
  }
}

}  // namespace

int launch_time_gather(const float* const* src, const int* src_len, const int* src_off, const int* begin, int world,
                       float* out, int rows, int T, cudaStream_t stream) {
  SATB_REQUIRE(world >= 1 && world <= kKvGatherMaxRanks, "time gather: world must be 1 .. 8");
  SATB_REQUIRE(out && rows >= 1 && T >= 1 && begin[0] == 0 && begin[world] == T, "time gather: bad shape");
  // 16-byte units when every pointer, row length and offset allows them
  bool vec = (reinterpret_cast<uintptr_t>(out) & 15) == 0 && T % 4 == 0;
  for (int q = 0; q < world; ++q) {
    SATB_REQUIRE(src[q] && begin[q + 1] > begin[q] && src_off[q] >= 0 && src_off[q] + begin[q + 1] - begin[q] <= src_len[q],
                 "time gather: every rank needs a non-empty kept range inside its output");
    vec = vec && (reinterpret_cast<uintptr_t>(src[q]) & 15) == 0 && src_len[q] % 4 == 0 && src_off[q] % 4 == 0 &&
          begin[q] % 4 == 0;
  }
  const int u = vec ? 4 : 1;
  TimeGatherArgs a = {};
  a.world = world;
  for (int q = 0; q < world; ++q) {
    a.src[q] = src[q];
    a.src_ld[q] = src_len[q] / u;
    a.src_off[q] = src_off[q] / u;
    a.begin[q] = begin[q] / u;
  }
  for (int q = world; q <= kKvGatherMaxRanks; ++q) a.begin[q] = T / u;
  const int Tu = T / u;
  int gx = ceil_div(Tu, kTimeGatherThreads * kTimeGatherUnroll);
  if (gx > 1024) gx = 1024;
  const dim3 grid(gx, rows < 65535 ? rows : 65535);
  if (vec)
    time_gather_kernel<float4><<<grid, kTimeGatherThreads, 0, stream>>>(a, reinterpret_cast<float4*>(out), Tu, rows);
  else
    time_gather_kernel<float><<<grid, kTimeGatherThreads, 0, stream>>>(a, out, Tu, rows);
  count_launch();
  SATB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace satb
