// Host-side GEMM plumbing shared by the model handles (dit.cu, t5.cu): device workspaces, a tensor-map cache and the
// flat Linear launch with its N-tile choice.
#pragma once
#include <cmath>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "gemm.cuh"

namespace satb {

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  int ensure(size_t need) {
    if (need <= bytes) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    cudaError_t e = cudaMalloc(&p, need);
    if (e != cudaSuccess) {
      set_last_error(std::string("cudaMalloc failed: ") + cudaGetErrorString(e) + " (" + std::to_string(need) + " B)");
      return -2;
    }
    bytes = need;
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
  template <class T>
  T* as() const {
    return static_cast<T*>(p);
  }
};

// v into buf (grown as needed, at least 256 bytes), ordered on st: the per-item offsets and lengths the encoders'
// attention kernels read.
inline int dev_int_upload(DevBuf& buf, const std::vector<int>& v, cudaStream_t st) {
  SATB_PROPAGATE(buf.ensure(v.size() * sizeof(int) < 256 ? 256 : v.size() * sizeof(int)));
  SATB_CHECK_CUDA(cudaMemcpyAsync(buf.p, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  return 0;
}

// Tensor maps by (pointer, shape, strides, box rows, element bytes): one buffer may be read as 16-bit and as e4m3 rows.
struct TmapCache {
  typedef std::tuple<const void*, int, int, int, int64_t, int64_t, int, int> Key;
  std::map<Key, CUtensorMap> maps;
  int get_a(const void* ptr, int K, int L, int batches, int64_t rs, int64_t bs, const CUtensorMap** out,
            int elem_bytes = 2) {
    Key k(ptr, K, L, batches, rs, bs, -1, elem_bytes);
    auto it = maps.find(k);
    if (it == maps.end()) {
      CUtensorMap m;
      SATB_PROPAGATE(make_tmap_a(&m, ptr, K, L, batches, rs, bs, 1, kBlockM, elem_bytes));
      it = maps.emplace(k, m).first;
    }
    *out = &it->second;
    return 0;
  }
  int get_b(const void* ptr, int K, int rows, int64_t rs, int box_rows, const CUtensorMap** out, int elem_bytes = 2) {
    Key k(ptr, K, rows, 0, rs, 0, box_rows, elem_bytes);
    auto it = maps.find(k);
    if (it == maps.end()) {
      CUtensorMap m;
      SATB_PROPAGATE(make_tmap_b(&m, ptr, K, rows, rs, box_rows, elem_bytes));
      it = maps.emplace(k, m).first;
    }
    *out = &it->second;
    return 0;
  }
};

// Flat Linear: C[M, N] = A[M, K] * W[N, K]^T with a fused epilogue.  b_static = 1: W is a weight matrix prepared at
// finalize time, so its first tiles may be fetched before the dependency wait (every product call); satb_gemm_probe
// also runs 0.  FP8: A and W are e4m3 rows (lda in elements = bytes) with their row scales in sc.
template <class Epi, int BN, bool BF16, bool FP8 = false>
static int linear(TmapCache& tc, const void* A, int64_t lda, int M, int K, const void* W, int N,
                  const typename Epi::Params& ep, cudaStream_t stream, int b_static = 1, const Fp8Scales& sc = Fp8Scales{}) {
  const int eb = FP8 ? 1 : 2;
  const CUtensorMap *ta, *tb;
  SATB_PROPAGATE(tc.get_a(A, K, M, 1, lda, static_cast<int64_t>(M) * lda, &ta, eb));
  GemmShape s;
  s.L = M; s.batches = 1; s.N = N; s.K = K; s.n_taps = 1; s.tap_base = 0; s.tap_step = 0; s.b_tap_rows = N; s.stride = 1;
  s.b_static = b_static;
  SATB_PROPAGATE(tc.get_b(W, K, N, K, BN, &tb, eb));
  return launch_gemm<Epi, BN, BF16, FP8>(*ta, *tb, s, ep, stream, nullptr, sc);
}

// Picks the N tile (256 or 128) that wastes less of the last wave of the persistent grid; the
// 128-wide tile streams as many smem bytes per MMA cycle as the tensor pipe can take, so it is
// only preferred when it clearly wins on wave quantisation.
static int auto_bn(int m_tiles, int N) {
  const double sms = device_sm_count();
  auto eff = [&](int bn) {
    const double waves = static_cast<double>(m_tiles) * ceil_div(N, bn) / sms;
    return waves / std::ceil(waves);
  };
  return N % 128 == 0 && eff(128) * 0.9 > eff(256) ? 128 : 256;
}

template <class Epi, bool BF16, bool FP8 = false>
static int linear_auto(TmapCache& tc, const void* A, int64_t lda, int M, int K, const void* W, int N,
                       const typename Epi::Params& ep, cudaStream_t stream, const Fp8Scales& sc = Fp8Scales{}) {
  if (auto_bn(ceil_div(M, kBlockM), N) == 128) return linear<Epi, 128, BF16, FP8>(tc, A, lda, M, K, W, N, ep, stream, 1, sc);
  return linear<Epi, 256, BF16, FP8>(tc, A, lda, M, K, W, N, ep, stream, 1, sc);
}

}  // namespace satb
