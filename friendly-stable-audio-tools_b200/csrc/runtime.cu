// Host-side runtime pieces shared by all kernels: error string, SM count, launch
// counter and TMA tensor-map construction (driver entry point fetched through the
// runtime so the library does not link libcuda and loads on CPU-only machines).
#include <mutex>

#include "common.cuh"
#include "gemm.cuh"
#include "kernels.h"

namespace satb {

static thread_local std::string g_last_error;
unsigned long long g_launch_count = 0;

void set_last_error(const std::string& msg) { g_last_error = msg; }
const char* get_last_error() { return g_last_error.c_str(); }

int device_sm_count() {
  static int cached[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    cudaDeviceGetAttribute(&cached[dev], cudaDevAttrMultiProcessorCount, dev);
    if (cached[dev] <= 0) cached[dev] = 132;
  }
  return cached[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// A operand: 16-bit (elem_bytes 2) or e4m3 (elem_bytes 1), dims (K, phase, rows, batches) with position =
// row*stride + phase (stride 1 for everything but strided convolutions), box (128 B of K, 1, 128, 1), 128B swizzle,
// zero OOB fill.  L = number of rows (positions / stride).
int make_tmap_a(CUtensorMap* m, const void* ptr, int K, int L, int batches, int64_t row_stride_elems,
                int64_t batch_stride_elems, int stride, int box_rows, int elem_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  SATB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA base must be 16B aligned");
  SATB_REQUIRE(elem_bytes == 1 || elem_bytes == 2, "TMA element size must be 1 or 2 bytes");
  const int eb = elem_bytes;
  SATB_REQUIRE((row_stride_elems * eb) % 16 == 0 && (batch_stride_elems * eb) % 16 == 0, "TMA strides must be 16B multiples");
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(stride), static_cast<cuuint64_t>(L),
                        static_cast<cuuint64_t>(batches)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(row_stride_elems) * eb,
                           static_cast<cuuint64_t>(row_stride_elems) * eb * stride,
                           static_cast<cuuint64_t>(batch_stride_elems) * eb};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(kBlockK * 2 / eb), 1, static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, eb == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(A) failed with CUresult " + std::to_string(static_cast<int>(r)) +
                   " K=" + std::to_string(K) + " L=" + std::to_string(L) + " batches=" + std::to_string(batches) +
                   " rs=" + std::to_string(row_stride_elems) + " bs=" + std::to_string(batch_stride_elems));
    return -3;
  }
  return 0;
}

// B operand (weights): 16-bit or e4m3 (elem_bytes 1), dims (K, rows), box (128 B of K, box_rows), 128B swizzle.
int make_tmap_b(CUtensorMap* m, const void* ptr, int K, int rows, int64_t row_stride_elems, int box_rows,
                int elem_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  SATB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA base must be 16B aligned");
  SATB_REQUIRE(elem_bytes == 1 || elem_bytes == 2, "TMA element size must be 1 or 2 bytes");
  const int eb = elem_bytes;
  SATB_REQUIRE((row_stride_elems * eb) % 16 == 0, "TMA strides must be 16B multiples");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(row_stride_elems) * eb};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kBlockK * 2 / eb), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, eb == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(B) failed with CUresult " + std::to_string(static_cast<int>(r)) +
                   " K=" + std::to_string(K) + " rows=" + std::to_string(rows));
    return -3;
  }
  return 0;
}

// Generic 2-D / 3-D map (rank = number of dims given, 2 or 3): dims[0] innermost (elements), strides in bytes of dims 1
// and 2, box per dim; zero OOB fill.  dtype: CU_TENSOR_MAP_DATA_TYPE_UINT8 or _FLOAT32.
int make_tmap_nd(CUtensorMap* m, const void* ptr, int rank, int dtype, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  SATB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  SATB_REQUIRE(rank == 2 || rank == 3, "tensor map rank must be 2 or 3");
  SATB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA base must be 16B aligned");
  for (int i = 0; i + 1 < rank; ++i) SATB_REQUIRE(strides_bytes[i] % 16 == 0, "TMA strides must be 16B multiples");
  cuuint64_t d[3], s[2];
  cuuint32_t b[3], e[3] = {1, 1, 1};
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
  CUresult r = fn(m, static_cast<CUtensorMapDataType>(dtype), rank, const_cast<void*>(ptr), d, s, b, e,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, static_cast<CUtensorMapSwizzle>(swizzle),
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)) + " dims " +
                   std::to_string(dims[0]) + " x " + std::to_string(dims[1]) + (rank == 3 ? " x " + std::to_string(dims[2]) : ""));
    return -3;
  }
  return 0;
}

}  // namespace satb
