// e4m3 quantisation helpers shared by the FP8 operand mode (elementwise.cu) and FP8 attention (attention_fp8.cu).
#pragma once
#include <cuda_fp8.h>
#include <stdint.h>

namespace satb {

// ------------------------------------------------------- FP8 (e4m3) operands with power-of-two row scales
// s = 2^e, e the smallest integer with amax <= 448 * 2^e (448: the largest finite e4m3), s = 1 for an all-zero row;
// q = e4m3_rn(x * 2^-e).  With 448 = 1.75 * 2^8 and amax = m * 2^E, m in [1, 2): e = E - 8 if m <= 1.75, else E - 7.
// e is kept >= -126 so that s and 2^-e are normal fp32 numbers (only rows with amax < 2^-117 are affected: their
// values fall into the e4m3 subnormals).  Integer arithmetic on the bits: exact, whatever the fast-math flags.
__device__ __forceinline__ int fp8_row_exp(float amax) {
  if (!(amax > 0.f)) return 0;
  const uint32_t b = __float_as_uint(amax);
  const int E = static_cast<int>(b >> 23) - 127;
  const int e = (b & 0x7FFFFFu) <= 0x600000u ? E - 8 : E - 7;
  return e < -126 ? -126 : e;
}
__device__ __forceinline__ float pow2f(int e) { return __uint_as_float(static_cast<uint32_t>(e + 127) << 23); }
// four values -> four e4m3 bytes (round to nearest even), the first value in the lowest byte
__device__ __forceinline__ uint32_t e4m3x4(float a, float b, float c, float d) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}

}  // namespace satb
