// The sampler arithmetic of one model call for every fixed-step sampler of inference/sampling.py, as one pass over the
// latents (satb_sampler_step; the algebra is documented with SatbSamplerStep in include/satb200.h).  Euler for
// rectified flow, Heun, DPM-2, linear multistep and DPM-Solver++(2S) ancestral are all linear in the state, the model
// output, a few stored tensors (the state before a two-stage step, earlier derivatives, earlier denoised estimates)
// and the noise, so the host turns each stage into the scalars of one launch; the VDenoiser combine, the inpainting
// callback's blend and the scaling of the next model input are folded in, and no torch op runs between two model
// calls.  satb_sampler_update (elementwise.cu) stays the route of the multistep SDE samplers without a callback.
#include "../../include/satb200.h"
#include "common.cuh"
#include "kernels.h"
#include "ptx.cuh"

namespace satb {

namespace {

constexpr int kSamplerStepThreads = 256;

__device__ __forceinline__ void to_arr(const float4 v, float (&a)[4]) {
  a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
}

__device__ __forceinline__ float4 from_arr(const float (&a)[4]) { return make_float4(a[0], a[1], a[2], a[3]); }

// Grid-strided over float4 units.  The parameter block lives in the constant bank; the buffer loop is unrolled so that
// p.buf / p.c are never indexed dynamically (which would copy them to the stack).
__global__ void __launch_bounds__(kSamplerStepThreads) sampler_step_kernel(const SatbSamplerStep p) {
  pdl_launch_dependents();
  pdl_wait();
  const long long n4 = p.n >> 2;
  float4* x4 = reinterpret_cast<float4*>(p.x);
  const float4* y4 = reinterpret_cast<const float4*>(p.y);
  for (long long i = blockIdx.x * static_cast<long long>(kSamplerStepThreads) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * kSamplerStepThreads) {
    float xs[4], ys[4], den[4], dd[4];
    to_arr(x4[i], xs);
    to_arr(y4[i], ys);
#pragma unroll
    for (int k = 0; k < 4; ++k) den[k] = fmaf(p.c_out, ys[k], p.c_skip * xs[k]);   // from the unblended x
    if (p.mask) {
      float ini[4], rn[4];
      to_arr(reinterpret_cast<const float4*>(p.init)[i], ini);
      to_arr(reinterpret_cast<const float4*>(p.renoise)[i], rn);
      int l = static_cast<int>((4 * i) % p.L);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        // torch.where(mask <= thr, 1, 0) selects exactly; init + renoise * sigma rounded as the two fp32 torch ops
        if (__ldg(p.mask + l) <= p.blend_thr) xs[k] = __fadd_rn(ini[k], __fmul_rn(rn[k], p.blend_sigma));
        if (++l == p.L) l = 0;
      }
      x4[i] = from_arr(xs);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) dd[k] = (xs[k] - den[k]) * p.inv_sigma;
    if (p.x_next || p.x_in_next) {
      float o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k] = fmaf(p.a, xs[k], fmaf(p.b, den[k], p.g * dd[k]));
#pragma unroll
      for (int j = 0; j < SATB_SAMPLER_STEP_BUFS; ++j) {
        if (p.buf[j]) {
          float t[4];
          to_arr(reinterpret_cast<const float4*>(p.buf[j])[i], t);
#pragma unroll
          for (int k = 0; k < 4; ++k) o[k] = fmaf(p.c[j], t[k], o[k]);
        }
      }
      if (p.noise) {
        float t[4];
        to_arr(reinterpret_cast<const float4*>(p.noise)[i], t);
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = fmaf(p.s, t[k], o[k]);
      }
      if (p.x_next) reinterpret_cast<float4*>(p.x_next)[i] = from_arr(o);
      if (p.x_in_next)
        reinterpret_cast<float4*>(p.x_in_next)[i] =
            make_float4(o[0] * p.c_in_next, o[1] * p.c_in_next, o[2] * p.c_in_next, o[3] * p.c_in_next);
    }
    if (p.den) reinterpret_cast<float4*>(p.den)[i] = from_arr(den);
    if (p.d) reinterpret_cast<float4*>(p.d)[i] = from_arr(dd);
  }
}

inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

}  // namespace

int launch_sampler_step(const SatbSamplerStep& p, cudaStream_t stream) {
  SATB_REQUIRE(p.n > 0 && p.n % 4 == 0, "sampler step: element count must be a positive multiple of 4");
  SATB_REQUIRE(p.x && p.y, "sampler step: null x or y");
  SATB_REQUIRE(p.den || p.d || p.x_next || p.x_in_next, "sampler step: no output requested");
  SATB_REQUIRE(!p.mask || (p.init && p.renoise && p.L >= 1 && p.n % p.L == 0),
               "sampler step: the inpainting blend needs init, renoise and an L >= 1 that divides n");
  bool al = aligned16(p.x) && aligned16(p.y) && aligned16(p.noise) && aligned16(p.init) && aligned16(p.renoise) &&
            aligned16(p.den) && aligned16(p.d) && aligned16(p.x_next) && aligned16(p.x_in_next);
  for (int j = 0; j < SATB_SAMPLER_STEP_BUFS; ++j) al = al && aligned16(p.buf[j]);
  SATB_REQUIRE(al, "sampler step: every tensor must be 16-byte aligned");
  const long long n4 = p.n / 4;
  int grid = static_cast<int>(ceil_div64(n4, kSamplerStepThreads));
  if (grid > 4 * device_sm_count()) grid = 4 * device_sm_count();
  SATB_CHECK_CUDA(launch_pdl(sampler_step_kernel, dim3(grid), dim3(kSamplerStepThreads), 0, stream, p));
  count_launch();
  return 0;
}

}  // namespace satb

extern "C" int satb_sampler_step(const SatbSamplerStep* p, void* stream) {
  SATB_REQUIRE(p, "null argument");
  return satb::launch_sampler_step(*p, static_cast<cudaStream_t>(stream));
}
