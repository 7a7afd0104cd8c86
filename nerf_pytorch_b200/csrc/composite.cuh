// composite.cuh -- the per-sample terms of volume_render_radiance_field (nerf/volume_rendering_utils.py:6-53) and the
// warp scan of its exclusive cumprod: shared by the compositing kernels (composite.cu) and the baked-field renderer
// (baked.cu).
#pragma once

#include "common.cuh"

namespace nerfb200 {

struct SampleTerms {
  float alpha, q, sigma_delta_exp, delta;  // alpha, 1 - alpha + 1e-10, exp(-sigma*delta), delta
  bool gate;                               // raw_sigma + noise > 0 (ReLU open)
};

__device__ __forceinline__ SampleTerms sample_terms(float raw_sigma, float noise, float noise_std, bool has_noise,
                                                    float z_i, float z_next, bool last, float dnorm) {
  SampleTerms t;
  float delta = last ? 1e10f : __fsub_rn(z_next, z_i);   // volume_rendering_utils.py:14-23
  delta = __fmul_rn(delta, dnorm);                       // :24
  float pre = raw_sigma;
  if (has_noise) pre = __fadd_rn(raw_sigma, __fmul_rn(noise, noise_std));  // :27-38
  t.gate = pre > 0.f;
  const float sigma = fmaxf(pre, 0.f);
  const float e = expf(-__fmul_rn(sigma, delta));        // :39
  t.alpha = __fsub_rn(1.0f, e);
  t.q = __fadd_rn(__fsub_rn(1.0f, t.alpha), 1e-10f);     // :40
  t.sigma_delta_exp = e;
  t.delta = delta;
  return t;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// exclusive multiplicative scan across lanes
__device__ __forceinline__ float warp_excl_prod(float v, int lane) {
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc *= n;
  }
  const float ex = __shfl_up_sync(0xffffffffu, inc, 1);
  return lane == 0 ? 1.0f : ex;
}

}  // namespace nerfb200
