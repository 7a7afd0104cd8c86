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

// the upstream coefficients of a ray's samples, L = sum_i w_i v_i with v_i = g_rgb . c_i + G_acc + G_depth z_i: adds to
// G_acc and G_depth the terms of the white background (rgb_map += 1 - acc, :50-51) and of disp = 1 / max(1e-10,
// depth / acc) (:48), given the ray's upstream rgb / disp gradient g0 and its totals depth and acc
__device__ __forceinline__ void composite_upstream(const float4& g0, int white_bkgd, float adepth, float aacc,
                                                   float& G_acc, float& G_depth) {
  if (white_bkgd) G_acc -= (g0.x + g0.y + g0.z);
  if (g0.w != 0.f) {
    const float ratio = adepth / aacc;
    if (ratio > 1e-10f || ratio != ratio) {
      const float disp = 1.0f / ratio;
      G_depth += g0.w * (-disp * disp) / aacc;
      G_acc += g0.w * (disp * disp) * adepth / (aacc * aacc);
    }
  }
}

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
