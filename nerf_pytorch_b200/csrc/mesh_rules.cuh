// mesh_rules.cuh -- the lattice of include/nerfb200.h "meshes" and its vertex, gradient and view-direction rules:
// shared by the marching cubes (mesh_common.cuh) and the attributes of baked-field meshes (baked.cu).
#pragma once

#include "common.cuh"

namespace nerfb200 {

namespace {

struct Lattice {
  int n[3];        // points per axis = res + 1
  int res[3];
  float lo[3], hi[3];
  int64_t n01;     // points per z plane
  int64_t total;   // lattice points
};

Lattice make_lattice(const nerfb200_grid_t& g) {
  Lattice L;
  for (int c = 0; c < 3; ++c) {
    L.res[c] = g.res[c];
    L.n[c] = g.res[c] + 1;
    L.lo[c] = g.lo[c];
    L.hi[c] = g.hi[c];
  }
  L.n01 = (int64_t)L.n[0] * L.n[1];
  L.total = L.n01 * L.n[2];
  return L;
}

// p_c(i) of the header: lo + ((hi - lo) * i) / res, each op rounded (the host evaluates the same fp32 operations)
__host__ __device__ __forceinline__ float lattice_coord(const Lattice& L, int c, int i) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(L.lo[c], __fdiv_rn(__fmul_rn(__fsub_rn(L.hi[c], L.lo[c]), (float)i), (float)L.res[c]));
#else
  return L.lo[c] + ((L.hi[c] - L.lo[c]) * (float)i) / (float)L.res[c];
#endif
}

// the header's vertex on a crossing edge along axis a from lattice index ia: t, and the coordinate along a
__device__ __forceinline__ float edge_t(float level, float v0, float v1) {
  return __fdiv_rn(__fsub_rn(level, v0), __fsub_rn(v1, v0));
}
__device__ __forceinline__ float edge_coord(const Lattice& L, int a, int ia, float p0a, float t) {
  return __fadd_rn(p0a, __fmul_rn(t, __fsub_rn(lattice_coord(L, a, ia + 1), p0a)));
}

// one component of the header's lattice gradient: (v[hi] - v[lo]) / (h_c * (hi - lo))
__device__ __forceinline__ float grad_component(const Lattice& L, int c, float v_hi, float v_lo, int hi, int lo) {
  const float h = __fdiv_rn(__fsub_rn(L.hi[c], L.lo[c]), (float)L.res[c]);
  return __fdiv_rn(__fsub_rn(v_hi, v_lo), __fmul_rn(h, (float)(hi - lo)));
}

// the header's view direction from the gradients at the edge's two ends; false where it fell back to (0, 0, 1)
__device__ __forceinline__ bool edge_dir(const float g0[3], const float g1[3], float t, float d[3]) {
  float g[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) g[c] = __fadd_rn(g0[c], __fmul_rn(t, __fsub_rn(g1[c], g0[c])));
  const float s = __fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2]));
  d[0] = 0.f;
  d[1] = 0.f;
  d[2] = 1.f;
  const bool ok = s > 0.f && s < INFINITY;
  if (ok) {
    const float r = __fsqrt_rn(s);
#pragma unroll
    for (int c = 0; c < 3; ++c) d[c] = __fdiv_rn(g[c], r);
  }
  return ok;
}

}  // namespace

}  // namespace nerfb200
