// mesh_common.cuh -- what the dense (mesh.cu) and the sparse (mesh_sparse.cu) marching cubes share: the lattice of
// include/nerfb200.h "meshes", its vertex and view-direction rules, and the one-CTA scan of per-tile totals.
#pragma once

#include "common.cuh"

namespace nerfb200 {

namespace {

constexpr int kMeshScanThreads = 1024;
constexpr int kCtasPerSm = 8;

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

// the header's view direction from the gradients at the edge's two ends
__device__ __forceinline__ void edge_dir(const float g0[3], const float g1[3], float t, float d[3]) {
  float g[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) g[c] = __fadd_rn(g0[c], __fmul_rn(t, __fsub_rn(g1[c], g0[c])));
  const float s = __fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2]));
  d[0] = 0.f;
  d[1] = 0.f;
  d[2] = 1.f;
  if (s > 0.f && s < INFINITY) {
    const float r = __fsqrt_rn(s);
#pragma unroll
    for (int c = 0; c < 3; ++c) d[c] = __fdiv_rn(g[c], r);
  }
}

// exclusive prefix sums of the tile totals, one CTA: each thread sums a contiguous run of tiles, the runs are scanned in
// shared memory, then each thread writes its run's offsets
__global__ void __launch_bounds__(kMeshScanThreads)
mesh_scan_kernel(const int* __restrict__ tile_v, const int* __restrict__ tile_f, int64_t n_tiles,
                 long long* __restrict__ voff, long long* __restrict__ foff, long long* __restrict__ totals) {
  __shared__ long long sv[kMeshScanThreads], sf[kMeshScanThreads];
  const int tid = threadIdx.x;
  const int64_t run = (n_tiles + kMeshScanThreads - 1) / kMeshScanThreads;
  const int64_t b0 = min(n_tiles, tid * run), b1 = min(n_tiles, b0 + run);
  long long v = 0, f = 0;
  for (int64_t b = b0; b < b1; ++b) {
    v += tile_v[b];
    f += tile_f[b];
  }
  sv[tid] = v;
  sf[tid] = f;
  __syncthreads();
  for (int o = 1; o < kMeshScanThreads; o <<= 1) {
    const long long av = tid >= o ? sv[tid - o] : 0, af = tid >= o ? sf[tid - o] : 0;
    __syncthreads();
    sv[tid] += av;
    sf[tid] += af;
    __syncthreads();
  }
  long long rv = sv[tid] - v, rf = sf[tid] - f;
  for (int64_t b = b0; b < b1; ++b) {
    voff[b] = rv;
    foff[b] = rf;
    rv += tile_v[b];
    rf += tile_f[b];
  }
  if (tid == kMeshScanThreads - 1) {
    totals[0] = sv[tid];
    totals[1] = sf[tid];
  }
}

// CTAs of a tile loop: enough to fill every SM several times over, few enough that each loads the case table into
// shared memory once for many tiles
unsigned grid_for(int64_t tiles) {
  const int64_t cap = (int64_t)device_sms() * kCtasPerSm;
  return (unsigned)(tiles < cap ? tiles : cap);
}

}  // namespace

}  // namespace nerfb200
