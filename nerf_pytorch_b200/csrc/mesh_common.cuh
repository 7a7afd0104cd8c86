// mesh_common.cuh -- what the dense (mesh.cu) and the sparse (mesh_sparse.cu) marching cubes share: the lattice and
// rules of mesh_rules.cuh, and the one-CTA scan of per-tile totals.
#pragma once

#include "mesh_rules.cuh"

namespace nerfb200 {

namespace {

constexpr int kMeshScanThreads = 1024;
constexpr int kCtasPerSm = 8;

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
