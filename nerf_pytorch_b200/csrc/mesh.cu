// mesh.cu -- marching cubes over a lattice of values (include/nerfb200.h "meshes").
// Three launches over tiles of 256 consecutive lattice points, one thread per point; classify and emit loop over the
// tiles with a bounded grid, so each CTA loads the case table into shared memory once:
//   classify  each point's three owned edges (+x, +y, +z) that cross the level, as three warp ballots, and its cube's
//             triangle count; per warp the ballots and the warp's first vertex relative to its tile, per tile its totals.
//   scan      one CTA: exclusive prefix sums of the tile totals -> each tile's first vertex and first face; the two
//             grand totals stay in device memory.
//   emit      vertices of each point's crossing edges, and its cube's triangles.  A vertex id is a pure function of the
//             workspace: tile offset + warp offset + the ballot bits below the point's lane + its own lower axes, so a
//             cube finds the ids of edges owned by its neighbours without any per-point array.
// No atomics: the mesh is a function of the volume and the level.
#include <cmath>

#include "mc_table.cuh"
#include "mesh_common.cuh"

namespace nerfb200 {

namespace {

constexpr int kMeshThreads = 256;  // lattice points per tile, one CTA's threads: 8 warps
constexpr int kWarps = kMeshThreads / 32;

struct Workspace {
  uint4* warp;       // per warp: +x, +y, +z crossing ballots, first vertex relative to the tile
  int* tile_v;       // per tile: vertices, faces
  int* tile_f;
  long long* voff;   // per tile: first vertex, first face
  long long* foff;
  int64_t bytes;
};

inline int64_t align16(int64_t b) { return (b + 15) & ~int64_t(15); }

Workspace workspace_layout(const Lattice& L, void* base) {
  const int64_t tiles = (L.total + kMeshThreads - 1) / kMeshThreads;
  char* p = static_cast<char*>(base);
  Workspace w;
  int64_t off = 0;
  w.warp = reinterpret_cast<uint4*>(p + off);
  off += align16(tiles * kWarps * (int64_t)sizeof(uint4));
  w.tile_v = reinterpret_cast<int*>(p + off);
  off += align16(tiles * 4);
  w.tile_f = reinterpret_cast<int*>(p + off);
  off += align16(tiles * 4);
  w.voff = reinterpret_cast<long long*>(p + off);
  off += align16(tiles * 8);
  w.foff = reinterpret_cast<long long*>(p + off);
  off += align16(tiles * 8);
  w.bytes = off;
  return w;
}

__device__ __forceinline__ int64_t axis_stride(const Lattice& L, int a) {
  return a == 0 ? 1 : (a == 1 ? (int64_t)L.n[0] : L.n01);
}

__device__ __forceinline__ int cube_case(const Lattice& L, const float* __restrict__ vol, int64_t p, float level) {
  int cs = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int64_t q = p + (c & 1) + ((c >> 1) & 1) * (int64_t)L.n[0] + (c >> 2) * L.n01;
    cs |= (vol[q] > level ? 1 : 0) << c;
  }
  return cs;
}

// id of the vertex on lattice edge (q, a), which must cross
__device__ __forceinline__ long long vertex_id(const uint4* __restrict__ warp, const long long* __restrict__ voff,
                                               int64_t q, int a) {
  const uint4 w = warp[q >> 5];
  const int l = (int)(q & 31);
  const unsigned below = (1u << l) - 1u;
  long long id = voff[q / kMeshThreads] + (long long)w.w + __popc(w.x & below) + __popc(w.y & below) +
                 __popc(w.z & below);
  if (a >= 1) id += (w.x >> l) & 1u;
  if (a >= 2) id += (w.y >> l) & 1u;
  return id;
}

// the header's gradient at lattice point q = (i[0], i[1], i[2])
__device__ __forceinline__ void lattice_grad(const Lattice& L, const float* __restrict__ vol, int64_t q, const int i[3],
                                             float g[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int lo = i[c] > 0 ? i[c] - 1 : 0, hi = i[c] + 1 < L.n[c] ? i[c] + 1 : L.n[c] - 1;
    const int64_t s = axis_stride(L, c);
    g[c] = grad_component(L, c, vol[q + (hi - i[c]) * s], vol[q + (lo - i[c]) * s], hi, lo);
  }
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_classify_kernel(const Lattice L, const float* __restrict__ vol, float level, int64_t n_tiles,
                     uint4* __restrict__ warp_info, int* __restrict__ tile_v, int* __restrict__ tile_f) {
  __shared__ unsigned char tri_count[256];
  __shared__ int wv[kWarps], wf[kWarps];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int k = tid; k < 256; k += kMeshThreads) tri_count[k] = kMcTriCount[k];
  __syncthreads();
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t p = tile * kMeshThreads + tid;
    unsigned flags = 0;
    int tris = 0;
    if (p < L.total) {
      const int x = (int)(p % L.n[0]), y = (int)((p / L.n[0]) % L.n[1]), z = (int)(p / L.n01);
      const bool in0 = vol[p] > level;
      if (x + 1 < L.n[0] && in0 != (vol[p + 1] > level)) flags |= 1u;
      if (y + 1 < L.n[1] && in0 != (vol[p + L.n[0]] > level)) flags |= 2u;
      if (z + 1 < L.n[2] && in0 != (vol[p + L.n01] > level)) flags |= 4u;
      if (x + 1 < L.n[0] && y + 1 < L.n[1] && z + 1 < L.n[2]) tris = tri_count[cube_case(L, vol, p, level)];
    }
    const unsigned bx = __ballot_sync(0xffffffffu, flags & 1u), by = __ballot_sync(0xffffffffu, flags & 2u),
                   bz = __ballot_sync(0xffffffffu, flags & 4u);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tris += __shfl_xor_sync(0xffffffffu, tris, o);
    if (lane == 0) {
      wv[wid] = __popc(bx) + __popc(by) + __popc(bz);
      wf[wid] = tris;
    }
    __syncthreads();
    if (lane == 0) {
      int before = 0;
      for (int w = 0; w < wid; ++w) before += wv[w];
      warp_info[tile * kWarps + wid] = make_uint4(bx, by, bz, (unsigned)before);
    }
    if (tid == 0) {
      int v = 0, f = 0;
      for (int w = 0; w < kWarps; ++w) {
        v += wv[w];
        f += wf[w];
      }
      tile_v[tile] = v;
      tile_f[tile] = f;
    }
    __syncthreads();  // wv / wf are rewritten by the next tile
  }
}

__global__ void __launch_bounds__(kMeshThreads)
mesh_emit_kernel(const Lattice L, const float* __restrict__ vol, float level, int64_t n_tiles,
                 const uint4* __restrict__ warp_info, const long long* __restrict__ voff,
                 const long long* __restrict__ foff, int64_t max_v, int64_t max_f, float* __restrict__ verts,
                 int* __restrict__ faces, float* __restrict__ dirs) {
  __shared__ unsigned char tri_count[256];
  __shared__ signed char tri_edges[256][3 * NERFB200_MC_MAX_TRIS];
  __shared__ int wf[kWarps];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int k = tid; k < 256; k += kMeshThreads) tri_count[k] = kMcTriCount[k];
  for (int k = tid; k < 256 * 3 * NERFB200_MC_MAX_TRIS; k += kMeshThreads)
    (&tri_edges[0][0])[k] = (&kMcTris[0][0])[k];
  __syncthreads();
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t p = tile * kMeshThreads + tid;
    int cs = 0, tris = 0;
    if (p < L.total) {
      int i[3];
      i[0] = (int)(p % L.n[0]);
      i[1] = (int)((p / L.n[0]) % L.n[1]);
      i[2] = (int)(p / L.n01);
      const uint4 w = warp_info[p >> 5];
      const unsigned bits[3] = {w.x, w.y, w.z};
      const int l = (int)(p & 31);
      float p0[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) p0[c] = lattice_coord(L, c, i[c]);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (!((bits[a] >> l) & 1u)) continue;
        const long long id = vertex_id(warp_info, voff, p, a);
        if (id >= max_v) continue;
        const int64_t q1 = p + axis_stride(L, a);
        const float v0 = vol[p], v1 = vol[q1];
        const float t = edge_t(level, v0, v1);
        float x[3] = {p0[0], p0[1], p0[2]};
        x[a] = edge_coord(L, a, i[a], p0[a], t);
#pragma unroll
        for (int c = 0; c < 3; ++c) verts[3 * id + c] = x[c];
        if (dirs) {
          int j[3] = {i[0], i[1], i[2]};
          j[a] += 1;
          float g0[3], g1[3], d[3];
          lattice_grad(L, vol, p, i, g0);
          lattice_grad(L, vol, q1, j, g1);
          edge_dir(g0, g1, t, d);
#pragma unroll
          for (int c = 0; c < 3; ++c) dirs[3 * id + c] = d[c];
        }
      }
      if (i[0] + 1 < L.n[0] && i[1] + 1 < L.n[1] && i[2] + 1 < L.n[2]) {
        cs = cube_case(L, vol, p, level);
        tris = tri_count[cs];
      }
    }
    // the tile's exclusive prefix of triangle counts, in point order
    int inc = tris;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) wf[wid] = inc;
    __syncthreads();
    if (tris > 0) {
      int before = 0;
      for (int w = 0; w < wid; ++w) before += wf[w];
      const long long f0 = foff[tile] + before + inc - tris;
      for (int t = 0; t < tris && f0 + t < max_f; ++t) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int e = tri_edges[cs][3 * t + k];
          const int a = e >> 2, m = e & 3;
          // the edge's low corner: the cube's corner plus the bits of m on the other two axes, lower axis first
          const int u = a == 0 ? 1 : 0, v = a == 2 ? 1 : 2;
          const int64_t q = p + (m & 1) * axis_stride(L, u) + (m >> 1) * axis_stride(L, v);
          faces[3 * (f0 + t) + k] = (int)vertex_id(warp_info, voff, q, a);
        }
      }
    }
    __syncthreads();  // wf is rewritten by the next tile
  }
}

__global__ void mesh_lattice_points_kernel(const Lattice L, int z0, int64_t n, float* __restrict__ pts) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int x = (int)(k % L.n[0]), y = (int)((k / L.n[0]) % L.n[1]), z = z0 + (int)(k / L.n01);
  pts[3 * k + 0] = lattice_coord(L, 0, x);
  pts[3 * k + 1] = lattice_coord(L, 1, y);
  pts[3 * k + 2] = lattice_coord(L, 2, z);
}

int check_box(const nerfb200_grid_t* box, const char* what) {
  if (int rc = check_grid(box, what)) return rc;
  const Lattice L = make_lattice(*box);
  if (L.total > (int64_t(1) << 31)) {
    set_error("%s: %lld lattice points, more than 2^31", what, (long long)L.total);
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

}  // namespace

}  // namespace nerfb200

using namespace nerfb200;

extern "C" {

int64_t nerfb200_mesh_workspace_bytes(const nerfb200_grid_t* box) {
  if (check_box(box, "mesh_workspace_bytes") != NERFB200_OK) return -1;
  return workspace_layout(make_lattice(*box), nullptr).bytes;
}

int32_t nerfb200_mesh_lattice_points(const nerfb200_grid_t* box, int32_t z0, int32_t nz, float* pts, void* stream) {
  if (int rc = check_box(box, "mesh_lattice_points")) return rc;
  const Lattice L = make_lattice(*box);
  if (!pts || nz <= 0 || z0 < 0 || (int64_t)z0 + nz > L.n[2]) {
    set_error("mesh_lattice_points: null pointer or planes %d .. %d outside 0 .. %d", z0, z0 + nz - 1, L.n[2] - 1);
    return NERFB200_ERR_INVALID;
  }
  const int64_t n = L.n01 * nz;
  mesh_lattice_points_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(L, z0, n, pts);
  count_launch();
  return check_cuda(cudaGetLastError(), "mesh_lattice_points launch");
}

int32_t nerfb200_mesh_count(const nerfb200_grid_t* box, const float* volume, float level, void* workspace,
                            int64_t* totals, void* stream) {
  if (int rc = check_box(box, "mesh_count")) return rc;
  if (!volume || !workspace || !totals || !std::isfinite(level)) {
    set_error("mesh_count: null pointer or non-finite level");
    return NERFB200_ERR_INVALID;
  }
  const Lattice L = make_lattice(*box);
  const Workspace w = workspace_layout(L, workspace);
  const int64_t tiles = (L.total + kMeshThreads - 1) / kMeshThreads;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  mesh_classify_kernel<<<grid_for(tiles), kMeshThreads, 0, s>>>(L, volume, level, tiles, w.warp, w.tile_v, w.tile_f);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "mesh_classify launch")) return rc;
  mesh_scan_kernel<<<1, kMeshScanThreads, 0, s>>>(w.tile_v, w.tile_f, tiles, w.voff, w.foff,
                                                  reinterpret_cast<long long*>(totals));
  count_launch();
  return check_cuda(cudaGetLastError(), "mesh_scan launch");
}

int32_t nerfb200_mesh_emit(const nerfb200_grid_t* box, const float* volume, float level, const void* workspace,
                           int64_t max_vertices, int64_t max_faces, float* vertices, int32_t* faces, float* view_dirs,
                           void* stream) {
  if (int rc = check_box(box, "mesh_emit")) return rc;
  if (!volume || !workspace || !std::isfinite(level) || max_vertices < 0 || max_faces < 0 ||
      (max_vertices > 0 && !vertices) || (max_faces > 0 && !faces)) {
    set_error("mesh_emit: null pointer, negative size or non-finite level");
    return NERFB200_ERR_INVALID;
  }
  if (max_vertices > (int64_t(1) << 31)) {
    set_error("mesh_emit: %lld vertices do not fit int32 face indices", (long long)max_vertices);
    return NERFB200_ERR_UNSUPPORTED;
  }
  const Lattice L = make_lattice(*box);
  const Workspace w = workspace_layout(L, const_cast<void*>(workspace));
  const int64_t tiles = (L.total + kMeshThreads - 1) / kMeshThreads;
  mesh_emit_kernel<<<grid_for(tiles), kMeshThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      L, volume, level, tiles, w.warp, w.voff, w.foff, max_vertices, max_faces, vertices, faces, view_dirs);
  count_launch();
  return check_cuda(cudaGetLastError(), "mesh_emit launch");
}

}  // extern "C"
