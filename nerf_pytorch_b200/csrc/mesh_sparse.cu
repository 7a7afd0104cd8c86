// mesh_sparse.cu -- marching cubes over the occupied bricks of a lattice only (include/nerfb200.h "sparse meshes").
// The lattice is cut into bricks of kB^3 cubes.  Bricks:
//   cells     the grid's cell along each axis of every lattice coordinate (-1 outside the box): three short tables.
//   active    one thread per brick: its corners' axis cells from the tables (a corner outside the box makes the brick
//             active; otherwise each distinct cell the corners fall in is looked up); per tile of 256 bricks the
//             active count, as warp ballots.
//   scan      mesh_scan_kernel over the tile counts -> each tile's first slot.
//   compact   slot = tile offset + ballot rank: the brick map (brick -> slot, -1 inactive) and the list (slot -> brick).
// The caller evaluates its field at the active bricks' lattice points (sparse_points, brick-major), then, one CTA per
// active brick, looping over its (kB + 1)^3 corner points in three rounds of 256:
//   classify  each point's crossing edges that the brick owns, as warp ballots, and its cube's triangle count; per
//             32-point group the ballots and its first vertex relative to the brick, per brick its totals.
//   scan      mesh_scan_kernel over the brick totals -> each brick's first vertex and first face.
//   emit      the owned vertices, and the cubes' triangles.  An edge's owner is the lowest-index active brick with a cube
//             using it; the brick map finds the owner's slot, and its ballots the vertex id, as in mesh.cu.
// No atomics: the brick list and the mesh are functions of the grid, the field and the level.
#include <cmath>
#include <vector>

#include "mc_table.cuh"
#include "mesh_common.cuh"

namespace nerfb200 {

namespace {

constexpr int kB = NERFB200_MESH_BRICK;               // cubes per brick axis
constexpr int kBP = kB + 1;                           // corner points per brick axis
constexpr int kBrickPts = kBP * kBP * kBP;            // corner points per brick
constexpr int kGroups = (kBrickPts + 31) / 32;        // 32-point ballot groups per brick
constexpr int kSparseThreads = 256;
constexpr int kSparseWarps = kSparseThreads / 32;
constexpr int kRounds = (kBrickPts + kSparseThreads - 1) / kSparseThreads;
constexpr int kTileBricks = 256;                      // bricks per tile of the activity test, one per thread

// the bricks of a box and the layout of their values: brick-major, (p1)^3 points per brick with p1 = kB + 1 + 2 halo;
// corner point l (0 .. kB per axis) of slot s at s * pts + ((l2 + halo) * p1 + l1 + halo) * p1 + l0 + halo
struct Bricks {
  int nb[3];   // bricks per axis
  int halo;    // 0 or 1
  int p1;
  int64_t pts;
};

Bricks make_bricks(const nerfb200_grid_t& box, int halo) {
  Bricks K;
  for (int c = 0; c < 3; ++c) K.nb[c] = (box.res[c] + kB - 1) / kB;
  K.halo = halo;
  K.p1 = kBP + 2 * halo;
  K.pts = (int64_t)K.p1 * K.p1 * K.p1;
  return K;
}

inline int64_t brick_count(const Bricks& K) { return (int64_t)K.nb[0] * K.nb[1] * K.nb[2]; }

__host__ __device__ __forceinline__ void brick_coords(const Bricks& K, int b, int bc[3]) {
  bc[0] = b % K.nb[0];
  bc[1] = (b / K.nb[0]) % K.nb[1];
  bc[2] = b / (K.nb[0] * K.nb[1]);
}

__device__ __forceinline__ int value_index(const Bricks& K, int l0, int l1, int l2) {
  return ((l2 + K.halo) * K.p1 + l1 + K.halo) * K.p1 + l0 + K.halo;
}

// the grid's cell index along axis c of coordinate x, or -1 outside [lo, hi): the header's cell rule, per axis
__host__ __device__ __forceinline__ int axis_cell(const nerfb200_grid_t& g, int c, float x) {
#ifdef __CUDA_ARCH__
  const float scale = __fdiv_rn((float)g.res[c], __fsub_rn(g.hi[c], g.lo[c]));
  const float t = __fmul_rn(__fsub_rn(x, g.lo[c]), scale);
#else
  const float scale = (float)g.res[c] / (g.hi[c] - g.lo[c]);
  const float t = (x - g.lo[c]) * scale;
#endif
  return (t >= 0.f && t < (float)g.res[c]) ? (int)t : -1;
}

constexpr int kAxisMax = NERFB200_GRID_MAX_RES + 1;  // lattice indices per axis, at most

// axis_cells[c * kAxisMax + i] = the grid's cell along axis c of lattice coordinate p_c(i), or -1 outside the box
__host__ __device__ __forceinline__ int lattice_axis_cell(const Lattice& L, const nerfb200_grid_t& g, int c, int i) {
  return axis_cell(g, c, lattice_coord(L, c, i));
}

// The header's activity rule.  A point is outside the box when one of its coordinates is, and its cell is its three
// axis cells, so a brick whose corners are all inside falls in the product of each axis's cells; consecutive corners
// share cells, so each distinct cell is looked up once.
__host__ __device__ inline bool brick_active(const Lattice& L, const int* axis_cells, const nerfb200_grid_t& g,
                                             const uint32_t* bits, const int bc[3]) {
  int i0[3], i1[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    i0[c] = bc[c] * kB;
    i1[c] = i0[c] + kB < L.res[c] ? i0[c] + kB : L.res[c];
    for (int i = i0[c]; i <= i1[c]; ++i)
      if (axis_cells[c * kAxisMax + i] < 0) return true;
  }
  for (int k2 = i0[2], p2 = -1; k2 <= i1[2]; ++k2) {
    const int c2 = axis_cells[2 * kAxisMax + k2];
    if (c2 == p2) continue;
    p2 = c2;
    for (int k1 = i0[1], p1 = -1; k1 <= i1[1]; ++k1) {
      const int c1 = axis_cells[kAxisMax + k1];
      if (c1 == p1) continue;
      p1 = c1;
      for (int k0 = i0[0], p0 = -1; k0 <= i1[0]; ++k0) {
        const int c0 = axis_cells[k0];
        if (c0 == p0) continue;
        p0 = c0;
        const int64_t idx = ((int64_t)c2 * g.res[1] + c1) * g.res[0] + c0;
        if ((bits[idx >> 5] >> (idx & 31)) & 1u) return true;
      }
    }
  }
  return false;
}

__global__ void sparse_axis_cells_kernel(const Lattice L, const nerfb200_grid_t g, int* __restrict__ axis_cells) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    if (i <= L.res[c]) axis_cells[c * kAxisMax + i] = lattice_axis_cell(L, g, c, i);
}

__global__ void __launch_bounds__(kTileBricks)
sparse_active_kernel(const Lattice L, const nerfb200_grid_t g, const uint32_t* __restrict__ bits, const Bricks K,
                     int64_t n_bricks, const int* __restrict__ axis_cells, int* __restrict__ map,
                     int* __restrict__ tile_cnt) {
  __shared__ int wc[kTileBricks / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int64_t b = (int64_t)blockIdx.x * kTileBricks + tid;
  bool act = false;
  if (b < n_bricks) {
    int bc[3];
    brick_coords(K, (int)b, bc);
    act = brick_active(L, axis_cells, g, bits, bc);
    map[b] = act ? 1 : 0;
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, act);
  if (lane == 0) wc[wid] = __popc(ballot);
  __syncthreads();
  if (tid == 0) {
    int n = 0;
    for (int w = 0; w < kTileBricks / 32; ++w) n += wc[w];
    tile_cnt[blockIdx.x] = n;
  }
}

__global__ void __launch_bounds__(kTileBricks)
sparse_compact_kernel(int64_t n_bricks, const long long* __restrict__ tile_off, const long long* __restrict__ totals,
                      int* __restrict__ map, int* __restrict__ bricks, int64_t* __restrict__ n_active) {
  __shared__ int wc[kTileBricks / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int64_t b = (int64_t)blockIdx.x * kTileBricks + tid;
  const bool act = b < n_bricks && map[b] == 1;
  const unsigned ballot = __ballot_sync(0xffffffffu, act);
  if (lane == 0) wc[wid] = __popc(ballot);
  __syncthreads();
  int before = 0;
  for (int w = 0; w < wid; ++w) before += wc[w];
  if (b < n_bricks) {
    const long long slot = tile_off[blockIdx.x] + before + __popc(ballot & ((1u << lane) - 1u));
    map[b] = act ? (int)slot : -1;
    if (act) bricks[slot] = (int)b;
  }
  if (blockIdx.x == 0 && tid == 0) *n_active = totals[0];
}

__global__ void sparse_points_kernel(const Lattice L, const Bricks K, const int* __restrict__ bricks, int64_t first,
                                     int64_t n, float* __restrict__ pts) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int64_t slot = first + k / K.pts;
  const int lp = (int)(k % K.pts);
  const int l[3] = {lp % K.p1, (lp / K.p1) % K.p1, lp / (K.p1 * K.p1)};
  int bc[3];
  brick_coords(K, bricks[slot], bc);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int i = bc[c] * kB + l[c] - K.halo;
    i = i < 0 ? 0 : (i > L.res[c] ? L.res[c] : i);  // points past the lattice are never read; keep them on it
    pts[3 * k + c] = lattice_coord(L, c, i);
  }
}

// the lowest-index active brick with a cube that uses lattice edge (q, a): those cubes are q less 0 or 1 along each of
// the other two axes; -1 when none of their bricks is active
__device__ __forceinline__ int edge_owner(const Lattice& L, const Bricks& K, const int* __restrict__ map, const int q[3],
                                          int a) {
  const int u = a == 0 ? 1 : 0;
  int best = -1;
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    int bc[3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int cq = q[c] - (c == a ? 0 : (c == u ? (d & 1) : (d >> 1)));
      ok = ok && cq >= 0 && cq < L.res[c];
      bc[c] = cq / kB;
    }
    if (!ok) continue;
    const int idx = (bc[2] * K.nb[1] + bc[1]) * K.nb[0] + bc[0];
    if ((best < 0 || idx < best) && map[idx] >= 0) best = idx;
  }
  return best;
}

// id of the vertex on the edge along axis a from corner point lp of slot s, which owns it and where it crosses
__device__ __forceinline__ long long sparse_vertex_id(const uint4* __restrict__ ginfo, const long long* __restrict__ voff,
                                                      int64_t s, int lp, int a) {
  const uint4 w = ginfo[s * kGroups + (lp >> 5)];
  const int l = lp & 31;
  const unsigned below = (1u << l) - 1u;
  long long id = voff[s] + (long long)w.w + __popc(w.x & below) + __popc(w.y & below) + __popc(w.z & below);
  if (a >= 1) id += (w.x >> l) & 1u;
  if (a >= 2) id += (w.y >> l) & 1u;
  return id;
}

__device__ __forceinline__ int sparse_case(const Bricks& K, const float* __restrict__ vb, const int l[3], float level) {
  int cs = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) cs |= (vb[value_index(K, l[0] + (c & 1), l[1] + ((c >> 1) & 1), l[2] + (c >> 2))] > level
                                         ? 1 : 0) << c;
  return cs;
}

// the header's gradient at lattice point q, corner l of the brick whose values vb holds (with the halo)
__device__ __forceinline__ void sparse_grad(const Lattice& L, const Bricks& K, const float* __restrict__ vb,
                                            const int l[3], const int q[3], float g[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int lo = q[c] > 0 ? q[c] - 1 : 0, hi = q[c] + 1 < L.n[c] ? q[c] + 1 : L.n[c] - 1;
    int lh[3] = {l[0], l[1], l[2]}, ll[3] = {l[0], l[1], l[2]};
    lh[c] += hi - q[c];
    ll[c] += lo - q[c];
    g[c] = grad_component(L, c, vb[value_index(K, lh[0], lh[1], lh[2])], vb[value_index(K, ll[0], ll[1], ll[2])], hi,
                          lo);
  }
}

// corner point lp of brick bc: its local (l) and lattice (q) indices, and whether it is a lattice point
__device__ __forceinline__ bool corner(const Lattice& L, const int bc[3], int lp, int l[3], int q[3]) {
  l[0] = lp % kBP;
  l[1] = (lp / kBP) % kBP;
  l[2] = lp / (kBP * kBP);
  bool ok = lp < kBrickPts;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    q[c] = bc[c] * kB + l[c];
    ok = ok && q[c] <= L.res[c];
  }
  return ok;
}

__device__ __forceinline__ bool has_cube(const Lattice& L, const int l[3], const int q[3]) {
  return l[0] < kB && l[1] < kB && l[2] < kB && q[0] < L.res[0] && q[1] < L.res[1] && q[2] < L.res[2];
}

__global__ void __launch_bounds__(kSparseThreads)
sparse_classify_kernel(const Lattice L, const Bricks K, const int* __restrict__ map, const int* __restrict__ bricks,
                       int64_t n_active, const float* __restrict__ vals, float level, uint4* __restrict__ ginfo,
                       int* __restrict__ brick_v, int* __restrict__ brick_f) {
  __shared__ unsigned char tri_count[256];
  __shared__ int wv[kSparseWarps], wf[kSparseWarps];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int k = tid; k < 256; k += kSparseThreads) tri_count[k] = kMcTriCount[k];
  __syncthreads();
  for (int64_t s = blockIdx.x; s < n_active; s += gridDim.x) {
    const int b = bricks[s];
    int bc[3];
    brick_coords(K, b, bc);
    const float* vb = vals + s * K.pts;
    int run_v = 0, run_f = 0;
    for (int r = 0; r < kRounds; ++r) {
      const int lp = r * kSparseThreads + tid;
      int l[3], q[3];
      unsigned flags = 0;
      int tris = 0;
      if (corner(L, bc, lp, l, q)) {
        const bool in0 = vb[value_index(K, l[0], l[1], l[2])] > level;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          if (l[a] == kB || q[a] == L.res[a]) continue;
          int m[3] = {l[0], l[1], l[2]};
          m[a] += 1;
          if (in0 == (vb[value_index(K, m[0], m[1], m[2])] > level)) continue;
          const int u = a == 0 ? 1 : 0, v = a == 2 ? 1 : 2;
          // an edge off the brick's low faces on both other axes is used by this brick's cubes and later bricks' only
          if ((l[u] > 0 && l[v] > 0) || edge_owner(L, K, map, q, a) == b) flags |= 1u << a;
        }
        if (has_cube(L, l, q)) tris = tri_count[sparse_case(K, vb, l, level)];
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
      int before = run_v;
      for (int w = 0; w < kSparseWarps; ++w) {
        if (w < wid) before += wv[w];
        run_v += wv[w];
        run_f += wf[w];
      }
      const int grp = r * kSparseWarps + wid;
      if (lane == 0 && grp < kGroups) ginfo[s * kGroups + grp] = make_uint4(bx, by, bz, (unsigned)before);
      __syncthreads();  // wv / wf are rewritten by the next round
    }
    if (tid == 0) {
      brick_v[s] = run_v;
      brick_f[s] = run_f;
    }
  }
}

__global__ void __launch_bounds__(kSparseThreads)
sparse_emit_kernel(const Lattice L, const Bricks K, const int* __restrict__ map, const int* __restrict__ bricks,
                   int64_t n_active, const float* __restrict__ vals, float level, const uint4* __restrict__ ginfo,
                   const long long* __restrict__ voff, const long long* __restrict__ foff, int64_t max_v,
                   int64_t max_f, float* __restrict__ verts, int* __restrict__ faces, float* __restrict__ dirs,
                   int64_t* __restrict__ keys) {
  __shared__ unsigned char tri_count[256];
  __shared__ signed char tri_edges[256][3 * NERFB200_MC_MAX_TRIS];
  __shared__ int wf[kSparseWarps];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int k = tid; k < 256; k += kSparseThreads) tri_count[k] = kMcTriCount[k];
  for (int k = tid; k < 256 * 3 * NERFB200_MC_MAX_TRIS; k += kSparseThreads)
    (&tri_edges[0][0])[k] = (&kMcTris[0][0])[k];
  __syncthreads();
  for (int64_t s = blockIdx.x; s < n_active; s += gridDim.x) {
    int bc[3];
    brick_coords(K, bricks[s], bc);
    const float* vb = vals + s * K.pts;
    int run_f = 0;
    for (int r = 0; r < kRounds; ++r) {
      const int lp = r * kSparseThreads + tid;
      int l[3], q[3];
      int cs = 0, tris = 0;
      if (corner(L, bc, lp, l, q)) {
        const uint4 w = ginfo[s * kGroups + (lp >> 5)];
        const unsigned bits[3] = {w.x, w.y, w.z};
        const int ln = lp & 31;
        float p0[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) p0[c] = lattice_coord(L, c, q[c]);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          if (!((bits[a] >> ln) & 1u)) continue;
          const long long id = sparse_vertex_id(ginfo, voff, s, lp, a);
          if (id >= max_v) continue;
          int m[3] = {l[0], l[1], l[2]};
          m[a] += 1;
          const float v0 = vb[value_index(K, l[0], l[1], l[2])], v1 = vb[value_index(K, m[0], m[1], m[2])];
          const float t = edge_t(level, v0, v1);
          float x[3] = {p0[0], p0[1], p0[2]};
          x[a] = edge_coord(L, a, q[a], p0[a], t);
#pragma unroll
          for (int c = 0; c < 3; ++c) verts[3 * id + c] = x[c];
          if (keys) keys[id] = (((int64_t)q[2] * L.n[1] + q[1]) * L.n[0] + q[0]) * 3 + a;
          if (dirs) {
            int j[3] = {q[0], q[1], q[2]};
            j[a] += 1;
            float g0[3], g1[3], d[3];
            sparse_grad(L, K, vb, l, q, g0);
            sparse_grad(L, K, vb, m, j, g1);
            edge_dir(g0, g1, t, d);
#pragma unroll
            for (int c = 0; c < 3; ++c) dirs[3 * id + c] = d[c];
          }
        }
        if (has_cube(L, l, q)) {
          cs = sparse_case(K, vb, l, level);
          tris = tri_count[cs];
        }
      }
      // the brick's exclusive prefix of triangle counts, in cube order
      int inc = tris;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
      }
      if (lane == 31) wf[wid] = inc;
      __syncthreads();
      int before = run_f;
      for (int w = 0; w < kSparseWarps; ++w) {
        if (w < wid) before += wf[w];
        run_f += wf[w];
      }
      if (tris > 0) {
        const long long f0 = foff[s] + before + inc - tris;
        for (int t = 0; t < tris && f0 + t < max_f; ++t) {
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int e = tri_edges[cs][3 * t + k];
            const int a = e >> 2, m = e & 3;
            // the edge's low corner: the cube's corner plus the bits of m on the other two axes, lower axis first
            const int qe[3] = {q[0] + (a != 0 ? (m & 1) : 0), q[1] + (a == 0 ? (m & 1) : (a == 2 ? (m >> 1) : 0)),
                               q[2] + (a != 2 ? (m >> 1) : 0)};
            const int o = edge_owner(L, K, map, qe, a);  // this brick uses the edge, so o >= 0
            int oc[3];
            brick_coords(K, o, oc);
            const int olp = ((qe[2] - oc[2] * kB) * kBP + qe[1] - oc[1] * kB) * kBP + qe[0] - oc[0] * kB;
            faces[3 * (f0 + t) + k] = (int)sparse_vertex_id(ginfo, voff, map[o], olp, a);
          }
        }
      }
      __syncthreads();  // wf is rewritten by the next round
    }
  }
}

struct Workspace {
  uint4* ginfo;      // per brick and 32-point group: +x, +y, +z owned crossing ballots, first vertex in the brick
  int* brick_v;      // per brick: vertices, faces
  int* brick_f;
  long long* voff;   // per brick: first vertex, first face
  long long* foff;
  int64_t bytes;
};

inline int64_t align16(int64_t b) { return (b + 15) & ~int64_t(15); }

Workspace workspace_layout(int64_t n_active, void* base) {
  char* p = static_cast<char*>(base);
  Workspace w;
  int64_t off = 0;
  w.ginfo = reinterpret_cast<uint4*>(p + off);
  off += align16(n_active * kGroups * (int64_t)sizeof(uint4));
  w.brick_v = reinterpret_cast<int*>(p + off);
  off += align16(n_active * 4);
  w.brick_f = reinterpret_cast<int*>(p + off);
  off += align16(n_active * 4);
  w.voff = reinterpret_cast<long long*>(p + off);
  off += align16(n_active * 8);
  w.foff = reinterpret_cast<long long*>(p + off);
  off += align16(n_active * 8);
  w.bytes = off;
  return w;
}

struct Scratch {
  int* axis_cells;     // [3][kAxisMax]
  int* tile_cnt;       // per tile of bricks: active bricks
  long long* tile_off; // per tile: first slot
  long long* unused;   // the scan's second column
  long long* totals;   // [2]
  int64_t bytes;
};

Scratch scratch_layout(int64_t n_bricks, void* base) {
  const int64_t tiles = (n_bricks + kTileBricks - 1) / kTileBricks;
  char* p = static_cast<char*>(base);
  Scratch w;
  int64_t off = 0;
  w.axis_cells = reinterpret_cast<int*>(p + off);
  off += align16(3 * kAxisMax * 4);
  w.tile_cnt = reinterpret_cast<int*>(p + off);
  off += align16(tiles * 4);
  w.tile_off = reinterpret_cast<long long*>(p + off);
  off += align16(tiles * 8);
  w.unused = reinterpret_cast<long long*>(p + off);
  off += align16(tiles * 8);
  w.totals = reinterpret_cast<long long*>(p + off);
  off += align16(2 * 8);
  w.bytes = off;
  return w;
}

int check_sparse(const nerfb200_grid_t* box, const nerfb200_grid_t* grid, bool need_grid, const char* what) {
  if (int rc = check_grid(box, what)) return rc;
  if (need_grid)
    if (int rc = check_grid(grid, what)) return rc;
  return NERFB200_OK;
}

// the arguments count and emit share
int check_bricks(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks, int64_t n_active,
                 const float* values, int32_t halo, float level, const char* what) {
  if (int rc = check_grid(box, what)) return rc;
  const int64_t n_bricks = brick_count(make_bricks(*box, 0));
  if (!brick_map || (n_active > 0 && (!bricks || !values)) || n_active < 0 || n_active > n_bricks ||
      (halo != 0 && halo != 1) || !std::isfinite(level)) {
    set_error("%s: null pointer, %lld active bricks of %lld, halo %d or non-finite level", what, (long long)n_active,
              (long long)n_bricks, halo);
    return NERFB200_ERR_INVALID;
  }
  return NERFB200_OK;
}

}  // namespace

}  // namespace nerfb200

using namespace nerfb200;

extern "C" {

int32_t nerfb200_mesh_brick(void) { return kB; }

int64_t nerfb200_mesh_sparse_brick_count(const nerfb200_grid_t* box) {
  if (check_grid(box, "mesh_sparse_brick_count") != NERFB200_OK) return -1;
  return brick_count(make_bricks(*box, 0));
}

int64_t nerfb200_mesh_sparse_scratch_bytes(const nerfb200_grid_t* box) {
  if (check_grid(box, "mesh_sparse_scratch_bytes") != NERFB200_OK) return -1;
  return scratch_layout(brick_count(make_bricks(*box, 0)), nullptr).bytes;
}

int64_t nerfb200_mesh_sparse_workspace_bytes(const nerfb200_grid_t* box, int64_t n_active) {
  if (check_grid(box, "mesh_sparse_workspace_bytes") != NERFB200_OK) return -1;
  if (n_active < 0 || n_active > brick_count(make_bricks(*box, 0))) return -1;
  return workspace_layout(n_active, nullptr).bytes;
}

int32_t nerfb200_mesh_sparse_bricks(const nerfb200_grid_t* box, const nerfb200_grid_t* grid, const uint32_t* bits,
                                    int32_t* brick_map, int32_t* bricks, int64_t* n_active, void* scratch,
                                    void* stream) {
  if (int rc = check_sparse(box, grid, true, "mesh_sparse_bricks")) return rc;
  if (!bits || !brick_map || !bricks || !n_active || !scratch) {
    set_error("mesh_sparse_bricks: null pointer");
    return NERFB200_ERR_INVALID;
  }
  const Lattice L = make_lattice(*box);
  const Bricks K = make_bricks(*box, 0);
  const int64_t n = brick_count(K), tiles = (n + kTileBricks - 1) / kTileBricks;
  const Scratch w = scratch_layout(n, scratch);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  sparse_axis_cells_kernel<<<(kAxisMax + 255) / 256, 256, 0, s>>>(L, *grid, w.axis_cells);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "mesh_sparse_axis_cells launch")) return rc;
  sparse_active_kernel<<<(unsigned)tiles, kTileBricks, 0, s>>>(L, *grid, bits, K, n, w.axis_cells, brick_map,
                                                               w.tile_cnt);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "mesh_sparse_active launch")) return rc;
  mesh_scan_kernel<<<1, kMeshScanThreads, 0, s>>>(w.tile_cnt, w.tile_cnt, tiles, w.tile_off, w.unused, w.totals);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "mesh_sparse_scan launch")) return rc;
  sparse_compact_kernel<<<(unsigned)tiles, kTileBricks, 0, s>>>(n, w.tile_off, w.totals, brick_map, bricks, n_active);
  count_launch();
  return check_cuda(cudaGetLastError(), "mesh_sparse_compact launch");
}

int32_t nerfb200_mesh_sparse_bricks_host(const nerfb200_grid_t* box, const nerfb200_grid_t* grid,
                                         const uint32_t* bits_host, uint8_t* active_host) {
  if (int rc = check_sparse(box, grid, true, "mesh_sparse_bricks_host")) return rc;
  if (!bits_host || !active_host) {
    set_error("mesh_sparse_bricks_host: null pointer");
    return NERFB200_ERR_INVALID;
  }
  const Lattice L = make_lattice(*box);
  const Bricks K = make_bricks(*box, 0);
  const int64_t n = brick_count(K);
  std::vector<int> axis_cells(3 * kAxisMax);
  for (int c = 0; c < 3; ++c)
    for (int i = 0; i <= L.res[c]; ++i) axis_cells[c * kAxisMax + i] = lattice_axis_cell(L, *grid, c, i);
  for (int64_t b = 0; b < n; ++b) {
    int bc[3];
    brick_coords(K, (int)b, bc);
    active_host[b] = brick_active(L, axis_cells.data(), *grid, bits_host, bc) ? 1 : 0;
  }
  return NERFB200_OK;
}

int32_t nerfb200_mesh_sparse_points(const nerfb200_grid_t* box, const int32_t* bricks, int64_t first, int64_t count,
                                    int32_t halo, float* pts, void* stream) {
  if (int rc = check_grid(box, "mesh_sparse_points")) return rc;
  const Bricks K = make_bricks(*box, halo == 1 ? 1 : 0);
  if (!bricks || !pts || first < 0 || count <= 0 || first + count > brick_count(K) || (halo != 0 && halo != 1)) {
    set_error("mesh_sparse_points: null pointer, halo %d or bricks %lld .. %lld", halo, (long long)first,
              (long long)(first + count - 1));
    return NERFB200_ERR_INVALID;
  }
  const int64_t n = count * K.pts;
  sparse_points_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      make_lattice(*box), K, bricks, first, n, pts);
  count_launch();
  return check_cuda(cudaGetLastError(), "mesh_sparse_points launch");
}

int32_t nerfb200_mesh_sparse_count(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                   int64_t n_active, const float* values, int32_t halo, float level, void* workspace,
                                   int64_t* totals, void* stream) {
  if (int rc = check_bricks(box, brick_map, bricks, n_active, values, halo, level, "mesh_sparse_count")) return rc;
  if (!workspace || !totals) {
    set_error("mesh_sparse_count: null workspace or totals");
    return NERFB200_ERR_INVALID;
  }
  const Workspace w = workspace_layout(n_active, workspace);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n_active > 0) {
    sparse_classify_kernel<<<grid_for(n_active), kSparseThreads, 0, s>>>(make_lattice(*box), make_bricks(*box, halo),
                                                                          brick_map, bricks, n_active, values, level,
                                                                          w.ginfo, w.brick_v, w.brick_f);
    count_launch();
    if (int rc = check_cuda(cudaGetLastError(), "mesh_sparse_classify launch")) return rc;
  }
  mesh_scan_kernel<<<1, kMeshScanThreads, 0, s>>>(w.brick_v, w.brick_f, n_active, w.voff, w.foff,
                                                  reinterpret_cast<long long*>(totals));
  count_launch();
  return check_cuda(cudaGetLastError(), "mesh_sparse_scan launch");
}

int32_t nerfb200_mesh_sparse_emit(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                  int64_t n_active, const float* values, int32_t halo, float level,
                                  const void* workspace, int64_t max_vertices, int64_t max_faces, float* vertices,
                                  int32_t* faces, float* view_dirs, int64_t* edge_keys, void* stream) {
  if (int rc = check_bricks(box, brick_map, bricks, n_active, values, halo, level, "mesh_sparse_emit")) return rc;
  if (!workspace || max_vertices < 0 || max_faces < 0 || (max_vertices > 0 && !vertices) ||
      (max_faces > 0 && !faces) || (view_dirs && !halo)) {
    set_error("mesh_sparse_emit: null pointer, negative size, or view directions without the halo");
    return NERFB200_ERR_INVALID;
  }
  if (max_vertices > (int64_t(1) << 31)) {
    set_error("mesh_sparse_emit: %lld vertices do not fit int32 face indices", (long long)max_vertices);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (n_active == 0) return NERFB200_OK;
  const Workspace w = workspace_layout(n_active, const_cast<void*>(workspace));
  sparse_emit_kernel<<<grid_for(n_active), kSparseThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      make_lattice(*box), make_bricks(*box, halo), brick_map, bricks, n_active, values, level, w.ginfo, w.voff,
      w.foff, max_vertices, max_faces, vertices, faces, view_dirs, edge_keys);
  count_launch();
  return check_cuda(cudaGetLastError(), "mesh_sparse_emit launch");
}

}  // extern "C"
