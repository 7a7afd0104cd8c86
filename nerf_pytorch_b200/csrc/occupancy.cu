// occupancy.cu -- sample compaction for occupancy-grid inference renders (include/nerfb200.h "occupancy grid").
// Three launches per pass, after the pass's depths exist and before its MLP:
//   mark     one CTA per group of kGridGroupRays consecutive rays: forms every sample's point as the MLP forward does,
//            looks its cell up, writes raw = [0 0 0 -inf] for a skipped sample and gives each evaluated sample its rank
//            among the group's evaluated samples (ballot + CTA prefix sum, in (ray, sample) order); the group's count.
//   scan     one CTA: exclusive prefix sum over the groups of their 64-row block counts -> each group's first block, the
//            block total and the evaluated total, both left in device memory.
//   scatter  one CTA per group: map[64 * first block + rank] = point, padding rows -1, and each block's first and last ray.
// No atomics: the map is a function of the inputs alone.
#include <cmath>

#include "common.cuh"

namespace nerfb200 {

namespace {

constexpr int kMarkThreads = 256;
constexpr int kScanThreads = 1024;

// The cell rule of nerfb200.h: cell index, or -1 outside the box.  Host and device evaluate the same fp32 operations.
__host__ __device__ inline int64_t grid_cell(const nerfb200_grid_t& g, const float x[3]) {
  int64_t idx = 0, mul = 1;
  for (int c = 0; c < 3; ++c) {
#ifdef __CUDA_ARCH__
    const float scale = __fdiv_rn((float)g.res[c], __fsub_rn(g.hi[c], g.lo[c]));
    const float t = __fmul_rn(__fsub_rn(x[c], g.lo[c]), scale);
#else
    const float scale = (float)g.res[c] / (g.hi[c] - g.lo[c]);
    const float t = (x[c] - g.lo[c]) * scale;
#endif
    if (!(t >= 0.f && t < (float)g.res[c])) return -1;
    idx += (int64_t)(int)t * mul;
    mul *= g.res[c];
  }
  return idx;
}

__device__ __forceinline__ int64_t group_end_ray(int64_t g, int64_t n_rays) {
  const int64_t e = (g + 1) * kGridGroupRays;
  return e < n_rays ? e : n_rays;
}

__global__ void __launch_bounds__(kMarkThreads)
grid_mark_kernel(const nerfb200_grid_t g, const uint32_t* __restrict__ bits, const float* __restrict__ rays,
                 int ray_stride, const float* __restrict__ z, int64_t n_rays, int S, float4* __restrict__ raw,
                 int* __restrict__ rank, int* __restrict__ counts) {
  __shared__ int warp_tot[kMarkThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t grp = blockIdx.x;
  const int64_t p_begin = grp * kGridGroupRays * S, p_end = group_end_ray(grp, n_rays) * S;
  int running = 0;
  for (int64_t base = p_begin; base < p_end; base += kMarkThreads) {
    const int64_t pt = base + tid;
    bool keep = false;
    if (pt < p_end) {
      const int64_t ray = pt / S;
      const float* rr = rays + ray * ray_stride;
      const float zz = z[pt];
      float x[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __fadd_rn(rr[c], __fmul_rn(rr[3 + c], zz));  // as the MLP prologue forms it
      const int64_t cell = grid_cell(g, x);
      keep = cell < 0 || ((bits[cell >> 5] >> (cell & 31)) & 1u);
      if (!keep) {
        raw[pt] = make_float4(0.f, 0.f, 0.f, -INFINITY);
        rank[pt] = -1;
      }
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_tot[warp] = __popc(ballot);
    __syncthreads();
    int before = running, total = 0;
#pragma unroll
    for (int w = 0; w < kMarkThreads / 32; ++w) {
      if (w < warp) before += warp_tot[w];
      total += warp_tot[w];
    }
    if (keep) rank[pt] = before + __popc(ballot & ((1u << lane) - 1u));
    running += total;
    __syncthreads();  // warp_tot is rewritten by the next round
  }
  if (tid == 0) counts[grp] = running;
}

// exclusive prefix sum of ceil(count / 64) over the groups, one CTA
__global__ void __launch_bounds__(kScanThreads)
grid_scan_kernel(const int* __restrict__ counts, int64_t n_groups, int* __restrict__ first_block,
                 int* __restrict__ n_blocks, int64_t* __restrict__ n_evaluated) {
  __shared__ int warp_sum[kScanThreads / 32];
  __shared__ long long warp_pts[kScanThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int carry = 0;
  long long pts = 0;
  for (int64_t base = 0; base < n_groups; base += kScanThreads) {
    const int64_t gi = base + tid;
    const int c = gi < n_groups ? counts[gi] : 0;
    const int nb = (c + 63) >> 6;
    int inc = nb;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    long long cp = c;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cp += __shfl_xor_sync(0xffffffffu, cp, o);
    if (lane == 31) warp_sum[warp] = inc;
    if (lane == 0) warp_pts[warp] = cp;
    __syncthreads();
    int before = carry, total = 0;
    long long round_pts = 0;
    for (int w = 0; w < kScanThreads / 32; ++w) {
      if (w < warp) before += warp_sum[w];
      total += warp_sum[w];
      round_pts += warp_pts[w];
    }
    if (gi < n_groups) first_block[gi] = before + inc - nb;
    carry += total;
    pts += round_pts;
    __syncthreads();
  }
  if (tid == 0) {
    *n_blocks = carry;
    if (n_evaluated) *n_evaluated = pts;
  }
}

__global__ void __launch_bounds__(kMarkThreads)
grid_scatter_kernel(const int* __restrict__ rank, const int* __restrict__ counts, const int* __restrict__ first_block,
                    int64_t n_rays, int S, int* __restrict__ map, int2* __restrict__ blocks) {
  const int64_t grp = blockIdx.x;
  const int64_t p_begin = grp * kGridGroupRays * S, p_end = group_end_ray(grp, n_rays) * S;
  const int cnt = counts[grp];
  const int64_t row0 = (int64_t)first_block[grp] * 64;
  int* bx = reinterpret_cast<int*>(blocks);
  for (int64_t pt = p_begin + threadIdx.x; pt < p_end; pt += kMarkThreads) {
    const int rk = rank[pt];
    if (rk < 0) continue;
    map[row0 + rk] = (int)pt;
    const int64_t b = first_block[grp] + (rk >> 6);
    if ((rk & 63) == 0) bx[2 * b] = (int)(pt / S);
    if ((rk & 63) == 63 || rk == cnt - 1) bx[2 * b + 1] = (int)(pt / S);
  }
  const int padded = (cnt + 63) & ~63;
  for (int r = cnt + (int)threadIdx.x; r < padded; r += kMarkThreads) map[row0 + r] = -1;
}

// ---- early ray termination (nerfb200.h "early ray termination"): one CTA per compaction group, one warp per ray ----
constexpr int kStopThreads = 32 * kGridGroupRays;

__device__ __forceinline__ int round_rows(int n_eval, int round) {
  const int left = n_eval - round * kStopRound;
  return left <= 0 ? 0 : left < kStopRound ? left : kStopRound;
}

// Each evaluated sample's place in its ray's order (ballots in sample order), the ray's count, T = 1, stop = S, and
// the group's rows in round 0.
__global__ void __launch_bounds__(kStopThreads)
stop_mark_kernel(const nerfb200_grid_t g, const uint32_t* __restrict__ bits, const float* __restrict__ rays,
                 int ray_stride, const float* __restrict__ z, int64_t n_rays, int S, float4* __restrict__ raw,
                 StopState st, int64_t* __restrict__ other_rows, int64_t other_value) {
  __shared__ int rows[kGridGroupRays];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * kGridGroupRays + w;
  int n = 0;
  if (r < n_rays) {
    const float* rr = rays + r * ray_stride;
    for (int j0 = 0; j0 < S; j0 += 32) {
      const int j = j0 + lane;
      bool keep = j < S;
      if (keep && bits) {
        const int64_t pt = r * S + j;
        const float zz = z[pt];
        float x[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) x[c] = __fadd_rn(rr[c], __fmul_rn(rr[3 + c], zz));  // as the MLP prologue forms it
        const int64_t cell = grid_cell(g, x);
        keep = cell < 0 || ((bits[cell >> 5] >> (cell & 31)) & 1u);
        if (!keep) raw[pt] = make_float4(0.f, 0.f, 0.f, -INFINITY);
      }
      const unsigned ballot = __ballot_sync(0xffffffffu, keep);
      if (keep) st.order[r * S + n + __popc(ballot & ((1u << lane) - 1u))] = j;
      n += __popc(ballot);
    }
    if (lane == 0) {
      st.n_eval[r] = n;
      st.T[r] = 1.f;
      if (st.stop) st.stop[r] = S;
    }
  }
  if (lane == 0) rows[w] = round_rows(n, 0);
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int i = 0; i < kGridGroupRays; ++i) total += rows[i];
    st.counts[blockIdx.x] = total;
    if (other_rows && blockIdx.x == 0) *other_rows = other_value;
  }
}

// Round k's rows of each live ray, in (ray, sample) order from the group's first block; padding rows -1, each block's
// first and last ray: the RowMap grid_scatter_kernel writes.
__global__ void __launch_bounds__(kStopThreads)
stop_scatter_kernel(StopState st, const int* __restrict__ first_block, int64_t n_rays, int S, int round,
                    int* __restrict__ map, int2* __restrict__ blocks) {
  __shared__ int rows[kGridGroupRays];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * kGridGroupRays + w;
  const int c = r < n_rays ? round_rows(st.n_eval[r], round) : 0;
  if (lane == 0) rows[w] = c;
  __syncthreads();
  int off = 0, cnt = 0;
#pragma unroll
  for (int i = 0; i < kGridGroupRays; ++i) {
    if (i < w) off += rows[i];
    cnt += rows[i];
  }
  const int fb = first_block[blockIdx.x];
  const int64_t row0 = (int64_t)fb * 64;
  int* bx = reinterpret_cast<int*>(blocks);
  const int* ord = st.order + r * S + round * kStopRound;
  for (int i = lane; i < c; i += 32) {
    const int rk = off + i;
    map[row0 + rk] = (int)(r * S + ord[i]);
    const int64_t b = fb + (rk >> 6);
    if ((rk & 63) == 0) bx[2 * b] = (int)r;
    if ((rk & 63) == 63 || rk == cnt - 1) bx[2 * b + 1] = (int)r;
  }
  const int padded = (cnt + 63) & ~63;
  for (int i = cnt + (int)threadIdx.x; i < padded; i += kStopThreads) map[row0 + i] = -1;
}

}  // namespace

int64_t stop_round_max_blocks(int64_t n_rays, int n_samples) {
  const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
  const int per_ray = n_samples < kStopRound ? n_samples : kStopRound;
  return groups * (((int64_t)kGridGroupRays * per_ray + 63) / 64);
}

int launch_stop_mark(const nerfb200_grid_t& g, const uint32_t* bits, const float* rays, int ray_stride, const float* z,
                     int64_t n_rays, int n_samples, float* raw, const StopState& st, int64_t* other_rows,
                     int64_t other_value, cudaStream_t s) {
  const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
  stop_mark_kernel<<<(unsigned)groups, kStopThreads, 0, s>>>(g, bits, rays, ray_stride, z, n_rays, n_samples,
                                                             reinterpret_cast<float4*>(raw), st, other_rows,
                                                             other_value);
  count_launch();
  return check_cuda(cudaGetLastError(), "stop_mark launch");
}

int launch_stop_scatter(const StopState& st, const int* first_block, int64_t n_rays, int n_samples, int round, int* map,
                        int* blocks, cudaStream_t s) {
  const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
  stop_scatter_kernel<<<(unsigned)groups, kStopThreads, 0, s>>>(st, first_block, n_rays, n_samples, round, map,
                                                                reinterpret_cast<int2*>(blocks));
  count_launch();
  return check_cuda(cudaGetLastError(), "stop_scatter launch");
}

int launch_grid_scan(const int* counts, int64_t n_groups, int* first_block, int* n_blocks, int64_t* n_rows,
                     cudaStream_t s) {
  grid_scan_kernel<<<1, kScanThreads, 0, s>>>(counts, n_groups, first_block, n_blocks, n_rows);
  count_launch();
  return check_cuda(cudaGetLastError(), "grid_scan launch");
}

int64_t grid_max_blocks(int64_t n_rays, int n_samples) {
  const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
  return groups * (((int64_t)kGridGroupRays * n_samples + 63) / 64);
}

int64_t grid_scratch_ints(int64_t n_rays, int n_samples) {
  const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
  return n_rays * n_samples + 2 * groups;
}

int check_grid(const nerfb200_grid_t* g, const char* what) {
  if (!g) {
    set_error("%s: null grid descriptor", what);
    return NERFB200_ERR_INVALID;
  }
  for (int c = 0; c < 3; ++c)
    if (!(g->res[c] >= 1 && g->res[c] <= NERFB200_GRID_MAX_RES) || !std::isfinite(g->lo[c]) ||
        !std::isfinite(g->hi[c]) || !(g->hi[c] > g->lo[c])) {
      set_error("%s: invalid grid (axis %d: res %d must be in 1..%d, lo %g < hi %g finite)", what, c, g->res[c],
                NERFB200_GRID_MAX_RES, g->lo[c], g->hi[c]);
      return NERFB200_ERR_INVALID;
    }
  return NERFB200_OK;
}

int launch_grid_compact(const nerfb200_grid_t& g, const uint32_t* bits, const float* rays, int ray_stride, const float* z,
                        int64_t n_rays, int n_samples, float* raw, int* map, int* blocks, int* n_blocks,
                        int64_t* n_evaluated, int* scratch, cudaStream_t s) {
  const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
  int* rank = scratch;
  int* counts = rank + n_rays * n_samples;
  int* first_block = counts + groups;
  grid_mark_kernel<<<(unsigned)groups, kMarkThreads, 0, s>>>(g, bits, rays, ray_stride, z, n_rays, n_samples,
                                                             reinterpret_cast<float4*>(raw), rank, counts);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "grid_mark launch")) return rc;
  grid_scan_kernel<<<1, kScanThreads, 0, s>>>(counts, groups, first_block, n_blocks, n_evaluated);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "grid_scan launch")) return rc;
  grid_scatter_kernel<<<(unsigned)groups, kMarkThreads, 0, s>>>(rank, counts, first_block, n_rays, n_samples, map,
                                                                reinterpret_cast<int2*>(blocks));
  count_launch();
  return check_cuda(cudaGetLastError(), "grid_scatter launch");
}

}  // namespace nerfb200

using namespace nerfb200;

extern "C" {

int64_t nerfb200_grid_words(const nerfb200_grid_t* grid) {
  if (check_grid(grid, "grid_words") != NERFB200_OK) return -1;
  const int64_t cells = (int64_t)grid->res[0] * grid->res[1] * grid->res[2];
  return (cells + 31) >> 5;
}

int32_t nerfb200_grid_locate(const nerfb200_grid_t* grid, const float* xyz_host, int64_t n, int64_t* cell_out) {
  if (int rc = check_grid(grid, "grid_locate")) return rc;
  if (!xyz_host || !cell_out || n < 0) {
    set_error("grid_locate: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  for (int64_t i = 0; i < n; ++i) cell_out[i] = grid_cell(*grid, xyz_host + 3 * i);
  return NERFB200_OK;
}

int64_t nerfb200_grid_max_blocks(int64_t n_rays, int32_t n_samples) {
  if (n_rays <= 0 || n_samples <= 0) return -1;
  return grid_max_blocks(n_rays, n_samples);
}

int64_t nerfb200_grid_scratch_ints(int64_t n_rays, int32_t n_samples) {
  if (n_rays <= 0 || n_samples <= 0) return -1;
  return grid_scratch_ints(n_rays, n_samples);
}

int32_t nerfb200_grid_compact(const nerfb200_grid_t* grid, const uint32_t* bits, const float* rays, int32_t ray_stride,
                              const float* z, int64_t n_rays, int32_t n_samples, float* raw, int32_t* map,
                              int32_t* blocks, int32_t* n_blocks, int64_t* n_evaluated, int32_t* scratch, void* stream) {
  if (int rc = check_grid(grid, "grid_compact")) return rc;
  if (!bits || !rays || !z || !raw || !map || !blocks || !n_blocks || !scratch || n_rays <= 0 || n_samples <= 0 ||
      ray_stride < 6) {
    set_error("grid_compact: null pointer, empty batch or ray_stride < 6");
    return NERFB200_ERR_INVALID;
  }
  if (n_rays * (int64_t)n_samples >= (int64_t(1) << 31)) {
    set_error("grid_compact: more than 2^31 points in one call; chunk the rays");
    return NERFB200_ERR_UNSUPPORTED;
  }
  return launch_grid_compact(*grid, bits, rays, ray_stride, z, n_rays, n_samples, raw, map, blocks, n_blocks,
                             n_evaluated, scratch, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
