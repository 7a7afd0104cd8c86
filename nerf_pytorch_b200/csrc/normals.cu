// normals.cu -- normal maps of a render's last pass (nerfb200.h "normal maps"): the samples the compositing gave a
// nonzero weight are compacted into a point list on the device (count, one-CTA scan, scatter: no atomics, no host
// read), density_grad_tc_kernel evaluates the gradient there reading the count from device memory, and a warp per ray
// sums w_i n_i in sample order.
#include "common.cuh"

namespace nerfb200 {

namespace {
constexpr int kNrmWarps = 8;     // rays per CTA of the per-ray kernels (a warp each)
constexpr int kScanThreads = 1024;

// count[r] = the samples of ray r with a nonzero weight
__global__ void __launch_bounds__(kNrmWarps * 32)
normal_count_kernel(const float* __restrict__ weights, int64_t n_rays, int S, int* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  const int64_t r = blockIdx.x * (int64_t)kNrmWarps + (threadIdx.x >> 5);
  if (r >= n_rays) return;
  int c = 0;
  for (int j0 = 0; j0 < S; j0 += 32) {
    const int j = j0 + lane;
    c += __popc(__ballot_sync(0xffffffffu, j < S && weights[r * S + j] != 0.f));
  }
  if (lane == 0) count[r] = c;
}

// first[r] = sum of count[r' < r], *total = the sum of all (one CTA: a contiguous run of rays per thread, then a
// shared-memory scan of the runs' sums)
__global__ void __launch_bounds__(kScanThreads)
normal_scan_kernel(const int* __restrict__ count, int64_t n_rays, int* __restrict__ first, int* __restrict__ total) {
  __shared__ int s[kScanThreads];
  const int t = threadIdx.x;
  const int64_t per = (n_rays + kScanThreads - 1) / kScanThreads;
  const int64_t r0 = t * per, r1 = min(n_rays, r0 + per);
  int sum = 0;
  for (int64_t r = r0; r < r1; ++r) sum += count[r];
  s[t] = sum;
  __syncthreads();
  for (int o = 1; o < kScanThreads; o <<= 1) {
    const int v = t >= o ? s[t - o] : 0;
    __syncthreads();
    s[t] += v;
    __syncthreads();
  }
  int run = s[t] - sum;  // exclusive
  for (int64_t r = r0; r < r1; ++r) {
    first[r] = run;
    run += count[r];
  }
  if (t == kScanThreads - 1) *total = s[t];
}

// pts[first[r] + k] = the point of ray r's k-th sample with a nonzero weight, o + d z as the MLP forms it
__global__ void __launch_bounds__(kNrmWarps * 32)
normal_scatter_kernel(const float* __restrict__ rays, int ray_stride, const float* __restrict__ z,
                      const float* __restrict__ weights, int64_t n_rays, int S, const int* __restrict__ first,
                      float* __restrict__ pts) {
  const int lane = threadIdx.x & 31;
  const int64_t r = blockIdx.x * (int64_t)kNrmWarps + (threadIdx.x >> 5);
  if (r >= n_rays) return;
  const float* rr = rays + r * ray_stride;
  int slot = first[r];
  for (int j0 = 0; j0 < S; j0 += 32) {
    const int j = j0 + lane;
    const bool on = j < S && weights[r * S + j] != 0.f;
    const uint32_t b = __ballot_sync(0xffffffffu, on);
    if (on) {
      const int k = slot + __popc(b & ((1u << lane) - 1u));
      const float zz = z[r * S + j];
#pragma unroll
      for (int c = 0; c < 3; ++c) pts[(int64_t)k * 3 + c] = __fadd_rn(rr[c], __fmul_rn(rr[3 + c], zz));
    }
    slot += __popc(b);
  }
}

// normals[r] = sum over the samples with a nonzero weight, in sample order, of w (-g / |g|) (0 where g = 0); kWorld maps
// each g by J^T at its NDC point pts[slot] first (nerfb200.h "NDC scenes")
template <bool kWorld>
__global__ void __launch_bounds__(kNrmWarps * 32)
normal_sum_kernel(const float* __restrict__ weights, int64_t n_rays, int S, const int* __restrict__ first,
                  const float* __restrict__ grad, float* __restrict__ normals, NdcMap m, const float* __restrict__ pts) {
  const int lane = threadIdx.x & 31;
  const int64_t r = blockIdx.x * (int64_t)kNrmWarps + (threadIdx.x >> 5);
  if (r >= n_rays) return;
  int slot = first[r];
  float N[3] = {0.f, 0.f, 0.f};
  for (int j0 = 0; j0 < S; j0 += 32) {
    const int j = j0 + lane;
    const float w = j < S ? weights[r * S + j] : 0.f;
    const bool on = w != 0.f;
    const uint32_t b = __ballot_sync(0xffffffffu, on);
    float t[3] = {0.f, 0.f, 0.f};  // w n of this lane's sample
    if (on) {
      const int k = slot + __popc(b & ((1u << lane) - 1u));
      float4 g = reinterpret_cast<const float4*>(grad)[k];
      if constexpr (kWorld) {
        const float q[3] = {pts[(int64_t)k * 3], pts[(int64_t)k * 3 + 1], pts[(int64_t)k * 3 + 2]};
        const float gn[3] = {g.y, g.z, g.w};
        float gw[3];
        ndc_grad_to_world(m, q, gn, gw);
        g.y = gw[0];
        g.z = gw[1];
        g.w = gw[2];
      }
      const float ss = __fadd_rn(__fadd_rn(__fmul_rn(g.y, g.y), __fmul_rn(g.z, g.z)), __fmul_rn(g.w, g.w));
      if (ss != 0.f) {
        const float len = __fsqrt_rn(ss);
        t[0] = __fmul_rn(w, -__fdiv_rn(g.y, len));
        t[1] = __fmul_rn(w, -__fdiv_rn(g.z, len));
        t[2] = __fmul_rn(w, -__fdiv_rn(g.w, len));
      }
    }
    // in sample order: every lane adds the 32 terms of this chunk one after the other
    for (uint32_t m = b; m; m &= m - 1) {
      const int src = __ffs(m) - 1;
#pragma unroll
      for (int c = 0; c < 3; ++c) N[c] = __fadd_rn(N[c], __shfl_sync(0xffffffffu, t[c], src));
    }
    slot += __popc(b);
  }
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < 3; ++c) normals[r * 3 + c] = N[c];
  }
}
}  // namespace

int launch_normal_compact(const float* rays, int ray_stride, const float* z, const float* weights, int64_t n_rays,
                          int n_samples, const NormalState& ns, cudaStream_t s) {
  const unsigned blocks = (unsigned)((n_rays + kNrmWarps - 1) / kNrmWarps);
  normal_count_kernel<<<blocks, kNrmWarps * 32, 0, s>>>(weights, n_rays, n_samples, ns.count);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "normal_count launch")) return rc;
  normal_scan_kernel<<<1, kScanThreads, 0, s>>>(ns.count, n_rays, ns.first, ns.total);
  count_launch();
  if (int rc = check_cuda(cudaGetLastError(), "normal_scan launch")) return rc;
  normal_scatter_kernel<<<blocks, kNrmWarps * 32, 0, s>>>(rays, ray_stride, z, weights, n_rays, n_samples, ns.first,
                                                          ns.pts);
  count_launch();
  return check_cuda(cudaGetLastError(), "normal_scatter launch");
}

int launch_normal_sum(const float* weights, int64_t n_rays, int n_samples, const NormalState& ns, float* normals,
                      cudaStream_t s, const NdcMap* world) {
  const unsigned blocks = (unsigned)((n_rays + kNrmWarps - 1) / kNrmWarps);
  if (world)
    normal_sum_kernel<true><<<blocks, kNrmWarps * 32, 0, s>>>(weights, n_rays, n_samples, ns.first, ns.grad, normals,
                                                              *world, ns.pts);
  else
    normal_sum_kernel<false><<<blocks, kNrmWarps * 32, 0, s>>>(weights, n_rays, n_samples, ns.first, ns.grad, normals,
                                                               NdcMap{0.f, 0.f}, nullptr);
  count_launch();
  return check_cuda(cudaGetLastError(), "normal_sum launch");
}

}  // namespace nerfb200
