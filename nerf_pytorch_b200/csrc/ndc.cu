// ndc.cu -- world-space geometry of forward-facing (NDC) scenes (nerfb200.h "NDC scenes"): meshes extracted in NDC mapped
// to world space, world points mapped to the NDC points the MLP encodes, and NDC density gradients mapped to world
// gradients.  Grid-stride loops, one element per thread and iteration; no atomics, no host synchronisation.
#include <math.h>

#include "common.cuh"

namespace nerfb200 {

namespace {
constexpr int kNdcThreads = 256;

unsigned ndc_blocks(int64_t n) {
  int64_t b = (n + kNdcThreads - 1) / kNdcThreads;
  const int64_t cap = (int64_t)device_sms() * 8;
  if (b > cap) b = cap;
  return (unsigned)(b > 0 ? b : 1);
}

// the header's unit world direction of v: v / sqrt(l) for 0 < l < inf, else (0, 0, 1)
__device__ __forceinline__ void unit_dir(const float v[3], float d[3]) {
  const float l = __fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2]));
  d[0] = 0.f;
  d[1] = 0.f;
  d[2] = 1.f;
  if (l > 0.f && l < INFINITY) {
    const float r = __fsqrt_rn(l);
#pragma unroll
    for (int c = 0; c < 3; ++c) d[c] = __fdiv_rn(v[c], r);
  }
}

// item i < n_vertices: vertex i (and its view direction); item i < n_faces: face i with its last two ids swapped
__global__ void __launch_bounds__(kNdcThreads)
ndc_mesh_to_world_kernel(NdcMap m, const float* vertices, const int32_t* faces, const float* view_dirs,
                         int64_t n_vertices, int64_t n_faces, float* world_vertices, int32_t* world_faces,
                         float* world_dirs) {
  const int64_t n = n_vertices > n_faces ? n_vertices : n_faces;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < n_vertices) {
      const float q[3] = {vertices[i * 3], vertices[i * 3 + 1], vertices[i * 3 + 2]};
      float p[3];
      ndc_inverse(m, q, p);
      if (world_dirs) {
        const float d[3] = {view_dirs[i * 3], view_dirs[i * 3 + 1], view_dirs[i * 3 + 2]};
        float g[3], u[3];
        ndc_grad_to_world(m, q, d, g);
        unit_dir(g, u);
#pragma unroll
        for (int c = 0; c < 3; ++c) world_dirs[i * 3 + c] = u[c];
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) world_vertices[i * 3 + c] = p[c];
    }
    if (i < n_faces) {
      const int32_t a = faces[i * 3], b = faces[i * 3 + 1], c = faces[i * 3 + 2];
      world_faces[i * 3] = a;
      world_faces[i * 3 + 1] = c;
      world_faces[i * 3 + 2] = b;
    }
  }
}

__global__ void __launch_bounds__(kNdcThreads)
ndc_from_world_kernel(NdcMap m, const float* __restrict__ p, int64_t n, float* __restrict__ q) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x[3] = {p[i * 3], p[i * 3 + 1], p[i * 3 + 2]};
    float y[3];
    ndc_forward(m, x, y);
#pragma unroll
    for (int c = 0; c < 3; ++c) q[i * 3 + c] = y[c];
  }
}

// rows and out may alias: each thread reads its row before writing it
__global__ void __launch_bounds__(kNdcThreads)
ndc_grad_to_world_kernel(NdcMap m, const float* __restrict__ q, const float* rows, int64_t n, float* out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 r = reinterpret_cast<const float4*>(rows)[i];
    const float x[3] = {q[i * 3], q[i * 3 + 1], q[i * 3 + 2]};
    const float g[3] = {r.y, r.z, r.w};
    float G[3];
    ndc_grad_to_world(m, x, g, G);
    reinterpret_cast<float4*>(out)[i] = make_float4(r.x, G[0], G[1], G[2]);
  }
}
}  // namespace

int make_ndc_map(const nerfb200_ndc_t* ndc, NdcMap* m, const char* what) {
  if (!ndc || ndc->height <= 0 || ndc->width <= 0 || !(ndc->focal > 0.f) || !isfinite(ndc->focal)) {
    set_error("%s: the NDC camera needs height, width > 0 and a finite focal > 0 (got %s)", what,
              ndc ? "a malformed camera" : "NULL");
    return NERFB200_ERR_INVALID;
  }
  // -1 / (W / (2 f)) in double, rounded once: raygen.cu finish_ray's sw / sh
  const double W = (double)(float)ndc->width, H = (double)(float)ndc->height, f = (double)ndc->focal;
  m->sw = (float)(-1.0 / (W / (2.0 * f)));
  m->sh = (float)(-1.0 / (H / (2.0 * f)));
  return NERFB200_OK;
}

int launch_ndc_mesh_to_world(const NdcMap& m, const float* vertices, const int32_t* faces, const float* view_dirs,
                             int64_t n_vertices, int64_t n_faces, float* world_vertices, int32_t* world_faces,
                             float* world_dirs, cudaStream_t s) {
  const int64_t n = n_vertices > n_faces ? n_vertices : n_faces;
  if (n == 0) return NERFB200_OK;
  ndc_mesh_to_world_kernel<<<ndc_blocks(n), kNdcThreads, 0, s>>>(m, vertices, faces, view_dirs, n_vertices, n_faces,
                                                                  world_vertices, world_faces, world_dirs);
  count_launch();
  return check_cuda(cudaGetLastError(), "ndc_mesh_to_world launch");
}

int launch_ndc_from_world(const NdcMap& m, const float* p, int64_t n, float* q, cudaStream_t s) {
  if (n == 0) return NERFB200_OK;
  ndc_from_world_kernel<<<ndc_blocks(n), kNdcThreads, 0, s>>>(m, p, n, q);
  count_launch();
  return check_cuda(cudaGetLastError(), "ndc_from_world launch");
}

int launch_ndc_grad_to_world(const NdcMap& m, const float* q, const float* rows, int64_t n, float* out, cudaStream_t s) {
  if (n == 0) return NERFB200_OK;
  ndc_grad_to_world_kernel<<<ndc_blocks(n), kNdcThreads, 0, s>>>(m, q, rows, n, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "ndc_grad_to_world launch");
}

}  // namespace nerfb200
