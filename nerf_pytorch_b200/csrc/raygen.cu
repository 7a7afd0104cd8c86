// raygen.cu -- ray generation and packing for the render driver: one kernel instead of the reference's chain of
// small torch ops (and instead of materialising all H*W rays to pick 4096 of them, train_nerf.py:213-226):
//   get_ray_bundle   nerf/nerf_helpers.py:67-110   directions = [(i - W/2)/f, -(j - H/2)/f, -1] . R^T, origin = c2w[:3, 3]
//   viewdirs         nerf/train_utils.py:143-148   rd / ||rd||  (from the pre-NDC directions)
//   ndc_rays         nerf/nerf_helpers.py:170-197  (near plane 1.0, train_utils.py:157-160)
//   packing          nerf/train_utils.py:164-168   [ro(3) rd(3) near far viewdir(3)]
// Every fp32 operation is performed in the reference's order with explicit round-to-nearest intrinsics (no FMA
// contraction), so rows are bit-identical to the reference's wherever torch's own op order is defined (everything
// except the 3-term sums / the norm, which match the oracle to the last bit in practice and to 1 ulp by contract).
#include "common.cuh"

namespace nerfb200 {

struct RayGenArgs {
  float c2w[12];       // rows of the 3 x 4 camera-to-world matrix (gen mode)
  int height, width;
  float focal;
  float half_w, half_h;  // float32(W * 0.5), float32(H * 0.5) as the reference's python floats convert
  int ndc;             // apply ndc_rays(H, W, focal, 1.0, ...)
  float near, far;
  int use_viewdirs;
  int out_stride;      // 11, 8 (packed rows) or 6 (origin + direction only: get_ray_bundle)
};

__device__ __forceinline__ void finish_ray(const RayGenArgs& a, float ox, float oy, float oz, float dx, float dy, float dz,
                                           float* __restrict__ row) {
  float vx = 0.f, vy = 0.f, vz = 0.f;
  if (a.use_viewdirs) {  // viewdirs / viewdirs.norm(p=2, dim=-1)  -- from the directions BEFORE the NDC warp
    // torch's 2-norm accumulates x*x with fused multiply-adds in element order (checked against torch CPU: this form is
    // bit-identical on 200 000 random vectors, the unfused sum only on 89 %)
    const float n2 = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
    const float n = __fsqrt_rn(n2);
    vx = __fdiv_rn(dx, n); vy = __fdiv_rn(dy, n); vz = __fdiv_rn(dz, n);
  }
  if (a.ndc) {
    const float near = 1.0f;
    const float W = (float)a.width, H = (float)a.height;
    // t = -(near + o_z) / d_z;  o = o + t d
    const float t = __fdiv_rn(-__fadd_rn(near, oz), dz);
    ox = __fadd_rn(ox, __fmul_rn(t, dx));
    oy = __fadd_rn(oy, __fmul_rn(t, dy));
    oz = __fadd_rn(oz, __fmul_rn(t, dz));
    // -1 / (W / (2 f)): evaluated in double by python, applied as an fp32 scalar
    const float sw = (float)(-1.0 / ((double)W / (2.0 * (double)a.focal)));
    const float sh = (float)(-1.0 / ((double)H / (2.0 * (double)a.focal)));
    const float o0 = __fdiv_rn(__fmul_rn(sw, ox), oz);
    const float o1 = __fdiv_rn(__fmul_rn(sh, oy), oz);
    const float o2 = __fadd_rn(1.0f, __fdiv_rn(2.0f * near, oz));
    const float d0 = __fmul_rn(sw, __fadd_rn(__fdiv_rn(dx, dz), -__fdiv_rn(ox, oz)));
    const float d1 = __fmul_rn(sh, __fadd_rn(__fdiv_rn(dy, dz), -__fdiv_rn(oy, oz)));
    const float d2 = __fdiv_rn(-2.0f * near, oz);
    ox = o0; oy = o1; oz = o2; dx = d0; dy = d1; dz = d2;
  }
  row[0] = ox; row[1] = oy; row[2] = oz; row[3] = dx; row[4] = dy; row[5] = dz;
  if (a.out_stride >= 8) { row[6] = a.near; row[7] = a.far; }
  if (a.out_stride >= 11) { row[8] = vx; row[9] = vy; row[10] = vz; }
}

// the ray of pixel id = j * W + i of the camera with 3 x 4 camera-to-world rows c2w
__device__ __forceinline__ void pixel_ray(const RayGenArgs& a, const float* c2w, int64_t id, float* __restrict__ row) {
  const int j = (int)(id / a.width), i = (int)(id - (int64_t)j * a.width);
  const float c0 = __fdiv_rn(__fadd_rn((float)i, -a.half_w), a.focal);
  const float c1 = __fdiv_rn(-__fadd_rn((float)j, -a.half_h), a.focal);
  const float c2 = -1.0f;
  float d[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)  // sum(directions[..., None, :] * c2w[:3, :3], dim=-1)
    d[r] = __fadd_rn(__fadd_rn(__fmul_rn(c0, c2w[4 * r]), __fmul_rn(c1, c2w[4 * r + 1])), __fmul_rn(c2, c2w[4 * r + 2]));
  finish_ray(a, c2w[3], c2w[7], c2w[11], d[0], d[1], d[2], row);
}

// rays from (pose, pixel ids): pix[k] = j * W + i (row-major over the image), or all H*W pixels when pix == nullptr
__global__ void gen_rays_kernel(const __grid_constant__ RayGenArgs a, const int64_t* __restrict__ pix, int64_t n,
                                float* __restrict__ out) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    pixel_ray(a, a.c2w, pix ? pix[k] : k, out + k * a.out_stride);
}

// the same rays with the pose read on the device: entry *image of a [n_images][pose_rows][4] table (pose_rows 3 or 4)
__global__ void gen_rays_posed_kernel(const __grid_constant__ RayGenArgs a, const float* __restrict__ poses, int pose_rows,
                                      const int64_t* __restrict__ image, const int64_t* __restrict__ pix, int64_t n,
                                      float* __restrict__ out) {
  const float* pose = poses + *image * pose_rows * 4;
  float c2w[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) c2w[e] = pose[e];
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    pixel_ray(a, c2w, pix[k], out + k * a.out_stride);
}

// packing of caller-supplied origins / directions (the reference API: run_one_iter_of_nerf takes the two tensors)
__global__ void pack_rays_kernel(const __grid_constant__ RayGenArgs a, const float* __restrict__ ro,
                                 const float* __restrict__ rd, int64_t n, float* __restrict__ out) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    finish_ray(a, ro[3 * k], ro[3 * k + 1], ro[3 * k + 2], rd[3 * k], rd[3 * k + 1], rd[3 * k + 2], out + k * a.out_stride);
}

static int fill_args(RayGenArgs* a, const float* c2w12, int height, int width, float focal, int ndc, float near, float far,
                     int use_viewdirs, int out_stride) {
  if (height <= 0 || width <= 0 || !(focal > 0.f) || (out_stride != 6 && out_stride != 8 && out_stride != 11) ||
      (use_viewdirs && out_stride != 11)) {
    set_error("ray generation: invalid argument (H %d, W %d, focal %g, stride %d)", height, width, (double)focal, out_stride);
    return NERFB200_ERR_INVALID;
  }
  for (int i = 0; i < 12; ++i) a->c2w[i] = c2w12 ? c2w12[i] : 0.f;
  a->height = height; a->width = width; a->focal = focal;
  a->half_w = (float)((double)width * 0.5); a->half_h = (float)((double)height * 0.5);
  a->ndc = ndc; a->near = near; a->far = far; a->use_viewdirs = use_viewdirs; a->out_stride = out_stride;
  return NERFB200_OK;
}

int launch_gen_rays(const float* c2w12_host, int height, int width, float focal, const int64_t* pix, int64_t n, int ndc,
                    float near, float far, int use_viewdirs, int out_stride, float* out, cudaStream_t s) {
  RayGenArgs a;
  int rc = fill_args(&a, c2w12_host, height, width, focal, ndc, near, far, use_viewdirs, out_stride);
  if (rc) return rc;
  int64_t blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  gen_rays_kernel<<<(unsigned)blocks, 256, 0, s>>>(a, pix, n, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "gen_rays launch");
}

int launch_gen_rays_posed(const float* poses, int pose_rows, const int64_t* image, int height, int width, float focal,
                          const int64_t* pix, int64_t n, int ndc, float near, float far, int use_viewdirs, int out_stride,
                          float* out, cudaStream_t s) {
  RayGenArgs a;
  int rc = fill_args(&a, nullptr, height, width, focal, ndc, near, far, use_viewdirs, out_stride);
  if (rc) return rc;
  int64_t blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  gen_rays_posed_kernel<<<(unsigned)blocks, 256, 0, s>>>(a, poses, pose_rows, image, pix, n, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "gen_rays_posed launch");
}

int launch_pack_rays(const float* ro, const float* rd, int64_t n, int height, int width, float focal, int ndc, float near,
                     float far, int use_viewdirs, int out_stride, float* out, cudaStream_t s) {
  RayGenArgs a;
  int rc = fill_args(&a, nullptr, height, width, focal, ndc, near, far, use_viewdirs, out_stride);
  if (rc) return rc;
  int64_t blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  pack_rays_kernel<<<(unsigned)blocks, 256, 0, s>>>(a, ro, rd, n, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "pack_rays launch");
}

}  // namespace nerfb200
