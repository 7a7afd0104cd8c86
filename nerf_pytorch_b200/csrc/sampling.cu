// sampling.cu -- the HBM-bound per-ray stages around the MLP:
//   * stratified depth sampling                nerf/train_utils.py:45-65
//   * positional encoding (stand-alone hook)   nerf/nerf_helpers.py:113-157
//   * inverse-CDF resampling + sorted merge    nerf/nerf_helpers.py:260-302, train_utils.py:96-105
//   * weight packing and the fused Adam step   (host plumbing; train_nerf.py:136-141,261-270)
// Arithmetic that the reference performs as separate torch ops is written with the _rn
// intrinsics so that nvcc cannot contract mul+add into FMA: the results are then the same
// IEEE operations the reference executes.
#include <math_constants.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace nerfb200 {

// ---------------------------------------------------------------------------------------------
// stratified z
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float coarse_depth(float near, float far, float t, int lindisp) {
  const float omt = __fsub_rn(1.0f, t);
  if (!lindisp) return __fadd_rn(__fmul_rn(near, omt), __fmul_rn(far, t));
  const float a = __fmul_rn(__fdiv_rn(1.0f, near), omt);
  const float b = __fmul_rn(__fdiv_rn(1.0f, far), t);
  return __fdiv_rn(1.0f, __fadd_rn(a, b));
}

__global__ void sample_coarse_kernel(const float* __restrict__ rays, int ray_stride, int64_t n_rays,
                                     const RandSrc t_rand, int nc, int perturb, int lindisp, float* __restrict__ z) {
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= n_rays * nc) return;
  const int64_t r = idx / nc;
  const int i = (int)(idx - r * nc);
  const float near = rays[r * ray_stride + 6], far = rays[r * ray_stride + 7];
  const float zi = coarse_depth(near, far, linspace01(i, nc), lindisp);
  if (!perturb) {
    z[idx] = zi;
    return;
  }
  float upper = zi, lower = zi;
  if (i + 1 < nc) upper = __fmul_rn(0.5f, __fadd_rn(coarse_depth(near, far, linspace01(i + 1, nc), lindisp), zi));
  if (i > 0) lower = __fmul_rn(0.5f, __fadd_rn(zi, coarse_depth(near, far, linspace01(i - 1, nc), lindisp)));
  z[idx] = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), t_rand.uniform(r, i)));
}

int launch_sample_coarse(const float* rays, int ray_stride, int64_t n_rays, const RandSrc& t_rand, int n_coarse,
                         int perturb, int lindisp, float* z, cudaStream_t s) {
  const int64_t total = n_rays * n_coarse;
  const int threads = 256;
  const int64_t blocks = (total + threads - 1) / threads;
  sample_coarse_kernel<<<(unsigned)blocks, threads, 0, s>>>(rays, ray_stride, n_rays, t_rand, n_coarse, perturb,
                                                            lindisp, z);
  count_launch();
  return check_cuda(cudaGetLastError(), "sample_coarse launch");
}

// ---------------------------------------------------------------------------------------------
// a seeded stream written out (nerfb200_random_fill): the same RandSrc calls the render kernels make
// ---------------------------------------------------------------------------------------------
__global__ void random_fill_kernel(const RandSrc src, int normal, int64_t n_rays, int per_ray, float* __restrict__ out) {
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= n_rays * per_ray) return;
  const int64_t r = idx / per_ray;
  const int j = (int)(idx - r * per_ray);
  out[idx] = normal ? src.normal(r, j) : src.uniform(r, j);
}

int launch_random_fill(const RandSrc& src, int stream_id, int64_t n_rays, int per_ray, float* out, cudaStream_t s) {
  const int64_t total = n_rays * per_ray;
  const int threads = 256;
  const int64_t blocks = (total + threads - 1) / threads;
  const int normal = stream_id == kRandNoiseC || stream_id == kRandNoiseF;
  random_fill_kernel<<<(unsigned)blocks, threads, 0, s>>>(src, normal, n_rays, per_ray, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "random_fill launch");
}

// the same with the step read from the device (src.ctr1 holds the stream id): a step >= 2^30, whose counter word would
// alias another step's, writes NaN instead
__global__ void random_fill_dev_kernel(RandSrc src, const int64_t* __restrict__ step, int normal, int64_t n_rays,
                                       int per_ray, float* __restrict__ out) {
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= n_rays * per_ray) return;
  const int64_t st = *step;
  if (st < 0 || st >= (int64_t(1) << 30)) {
    out[idx] = __int_as_float(0x7fc00000);
    return;
  }
  src.ctr1 += 4u * (uint32_t)st;
  const int64_t r = idx / per_ray;
  const int j = (int)(idx - r * per_ray);
  out[idx] = normal ? src.normal(r, j) : src.uniform(r, j);
}

int launch_random_fill_dev(const RandSrc& src, const int64_t* step, int stream_id, int64_t n_rays, int per_ray,
                           float* out, cudaStream_t s) {
  const int64_t total = n_rays * per_ray;
  const int threads = 256;
  const int64_t blocks = (total + threads - 1) / threads;
  const int normal = stream_id == kRandNoiseC || stream_id == kRandNoiseF;
  random_fill_dev_kernel<<<(unsigned)blocks, threads, 0, s>>>(src, step, normal, n_rays, per_ray, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "random_fill_dev launch");
}

// ---------------------------------------------------------------------------------------------
// stand-alone positional encoding (test hook; the MLP kernels encode in their prologue)
// ---------------------------------------------------------------------------------------------
__global__ void encode_kernel(Plan p, int which, const float* __restrict__ x, int64_t n, float* __restrict__ out) {
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= n * 3) return;
  const int64_t pt = idx / 3;
  const int c = (int)(idx - pt * 3);
  const int dim = which ? p.dim_dir : p.dim_xyz;
  const int nf = which ? p.n_freq_dir : p.n_freq_xyz;
  const int inc = which ? p.inc_dir : p.inc_xyz;
  const float* fr = which ? p.freq_dir : p.freq_xyz;
  encode_coord(x[idx], c, inc, 0, nf, fr, out + pt * dim);
}

int launch_encode(const Plan& p, int which, const float* x, int64_t n, float* out, cudaStream_t s) {
  const int threads = 256;
  const int64_t blocks = (n * 3 + threads - 1) / threads;
  encode_kernel<<<(unsigned)blocks, threads, 0, s>>>(p, which, x, n, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "encode launch");
}

// ---------------------------------------------------------------------------------------------
// sample_pdf + merge: one warp per ray
// ---------------------------------------------------------------------------------------------
constexpr int kPdfWarps = 4;

__global__ void __launch_bounds__(kPdfWarps * 32)
sample_pdf_merge_kernel(const float* __restrict__ z_coarse, const float* __restrict__ weights,
                        const RandSrc u, const float* __restrict__ cdf_in,
                        int64_t n_rays, int nc, int nf, int npow2, float* __restrict__ z_fine,
                        float* __restrict__ z_samples, int32_t* __restrict__ inds_out,
                        float* __restrict__ cdf_out) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = blockIdx.x * (int64_t)kPdfWarps + warp;
  if (r >= n_rays) return;  // whole warp exits together; only __syncwarp below
  const int nb = nc - 1;    // bins = mid-points = cdf entries
  const int nw = nc - 2;    // interior weights
  // per-warp buffers: sort[npow2] | cdf[nc] | bins[nc] | pdf[nc]  (pdf has its own region: npow2 can be smaller
  // than nc + (nc - 2) when n_fine < n_coarse - 2, so it must not live inside the sort buffer)
  float* sort = smem + (size_t)warp * (npow2 + 3 * nc);
  float* cdf = sort + npow2;
  float* bins = cdf + nc;
  float* pdf = bins + nc;

  const float* zc = z_coarse + r * nc;
  for (int i = lane; i < nc; i += 32) sort[i] = zc[i];
  __syncwarp();
  for (int j = lane; j < nb; j += 32) bins[j] = __fmul_rn(0.5f, __fadd_rn(sort[j + 1], sort[j]));

  if (cdf_in) {
    for (int j = lane; j < nb; j += 32) cdf[j] = cdf_in[r * nb + j];
  } else {
    // weights + 1e-5, pdf = w / sum(w), cdf = [0, cumsum(pdf)]  (nerf_helpers.py:265-270).
    // The sum is accumulated in fp64 and rounded once; the cumsum is a sequential fp64
    // accumulation rounded per element, which is what torch's CPU cumsum does for fp32 input.
    const float* w = weights + r * nc + 1;
    double part = 0.0;
    for (int j = lane; j < nw; j += 32) part += (double)__fadd_rn(w[j], 1e-5f);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    const float total = (float)part;
    for (int j = lane; j < nw; j += 32) pdf[j] = __fdiv_rn(__fadd_rn(w[j], 1e-5f), total);
    __syncwarp();
    if (lane == 0) {
      double acc = 0.0;
      cdf[0] = 0.f;
      for (int j = 0; j < nw; ++j) {
        acc += (double)pdf[j];
        cdf[j + 1] = (float)acc;
      }
    }
  }
  __syncwarp();
  if (cdf_out)
    for (int j = lane; j < nb; j += 32) cdf_out[r * nb + j] = cdf[j];

  // inverse CDF (nerf_helpers.py:286-300): searchsorted(cdf, u, side="right") by binary search
  for (int q = lane; q < nf; q += 32) {
    const float uq = u.present() ? u.uniform(r, q) : linspace01(q, nf);
    int lo = 0, hi = nb;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cdf[mid] <= uq) lo = mid + 1; else hi = mid;
    }
    const int below = max(0, lo - 1), above = min(nb - 1, lo);
    const float cb = cdf[below], ca = cdf[above], bb = bins[below], ba = bins[above];
    float denom = __fsub_rn(ca, cb);
    if (denom < 1e-5f) denom = 1.0f;
    const float t = __fdiv_rn(__fsub_rn(uq, cb), denom);
    const float smp = __fadd_rn(bb, __fmul_rn(t, __fsub_rn(ba, bb)));
    if (z_samples) z_samples[r * nf + q] = smp;
    if (inds_out) inds_out[r * nf + q] = lo;
    sort[nc + q] = smp;
  }
  for (int i = nc + nf + lane; i < npow2; i += 32) sort[i] = CUDART_INF_F;
  __syncwarp();

  // torch.sort(cat(z_vals, z_samples)) (train_utils.py:105): bitonic network over npow2 slots
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < npow2; i += 32) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const float a = sort[i], b = sort[ixj];
          const bool asc = (i & k) == 0;
          if ((a > b) == asc) {
            sort[i] = b;
            sort[ixj] = a;
          }
        }
      }
      __syncwarp();
    }
  }
  if (z_fine) {
    float* zf = z_fine + r * (int64_t)(nc + nf);
    for (int i = lane; i < nc + nf; i += 32) zf[i] = sort[i];
  }
}

int launch_sample_pdf_merge(const float* z_coarse, const float* weights_coarse, const RandSrc& u, const float* cdf_in, int64_t n_rays, int n_coarse, int n_fine, float* z_fine,
                            float* z_samples, int32_t* inds, float* cdf_out, cudaStream_t s) {
  int npow2 = 1;
  while (npow2 < n_coarse + n_fine) npow2 <<= 1;
  const size_t smem = (size_t)kPdfWarps * (npow2 + 3 * n_coarse) * sizeof(float);
  if (smem > 48 * 1024) {
    int rc = check_cuda(cudaFuncSetAttribute(sample_pdf_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem),
                        "sample_pdf smem attribute");
    if (rc) return rc;
  }
  const int64_t blocks = (n_rays + kPdfWarps - 1) / kPdfWarps;
  sample_pdf_merge_kernel<<<(unsigned)blocks, kPdfWarps * 32, smem, s>>>(
      z_coarse, weights_coarse, u, cdf_in, n_rays, n_coarse, n_fine, npow2, z_fine, z_samples, inds,
      cdf_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "sample_pdf_merge launch");
}

// ---------------------------------------------------------------------------------------------
// weight packing: flat torch-layout vector -> kernel blob (transposed / padded copies)
// ---------------------------------------------------------------------------------------------
__global__ void pack_kernel(Plan p, const float* __restrict__ flat, float* __restrict__ blob) {
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < p.blob_floats; idx += gridDim.x * blockDim.x) {
    float val = 0.f;
    bool found = false;
    for (int gi = 0; gi < p.n_gemm && !found; ++gi) {
      const GemmLayer& g = p.g[gi];
      const int in_real = g.k_h + g.enc_real;
      const int K = g.k_h + g.k_enc;
      if (idx >= g.wt_off && idx < g.wt_off + K * g.n) {
        const int k = (idx - g.wt_off) / g.n, j = (idx - g.wt_off) % g.n;
        int col = -1;
        if (k < g.k_h) col = k;
        else if (k - g.k_h < g.enc_real) col = k;
        if (col >= 0) val = flat[g.flat_w + j * in_real + col];
        found = true;
      } else if (idx >= g.wh_off && idx < g.wh_off + g.n * g.k_h) {
        const int nn = (idx - g.wh_off) / g.k_h, k = (idx - g.wh_off) % g.k_h;
        val = flat[g.flat_w + nn * in_real + k];
        found = true;
      } else if (idx >= g.b_off && idx < g.b_off + g.n) {
        val = flat[g.flat_b + (idx - g.b_off)];
        found = true;
      } else if (idx >= g.tc_off && idx < g.tc_off + 3 * ((g.k_tc + 15) & ~15) * g.n / 2) {
        // forward operand, three fp16 copies (tc_common.cuh split_w3): [k-step of 16][hs|h|l][slab 0|1][n][8 halves];
        // this float slot holds the halves of (n, k) and (n, k + 1) with k = kstep*16 + slab*8 + 2j (low half = k).
        // K is padded to a multiple of 16 with zeros.
        const int e = idx - g.tc_off;
        const int per_step = 24 * g.n;
        const int ks = e / per_step, r = e - ks * per_step;
        const int part = r / (8 * g.n), r2 = r - part * 8 * g.n;
        const int slab = r2 / (4 * g.n), r3 = r2 - slab * 4 * g.n;
        const int nn = r3 >> 2, j = r3 & 3;
        const int k = ks * 16 + slab * 8 + 2 * j;
        float w0 = 0.f, w1 = 0.f;
        if (k < g.k_tc && (k < g.k_h || k - g.k_h < g.enc_real)) w0 = flat[g.flat_w + nn * in_real + k];
        if (k + 1 < g.k_tc && (k + 1 < g.k_h || k + 1 - g.k_h < g.enc_real)) w1 = flat[g.flat_w + nn * in_real + k + 1];
        uint32_t hs, h, l;
        tc::split_w3(w0, w1, hs, h, l);
        val = __uint_as_float(part == 0 ? hs : (part == 1 ? h : l));
        found = true;
      } else if (idx >= g.tcd_off && idx < g.tcd_off + 3 * g.k_h * g.n / 2) {
        // dgrad operand, three fp16 copies: [k-step of 16 over n][hs|h|l][slab 0|1][k < k_h][8 halves]; this float
        // slot holds W[n][k] and W[n + 1][k] with n = kstep*16 + slab*8 + 2j
        const int e = idx - g.tcd_off;
        const int per_step = 24 * g.k_h;
        const int ks = e / per_step, r = e - ks * per_step;
        const int part = r / (8 * g.k_h), r2 = r - part * 8 * g.k_h;
        const int slab = r2 / (4 * g.k_h), r3 = r2 - slab * 4 * g.k_h;
        const int k = r3 >> 2, j = r3 & 3;
        const int nn = ks * 16 + slab * 8 + 2 * j;
        const float w0 = nn < g.n ? flat[g.flat_w + nn * in_real + k] : 0.f;
        const float w1 = nn + 1 < g.n ? flat[g.flat_w + (nn + 1) * in_real + k] : 0.f;
        uint32_t hs, h, l;
        tc::split_w3(w0, w1, hs, h, l);
        val = __uint_as_float(part == 0 ? hs : (part == 1 ? h : l));
        found = true;
      }
    }
    for (int hi = 0; hi < p.n_head && !found; ++hi) {
      const HeadLayer& h = p.h[hi];
      if (idx >= h.w_off && idx < h.b_off) {
        const int i = idx - h.w_off;
        if (i < h.n_out * h.k) val = flat[h.flat_w + i];
        found = true;
      } else if (idx >= h.b_off && idx < h.b_off + 4) {
        const int i = idx - h.b_off;
        if (i < h.n_out) val = flat[h.flat_b + i];
        found = true;
      }
    }
    blob[idx] = val;
  }
}

int launch_pack(const Plan& p, const float* flat, float* blob, cudaStream_t s) {
  const int threads = 256;
  int blocks = (p.blob_floats + threads - 1) / threads;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  pack_kernel<<<blocks, threads, 0, s>>>(p, flat, blob);
  count_launch();
  return check_cuda(cudaGetLastError(), "pack launch");
}

// ---------------------------------------------------------------------------------------------
// fused Adam over a flat vector (torch.optim.Adam, amsgrad off, weight_decay 0)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void adam_element(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                             float* __restrict__ v, int64_t i, float lr_over_bc1, float inv_sqrt_bc2,
                                             float b1, float b2, float eps, float grad_scale) {
  const float gi = g[i] * grad_scale;
  const float mi = m[i] + (gi - m[i]) * (1.f - b1);         // exp_avg.lerp_(grad, 1 - beta1)
  const float vi = v[i] * b2 + (1.f - b2) * gi * gi;        // exp_avg_sq.mul_(b2).addcmul_(g, g, 1 - b2)
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) * inv_sqrt_bc2 + eps;       // sqrt(v) / sqrt(bc2) + eps
  p[i] = p[i] - lr_over_bc1 * (mi / denom);                 // addcdiv_(m, denom, value=-lr/bc1)
}

__device__ __forceinline__ void adam_update(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                            float* __restrict__ v, int64_t n, float lr_over_bc1, float inv_sqrt_bc2,
                                            float b1, float b2, float eps, float grad_scale) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    adam_element(p, g, m, v, i, lr_over_bc1, inv_sqrt_bc2, b1, b2, eps, grad_scale);
}

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, int64_t n, float lr_over_bc1, float inv_sqrt_bc2, float b1,
                            float b2, float eps, float grad_scale) {
  adam_update(p, g, m, v, n, lr_over_bc1, inv_sqrt_bc2, b1, b2, eps, grad_scale);
}

int launch_adam(float* p, const float* g, float* m, float* v, int64_t n, int step, float lr, float b1, float b2,
                float eps, float grad_scale, cudaStream_t s) {
  const double bc1 = 1.0 - pow((double)b1, (double)step);
  const double bc2 = 1.0 - pow((double)b2, (double)step);
  const int threads = 256;
  int64_t blocks = (n + threads - 1) / threads;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  adam_kernel<<<(unsigned)blocks, threads, 0, s>>>(p, g, m, v, n, (float)(lr / bc1), (float)(1.0 / sqrt(bc2)), b1, b2,
                                                   eps, grad_scale);
  count_launch();
  return check_cuda(cudaGetLastError(), "adam launch");
}

// parallel.FusedAdam.current_lr after `done` steps, in fp64 and rounded once to fp32 as the float argument of adam_step
// is: lr0 * factor ** (max(done - 1, 0) / (decay * 1000)), or lr0 without a schedule (decay <= 0)
__device__ __forceinline__ float scheduled_lr(int64_t done, const LrSchedule& sch) {
  if (!(sch.decay > 0.0)) return (float)sch.lr0;
  const double e = (double)(done > 1 ? done - 1 : 0) / (sch.decay * 1000.0);
  return (float)(sch.lr0 * pow(sch.factor, e));
}

__global__ void lr_schedule_kernel(const int64_t* __restrict__ done, int64_t n, LrSchedule sch, float* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = scheduled_lr(done[i], sch);
}

int launch_lr_schedule(const int64_t* done, int64_t n, const LrSchedule& sch, float* out, cudaStream_t s) {
  lr_schedule_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(done, n, sch, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "lr_schedule launch");
}

// adam_kernel with the step count read from the device: *done steps before this one, so this is step *done + 1 at the
// rate of scheduled_lr(*done); the scalars are formed in fp64 as launch_adam forms them on the host
__global__ void adam_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                float* __restrict__ v, int64_t n, const int64_t* __restrict__ done, LrSchedule sch,
                                float b1, float b2, float eps, float grad_scale) {
  __shared__ float scal[2];
  if (threadIdx.x == 0) {
    const int64_t d = *done;
    const float lr = scheduled_lr(d, sch);
    const double step = (double)(d + 1);
    const double bc1 = 1.0 - pow((double)b1, step);
    const double bc2 = 1.0 - pow((double)b2, step);
    scal[0] = (float)(lr / bc1);
    scal[1] = (float)(1.0 / sqrt(bc2));
  }
  __syncthreads();
  adam_update(p, g, m, v, n, scal[0], scal[1], b1, b2, eps, grad_scale);
}

int launch_adam_dev(float* p, const float* g, float* m, float* v, int64_t n, const int64_t* done, const LrSchedule& sch,
                    float b1, float b2, float eps, float grad_scale, cudaStream_t s) {
  const int threads = 256;
  int64_t blocks = (n + threads - 1) / threads;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  adam_dev_kernel<<<(unsigned)blocks, threads, 0, s>>>(p, g, m, v, n, done, sch, b1, b2, eps, grad_scale);
  count_launch();
  return check_cuda(cudaGetLastError(), "adam_dev launch");
}

// adam_dev_kernel over baked values (rows of kBakeCh floats): channel 0 (sigma_raw) at the rate of `sigma`, channels
// 1 .. 27 (SH coefficients) at the rate of `sh`, channels 28 .. 31 untouched.  grad_scale is a kernel argument (1) as
// in adam_dev_kernel, so the compiler forms the update from the same operations and the bits match adam_step_dev's.
__global__ void baked_adam_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                      float* __restrict__ v, int64_t n, const int64_t* __restrict__ done,
                                      LrSchedule sigma, LrSchedule sh, float b1, float b2, float eps, float grad_scale) {
  __shared__ float scal[3];
  if (threadIdx.x == 0) {
    const int64_t d = *done;
    const double step = (double)(d + 1);
    const double bc1 = 1.0 - pow((double)b1, step);
    const double bc2 = 1.0 - pow((double)b2, step);
    scal[0] = (float)(scheduled_lr(d, sigma) / bc1);
    scal[1] = (float)(scheduled_lr(d, sh) / bc1);
    scal[2] = (float)(1.0 / sqrt(bc2));
  }
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i & (kBakeCh - 1));
    if (ch >= 1 + 3 * kBakeSh) continue;
    adam_element(p, g, m, v, i, ch == 0 ? scal[0] : scal[1], scal[2], b1, b2, eps, grad_scale);
  }
}

int launch_baked_adam_dev(float* p, const float* g, float* m, float* v, int64_t n, const int64_t* done,
                          const LrSchedule& sigma, const LrSchedule& sh, float b1, float b2, float eps, cudaStream_t s) {
  const int threads = 256;
  int64_t blocks = (n + threads - 1) / threads;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  baked_adam_dev_kernel<<<(unsigned)blocks, threads, 0, s>>>(p, g, m, v, n, done, sigma, sh, b1, b2, eps, 1.f);
  count_launch();
  return check_cuda(cudaGetLastError(), "baked_adam_dev launch");
}

}  // namespace nerfb200
