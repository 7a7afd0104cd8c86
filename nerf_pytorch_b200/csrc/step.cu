// step.cu -- the parts of a training step that the reference runs on the host or as ATen ops, for a step whose only
// changing input is a step counter in device memory (so that the whole step can be captured in one CUDA graph):
//   pixel draw      train_nerf.py:175-193, 213-226   one image uniformly, then n distinct pixels of it (np.random.choice
//                                                     with replace=False), from (seed, *step)
//   target gather   train_nerf.py:220-226            target_s = img_target[select_inds]
//   loss            train_nerf.py:244-258            mse(rgb_coarse, t) + mse(rgb_fine, t), and its upstream gradients
//   step counter                                     advanced once per step, after both networks' Adam updates
// The device-step variants of random_fill, gen_rays and adam_step are in sampling.cu and raygen.cu next to the kernels
// they share their arithmetic with.
#include "common.cuh"

namespace nerfb200 {

// ---------------------------------------------------------------------------------------------
// pixel draw: a 64-bit Philox key per pixel (counter layout in common.cuh), the n smallest (key, pixel id) pairs win.
// That is a uniform draw of n distinct pixels, exact and deterministic.  The pixels come out in ascending key order, which
// is a uniformly random order, like the prefix of a random permutation.
//   1. histogram of the keys' top `bits` bits (about 16 pixels per bin)
//   2. one CTA: the bin b* where the cumulative count reaches n; the image index
//   3. every pixel in a bin <= b* (n + a few) is appended to a candidate list
//   4. one CTA: bitonic sort of the candidates by (key, id) -- in shared memory when they fit, else in place in the
//      workspace (only when bin b* is crowded far beyond its expectation, or n is close to H*W) -- and the first n out
// ---------------------------------------------------------------------------------------------
constexpr int kDrawThreads = 1024;
constexpr int64_t kSortSmemEntries = 16384;  // 12 bytes each (key + id): 192 KB

struct DrawLayout {
  int bits;
  int64_t nbins, cap;            // cap: candidate capacity, a power of two >= n_pixels
  int64_t off_hist, off_keys, off_ids, total;
};

static int64_t pow2_ceil(int64_t x) {
  int64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

static DrawLayout draw_layout(int64_t n_pixels) {
  DrawLayout L;
  int lg = 0;
  while ((int64_t(1) << lg) < n_pixels) ++lg;
  L.bits = lg > 4 ? (lg - 4 < 24 ? lg - 4 : 24) : 0;
  L.nbins = int64_t(1) << L.bits;
  L.cap = pow2_ceil(n_pixels);
  L.off_hist = 256;  // header: candidate count, b*
  L.off_keys = L.off_hist + ((L.nbins * 4 + 255) & ~int64_t(255));
  L.off_ids = L.off_keys + L.cap * 8;
  L.total = L.off_ids + ((L.cap * 4 + 255) & ~int64_t(255));
  return L;
}

struct DrawKey {
  uint32_t k0, k1;  // the seed
};

__device__ __forceinline__ uint4 draw_block(const DrawKey& k, uint32_t q, uint32_t step, uint32_t purpose) {
  return philox4x32_10(make_uint4(q, step, purpose, 0x80000000u), k.k0, k.k1);
}

__device__ __forceinline__ uint64_t key_bin(uint64_t key, int bits) { return bits ? key >> (64 - bits) : 0; }

// each thread draws the keys of pixels 2q and 2q + 1 (one Philox block)
template <bool kCollect>
__global__ void draw_keys_kernel(DrawKey k, const int64_t* __restrict__ step, int64_t n_pixels, int bits,
                                 uint32_t* __restrict__ hdr, uint32_t* __restrict__ hist, uint64_t* __restrict__ keys,
                                 uint32_t* __restrict__ ids) {
  const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (2 * q >= n_pixels) return;
  const uint4 w = draw_block(k, (uint32_t)q, (uint32_t)*step, 0);
  const uint64_t key[2] = {(uint64_t)w.x << 32 | w.y, (uint64_t)w.z << 32 | w.w};
  const uint64_t bstar = kCollect ? hdr[1] : 0;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int64_t p = 2 * q + e;
    if (p >= n_pixels) break;
    const uint64_t b = key_bin(key[e], bits);
    if (!kCollect) {
      atomicAdd(hist + b, 1u);
    } else if (b <= bstar) {
      const uint32_t pos = atomicAdd(hdr, 1u);
      keys[pos] = key[e];
      ids[pos] = (uint32_t)p;
    }
  }
}

__global__ void draw_threshold_kernel(DrawKey k, const int64_t* __restrict__ step, const uint32_t* __restrict__ hist,
                                      int64_t nbins, int64_t n, int n_images, uint32_t* __restrict__ hdr,
                                      int64_t* __restrict__ image_out) {
  __shared__ int64_t warp_tot[kDrawThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t chunk = (nbins + kDrawThreads - 1) / kDrawThreads;
  const int64_t lo = t * chunk < nbins ? t * chunk : nbins, hi = lo + chunk < nbins ? lo + chunk : nbins;
  int64_t s = 0;
  for (int64_t b = lo; b < hi; ++b) s += hist[b];
  int64_t incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int64_t wt = warp_tot[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t v = __shfl_up_sync(0xffffffffu, wt, o);
      if (lane >= o) wt += v;
    }
    warp_tot[lane] = wt;
  }
  __syncthreads();
  const int64_t excl = incl - s + (warp ? warp_tot[warp - 1] : 0);
  if (excl < n && n <= excl + s) {  // exactly one thread's chunk holds the bin where the count reaches n
    int64_t c = excl;
    for (int64_t b = lo; b < hi; ++b) {
      c += hist[b];
      if (c >= n) {
        hdr[1] = (uint32_t)b;
        break;
      }
    }
  }
  if (t == 0) {
    // floor(r * n_images / 2^64) of a 64-bit uniform r: each image with probability 1 / n_images to within 2^-64 n_images
    const uint4 w = draw_block(k, 0, (uint32_t)*step, 1);
    *image_out = (int64_t)__umul64hi((uint64_t)w.x << 32 | w.y, (uint64_t)n_images);
  }
}

__global__ void draw_sort_kernel(const uint32_t* __restrict__ hdr, uint64_t* keys, uint32_t* ids, int64_t smem_entries,
                                 int64_t n, int64_t* __restrict__ ids_out) {
  extern __shared__ __align__(16) unsigned char sort_smem[];
  const int64_t count = hdr[0];
  int64_t P = 1;
  while (P < count) P <<= 1;
  const bool in_smem = P <= smem_entries;
  uint64_t* K = in_smem ? reinterpret_cast<uint64_t*>(sort_smem) : keys;
  uint32_t* I = in_smem ? reinterpret_cast<uint32_t*>(sort_smem + 8 * smem_entries) : ids;
  for (int64_t i = threadIdx.x; i < P; i += blockDim.x) {
    // padding sorts last: a real id is < 2^31
    const uint64_t kv = i < count ? keys[i] : ~uint64_t(0);
    const uint32_t iv = i < count ? ids[i] : ~0u;
    K[i] = kv;
    I[i] = iv;
  }
  __syncthreads();
  for (int64_t size = 2; size <= P; size <<= 1) {
    for (int64_t j = size >> 1; j > 0; j >>= 1) {
      for (int64_t i = threadIdx.x; i < P; i += blockDim.x) {
        const int64_t l = i ^ j;
        if (l <= i) continue;
        const uint64_t ki = K[i], kl = K[l];
        const uint32_t ii = I[i], il = I[l];
        const bool greater = ki > kl || (ki == kl && ii > il);  // (key, id) of i after that of l
        if (greater == ((i & size) == 0)) {
          K[i] = kl; K[l] = ki;
          I[i] = il; I[l] = ii;
        }
      }
      __syncthreads();  // also orders the global-memory path: one block, and __syncthreads makes its writes visible
    }
  }
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) ids_out[i] = (int64_t)I[i];
}

static int launch_draw(uint64_t seed, const int64_t* step, int n_images, int64_t n_pixels, int64_t n, int64_t* image_out,
                       int64_t* ids_out, void* workspace, cudaStream_t s) {
  const DrawLayout L = draw_layout(n_pixels);
  char* base = static_cast<char*>(workspace);
  uint32_t* hdr = reinterpret_cast<uint32_t*>(base);
  uint32_t* hist = reinterpret_cast<uint32_t*>(base + L.off_hist);
  uint64_t* keys = reinterpret_cast<uint64_t*>(base + L.off_keys);
  uint32_t* ids = reinterpret_cast<uint32_t*>(base + L.off_ids);
  const DrawKey k{(uint32_t)seed, (uint32_t)(seed >> 32)};
  int rc = check_cuda(cudaMemsetAsync(base, 0, (size_t)L.off_keys, s), "draw_pixels memset");
  if (rc) return rc;
  const int64_t pairs = (n_pixels + 1) / 2;
  const unsigned blocks = (unsigned)((pairs + 255) / 256);
  draw_keys_kernel<false><<<blocks, 256, 0, s>>>(k, step, n_pixels, L.bits, hdr, hist, keys, ids);
  count_launch();
  draw_threshold_kernel<<<1, kDrawThreads, 0, s>>>(k, step, hist, L.nbins, n, n_images, hdr, image_out);
  count_launch();
  draw_keys_kernel<true><<<blocks, 256, 0, s>>>(k, step, n_pixels, L.bits, hdr, hist, keys, ids);
  count_launch();
  const int64_t smem_entries = L.cap < kSortSmemEntries ? L.cap : kSortSmemEntries;
  const int smem = (int)(smem_entries * 12);
  rc = check_cuda(cudaFuncSetAttribute(draw_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem),
                  "draw_sort smem attribute");
  if (rc) return rc;
  draw_sort_kernel<<<1, kDrawThreads, smem, s>>>(hdr, keys, ids, smem_entries, n, ids_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "draw_pixels launch");
}

// ---------------------------------------------------------------------------------------------
// rows of the drawn image: out[k] = src[(*image * rows_per_image + ids[k])][0..2]
// ---------------------------------------------------------------------------------------------
__global__ void gather_rows_kernel(const float* __restrict__ src, int64_t rows_per_image, const int64_t* __restrict__ image,
                                   const int64_t* __restrict__ ids, int64_t n, float* __restrict__ out) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= 3 * n) return;
  const int64_t k = e / 3;
  out[e] = src[(*image * rows_per_image + ids[k]) * 3 + (e - 3 * k)];
}

// ---------------------------------------------------------------------------------------------
// loss: mse_loss(out[:, :3], t) for the coarse and (when given) the fine output, in one CTA.
// The upstream gradient is what autograd of torch's mean mse_loss gives (ATen mse_loss_backward: alpha * (x - t) * g
// with alpha = float(2 / numel) and g = 1): fp32(alpha * fp32(x - t)) in columns 0..2, zero in 3..7.  The loss sums the
// squared fp32 differences in fp64 (exact products, a fixed order) and rounds each mean once; torch's fp32 tree sum
// differs from that in the last bits.
// ---------------------------------------------------------------------------------------------
constexpr int kLossThreads = 1024;

__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kLossThreads / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}

__global__ void mse_loss_kernel(const float* __restrict__ out_c, const float* __restrict__ out_f,
                                const float* __restrict__ target, int64_t n, float alpha, float* __restrict__ loss,
                                float* __restrict__ g_c, float* __restrict__ g_f) {
  __shared__ double red[kLossThreads / 32];
  double sc = 0.0, sf = 0.0;
  for (int64_t e = threadIdx.x; e < 8 * n; e += kLossThreads) {
    const int64_t r = e >> 3;
    const int c = (int)(e & 7);
    float gc = 0.f, gf = 0.f;
    if (c < 3) {
      const float t = target[3 * r + c];
      const float dc = __fsub_rn(out_c[e], t);
      gc = __fmul_rn(alpha, dc);
      sc += (double)dc * (double)dc;
      if (out_f) {
        const float df = __fsub_rn(out_f[e], t);
        gf = __fmul_rn(alpha, df);
        sf += (double)df * (double)df;
      }
    }
    g_c[e] = gc;
    if (out_f) g_f[e] = gf;
  }
  sc = block_sum(sc, red);
  sf = block_sum(sf, red);
  if (threadIdx.x == 0) {
    const double numel = 3.0 * (double)n;
    const float lc = (float)(sc / numel);
    *loss = out_f ? __fadd_rn(lc, (float)(sf / numel)) : lc;
  }
}

__global__ void step_advance_kernel(int64_t* step) { *step += 1; }

}  // namespace nerfb200

using namespace nerfb200;

extern "C" {

int32_t nerfb200_random_fill_dev(const nerfb200_rng_t* rng, const int64_t* step_dev, int32_t stream_id, int64_t n_rays,
                                 int32_t per_ray, float* out, void* stream) {
  if (!rng || !step_dev || !out || n_rays <= 0 || per_ray <= 0 || stream_id < 0 || stream_id > 3 || rng->step != 0 ||
      rng->ray_offset < 0) {
    set_error("random_fill_dev: invalid argument (rng->step must be 0: the step is read from step_dev)");
    return NERFB200_ERR_INVALID;
  }
  return launch_random_fill_dev(rand_seeded(*rng, stream_id), step_dev, stream_id, n_rays, per_ray, out,
                                static_cast<cudaStream_t>(stream));
}

int64_t nerfb200_draw_workspace_bytes(int64_t n_pixels) {
  if (n_pixels <= 0 || n_pixels >= (int64_t(1) << 31)) return -1;
  return draw_layout(n_pixels).total;
}

int32_t nerfb200_draw_pixels(uint64_t seed, const int64_t* step_dev, int32_t n_images, int64_t n_pixels, int64_t n,
                             int64_t* image_out, int64_t* ids_out, void* workspace, void* stream) {
  if (!step_dev || !image_out || !ids_out || !workspace || n_images <= 0 || n_pixels <= 0 ||
      n_pixels >= (int64_t(1) << 31) || n <= 0) {
    set_error("draw_pixels: invalid argument (null pointer, no image, or n_pixels outside 1 .. 2^31 - 1)");
    return NERFB200_ERR_INVALID;
  }
  if (n > n_pixels) {
    set_error("draw_pixels: cannot draw %lld distinct pixels out of %lld", (long long)n, (long long)n_pixels);
    return NERFB200_ERR_INVALID;
  }
  return launch_draw(seed, step_dev, n_images, n_pixels, n, image_out, ids_out, workspace,
                     static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_gen_rays_posed(const float* poses, int32_t pose_rows, const int64_t* image, int32_t height,
                                int32_t width, float focal, const int64_t* pixel_ids, int64_t n, int32_t ndc, float near,
                                float far, int32_t use_viewdirs, int32_t out_stride, float* out, void* stream) {
  if (!poses || !image || !pixel_ids || !out || n <= 0 || (pose_rows != 3 && pose_rows != 4)) {
    set_error("gen_rays_posed: null pointer, empty batch or pose_rows not 3 or 4");
    return NERFB200_ERR_INVALID;
  }
  return launch_gen_rays_posed(poses, pose_rows, image, height, width, focal, pixel_ids, n, ndc, near, far, use_viewdirs,
                               out_stride, out, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_gather_rows(const float* src, int64_t rows_per_image, const int64_t* image, const int64_t* ids,
                             int64_t n, float* out, void* stream) {
  if (!src || !image || !ids || !out || n <= 0 || rows_per_image <= 0) {
    set_error("gather_rows: null pointer or empty batch");
    return NERFB200_ERR_INVALID;
  }
  gather_rows_kernel<<<(unsigned)((3 * n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, rows_per_image, image, ids, n, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "gather_rows launch");
}

int32_t nerfb200_mse_loss(const float* out_coarse, const float* out_fine, const float* target, int64_t n, float* loss,
                          float* g_coarse, float* g_fine, void* stream) {
  if (!out_coarse || !target || !loss || !g_coarse || n <= 0 || (out_fine != nullptr) != (g_fine != nullptr)) {
    set_error("mse_loss: null pointer or empty batch (g_fine must be given iff out_fine is)");
    return NERFB200_ERR_INVALID;
  }
  const float alpha = (float)(2.0 / (3.0 * (double)n));
  mse_loss_kernel<<<1, kLossThreads, 0, static_cast<cudaStream_t>(stream)>>>(out_coarse, out_fine, target, n, alpha, loss,
                                                                             g_coarse, g_fine);
  count_launch();
  return check_cuda(cudaGetLastError(), "mse_loss launch");
}

static int check_schedule(double lr0, double lr_decay, double factor, const char* what) {
  if (!(lr0 >= 0.0) || !(lr_decay >= 0.0) || !(factor > 0.0)) {
    set_error("%s: need lr0 >= 0, lr_decay >= 0 (0: no schedule) and lr_decay_factor > 0", what);
    return NERFB200_ERR_INVALID;
  }
  return NERFB200_OK;
}

int32_t nerfb200_lr_schedule(const int64_t* done, int64_t n, double lr0, double lr_decay, double lr_decay_factor,
                             float* lr_out, void* stream) {
  if (check_schedule(lr0, lr_decay, lr_decay_factor, "lr_schedule")) return NERFB200_ERR_INVALID;
  if (!done || !lr_out || n <= 0) {
    set_error("lr_schedule: null pointer or empty input");
    return NERFB200_ERR_INVALID;
  }
  return launch_lr_schedule(done, n, LrSchedule{lr0, lr_decay, lr_decay_factor}, lr_out,
                            static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_adam_step_dev(float* p, const float* g, float* m, float* v, int64_t n, const int64_t* step_dev,
                               double lr0, double lr_decay, double lr_decay_factor, float beta1, float beta2, float eps,
                               float grad_scale, void* stream) {
  if (check_schedule(lr0, lr_decay, lr_decay_factor, "adam_step_dev")) return NERFB200_ERR_INVALID;
  if (!p || !g || !m || !v || !step_dev || n <= 0) {
    set_error("adam_step_dev: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  return launch_adam_dev(p, g, m, v, n, step_dev, LrSchedule{lr0, lr_decay, lr_decay_factor}, beta1, beta2, eps,
                         grad_scale, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_baked_adam_step_dev(float* values, const float* g, float* m, float* v, int64_t n_active,
                                     const int64_t* step_dev, double lr_sigma, double lr_sh, double lr_decay,
                                     double lr_decay_factor, float beta1, float beta2, float eps, void* stream) {
  if (check_schedule(lr_sigma, lr_decay, lr_decay_factor, "baked_adam_step_dev") ||
      check_schedule(lr_sh, lr_decay, lr_decay_factor, "baked_adam_step_dev"))
    return NERFB200_ERR_INVALID;
  if (!values || !g || !m || !v || !step_dev || n_active <= 0) {
    set_error("baked_adam_step_dev: null pointer or n_active <= 0");
    return NERFB200_ERR_INVALID;
  }
  return launch_baked_adam_dev(values, g, m, v, n_active * kBakePts * kBakeCh, step_dev,
                               LrSchedule{lr_sigma, lr_decay, lr_decay_factor},
                               LrSchedule{lr_sh, lr_decay, lr_decay_factor}, beta1, beta2, eps,
                               static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_step_advance(int64_t* step_dev, void* stream) {
  if (!step_dev) {
    set_error("step_advance: null pointer");
    return NERFB200_ERR_INVALID;
  }
  step_advance_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(step_dev);
  count_launch();
  return check_cuda(cudaGetLastError(), "step_advance launch");
}

}  // extern "C"
