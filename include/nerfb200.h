/*
 * nerfb200.h -- C ABI of the H100-native NeRF per-ray hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b): the reference (krrish94/nerf-pytorch @ a14357d) has no
 * FFI; its hot path is plain Python behind two functions,
 *     run_one_iter_of_nerf            nerf/train_utils.py:130-202
 *     predict_and_render_radiance     nerf/train_utils.py:28-127
 * The host-side mirror of those two functions lives in nerf_pytorch_b200/train_utils.py and binds
 * this library with ctypes (see INTEGRATION.md for the stub a reference maintainer would add).
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless it says "host";
 *   - all tensors fp32, row-major, contiguous; indices int32 unless stated;
 *   - every entry point takes the CUDA stream to launch on (a cudaStream_t passed as void*),
 *     never synchronises, and returns 0 on success or a negative NERFB200_ERR_* code;
 *     nerfb200_last_error() returns a thread-local message for the last failure;
 *   - no exceptions cross the boundary; no global state besides the error string.
 */
#ifndef NERFB200_H_
#define NERFB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NERFB200_VERSION 101 /* 0.1.1 */

#define NERFB200_OK 0
#define NERFB200_ERR_INVALID (-1)     /* bad argument (null pointer, size <= 0, ...) */
#define NERFB200_ERR_UNSUPPORTED (-2) /* configuration outside what the kernels implement */
#define NERFB200_ERR_CUDA (-3)        /* CUDA runtime error, text in nerfb200_last_error() */

#define NERFB200_MAX_FREQS 16
#define NERFB200_MAX_LINEAR 24

/* Architecture of one FlexibleNeRFModel (nerf/models.py:185-231) + its encoders
 * (nerf/nerf_helpers.py:113-167).  The wide ("skip") layers are the ones __init__ allocates with
 * dim_xyz + hidden inputs: layers_xyz[i] with i % skip_every == 0 and i > 0 (models.py:210). */
typedef struct nerfb200_arch {
  int32_t num_layers;        /* layer1 + (num_layers - 1) layers_xyz                          */
  int32_t hidden;            /* hidden_size; 128 or 256                                        */
  int32_t skip_every;        /* skip_connect_every                                             */
  int32_t use_viewdirs;      /* 1: fc_feat/fc_alpha/layers_dir[0]/fc_rgb heads, 0: fc_out      */
  int32_t n_freq_xyz;        /* num_encoding_fn_xyz (<= NERFB200_MAX_FREQS)                    */
  int32_t n_freq_dir;        /* num_encoding_fn_dir                                            */
  int32_t include_input_xyz; /* positional_encoding(include_input=...)                         */
  int32_t include_input_dir;
  float freq_xyz[NERFB200_MAX_FREQS]; /* the frequency bands exactly as the reference builds  */
  float freq_dir[NERFB200_MAX_FREQS]; /* them (nerf_helpers.py:131-147), computed by the host  */
} nerfb200_arch_t;

/* Sampling / compositing options = options.nerf.<mode>.* of the reference (config/lego.yml:60-80). */
typedef struct nerfb200_render_opts {
  int32_t n_coarse;   /* num_coarse                                                            */
  int32_t n_fine;     /* num_fine (0: coarse only)                                             */
  int32_t perturb;    /* stratified jitter on (train_utils.py:58-65)                           */
  int32_t lindisp;    /* sample linearly in disparity (train_utils.py:52-55)                   */
  int32_t white_bkgd; /* volume_rendering_utils.py:50-51                                       */
  float noise_std;    /* radiance_field_noise_std (volume_rendering_utils.py:27-38)            */
} nerfb200_render_opts_t;

int32_t nerfb200_version(void);
const char* nerfb200_last_error(void);
/* number of CUDA kernels this library has launched in this process (all threads) */
int64_t nerfb200_launch_count(void);
/* HBM bytes the wgmma backward reads per point: one activation-tile row (4 bytes per feature: fp16 hi + lo) per
 * weight-gradient job, the ReLU bit masks and d_raw -- the algorithmic traffic of its roofline */
int64_t nerfb200_bwd_bytes_per_point(const nerfb200_arch_t* arch);
/* NERFB200_OK if `impl` (0 fp32 CUDA cores, 1 wgmma) can run this architecture forward AND backward with
 * n_samples samples per ray, else NERFB200_ERR_UNSUPPORTED (reason in nerfb200_last_error()); impl 0 refuses only
 * networks whose forward tiles exceed shared memory.  impl = 2 asks for the wgmma FORWARD alone (inference:
 * training = 0 in render_fwd / stash = NULL in mlp_fwd with impl = 1), which also covers hidden_size 256.  impl = 3
 * (the single-pass fp16 forward, see nerfb200_mlp_fwd) gives the same answer as 2.  Any other code:
 * NERFB200_ERR_INVALID. */
int32_t nerfb200_impl_supported(const nerfb200_arch_t* arch, int32_t n_samples, int32_t impl);

/* ---- parameters -------------------------------------------------------------------------------
 * Canonical order of the linears ("slots"): layer1, layers_xyz[0..num_layers-2], then
 * fc_feat, fc_alpha, layers_dir[0], fc_rgb (use_viewdirs) or fc_out.
 * The FLAT parameter / gradient vector is the concatenation, in that order, of weight[out][in]
 * then bias[out] exactly as torch stores them -- so slices of it can be handed to torch as
 * param / param.grad views.  The packed "blob" is the kernels' private layout (transposed and
 * padded copies); rebuild it with nerfb200_pack_weights whenever the parameters change. */
int64_t nerfb200_num_linear(const nerfb200_arch_t* arch);
int64_t nerfb200_flat_param_count(const nerfb200_arch_t* arch);
int64_t nerfb200_blob_floats(const nerfb200_arch_t* arch);
/* offsets (in floats) of weight and bias of linear `slot` inside the flat vector; also in/out. */
int32_t nerfb200_flat_layout(const nerfb200_arch_t* arch, int32_t slot, int64_t* w_off, int64_t* b_off,
                             int32_t* in_features, int32_t* out_features);
/* flat (device, fp32[flat_param_count]) -> blob (device, fp32[blob_floats]). */
int32_t nerfb200_pack_weights(const nerfb200_arch_t* arch, const float* flat, float* blob, void* stream);

/* ---- stage-level entry points (each is also a test hook; SURVEY.md section 8b) ------------------ */

/* Stratified depths, train_utils.py:45-65.  rays[n_rays][ray_stride] = [o(3) d(3) near far (viewdir(3))];
 * t_rand[n_rays][n_coarse] uniform [0,1) or NULL when !perturb.  The grid t = torch.linspace(0,1,n_coarse) is
 * computed in the kernel, bit for bit as torch's CUDA linspace computes it.  Writes z[n_rays][n_coarse]. */
int32_t nerfb200_sample_coarse(const float* rays, int32_t ray_stride, int64_t n_rays, const float* t_rand,
                               int32_t n_coarse, int32_t perturb, int32_t lindisp, float* z, void* stream);

/* Ray generation / packing in one launch (SURVEY.md section 8f-2).  Output rows of `out_stride` floats:
 *   11: [o(3) d(3) near far viewdir(3)]  (train_utils.py:164-168, use_viewdirs)   8: without the view direction
 *    6: [o(3) d(3)] only (get_ray_bundle, nerf_helpers.py:67-110)
 * ndc != 0 applies ndc_rays(H, W, focal, 1.0, ...) (nerf_helpers.py:170-197) AFTER the view directions were taken
 * from the original directions (train_utils.py:143-160).
 * gen_rays:  c2w12 = the 3 x 4 camera-to-world matrix, 12 floats in HOST memory; pixel_ids[n] (device, int64,
 *            j * width + i) or NULL for all height*width pixels in row-major order.
 * pack_rays: caller-supplied origins / directions ro, rd [n][3] (device), the reference call shape. */
int32_t nerfb200_gen_rays(const float* c2w12_host, int32_t height, int32_t width, float focal, const int64_t* pixel_ids,
                          int64_t n, int32_t ndc, float near, float far, int32_t use_viewdirs, int32_t out_stride,
                          float* out, void* stream);
int32_t nerfb200_pack_rays(const float* ro, const float* rd, int64_t n, int32_t height, int32_t width, float focal,
                           int32_t ndc, float near, float far, int32_t use_viewdirs, int32_t out_stride, float* out,
                           void* stream);

/* positional_encoding (nerf_helpers.py:113-157) of x[n][3] -> out[n][dim], dim = 3*include + 6*n_freq.
 * which = 0: xyz encoder of `arch`, 1: direction encoder. */
int32_t nerfb200_encode(const nerfb200_arch_t* arch, int32_t which, const float* x, int64_t n, float* out,
                        void* stream);

/* Fused point generation + encoding + FlexibleNeRFModel.forward (train_utils.py:67, :8-25;
 * models.py:233-256) for every sample of every ray: raw[n_rays][n_samples][4] = [r g b sigma].
 * stash: NULL (inference) or fp32[nerfb200_stash_floats(arch, n_rays*n_samples)] receiving the
 * post-activation output of every hidden linear (needed by the backward entry points; private layout of the
 * implementation that wrote it: the backward must run with the same impl).
 * impl: 0 = fp32 CUDA cores (bit-faithful fp32 FMA), 1 = wgmma tensor cores: every product as a three-term
 * split (fp16 x 2 operands with a 2^11-scaled residual, fp32 accumulation; ~22 significant bits per operand).
 * The split carries 22 bits for magnitudes in 6.1e-5 .. 65504 and resolves 1.5e-11 absolutely below; larger
 * activations / weights saturate (a NeRF's stay far inside; use impl 0 for networks that do not).
 * impl 3 = single-pass fp16 wgmma forward, INFERENCE ONLY: one product fp16(w) x fp16(activation / 16) per k-step,
 * fp32 accumulation (~11 significant bits per operand; the 1- and 3-wide heads and the direction term stay fp32).
 * Judged by the PSNR of the rendered image, not by parity with impl 0 / 1.  Accepted where impl 2 is; stash must be
 * NULL (NERFB200_ERR_UNSUPPORTED otherwise), and mlp_bwd, mlp_dgrad, mlp_wgrad, bwd_scratch_floats and render_bwd
 * refuse it.  |activation| >= 1.05e6 or |weight| >= 32 turns the output into inf / NaN, as with impl 1. */
int64_t nerfb200_stash_floats(const nerfb200_arch_t* arch, int64_t n_points);
int32_t nerfb200_mlp_fwd(const nerfb200_arch_t* arch, const float* blob, const float* rays, int32_t ray_stride,
                         const float* z, int64_t n_rays, int32_t n_samples, float* raw, float* stash,
                         int32_t impl, void* stream);

/* volume_render_radiance_field (volume_rendering_utils.py:6-53).  noise: unit normals
 * [n_rays][n_samples] or NULL (then noise_std is ignored).  out[n_rays][8] =
 * [r g b disp acc depth 0 0]; weights[n_rays][n_samples] may be NULL. */
int32_t nerfb200_composite_fwd(const float* raw, const float* z, const float* rays, int32_t ray_stride,
                               const float* noise, int64_t n_rays, int32_t n_samples, float noise_std,
                               int32_t white_bkgd, float* out, float* weights, void* stream);

/* Backward of the above w.r.t. raw.  g_out[n_rays][8] carries dL/d[r g b disp acc . . .] (depth
 * slot ignored: the reference API never returns depth).  Writes d_raw[n_rays][n_samples][4]. */
int32_t nerfb200_composite_bwd(const float* raw, const float* z, const float* rays, int32_t ray_stride,
                               const float* noise, const float* g_out, int64_t n_rays, int32_t n_samples,
                               float noise_std, int32_t white_bkgd, float* d_raw, void* stream);

/* sample_pdf_2 (nerf_helpers.py:260-302) + detach/cat/sort (train_utils.py:96-105):
 * bins = mid-points of z_coarse, weights_coarse[...,1:-1] + 1e-5 -> pdf -> cdf (63 entries for 64
 * coarse samples) -> inverse-CDF samples at u[n_rays][n_fine], or, u = NULL, at the det=True
 * torch.linspace(0,1,n_fine) computed in the kernel -> z_fine[n_rays][n_coarse+n_fine] ascending.
 * Optional outputs (NULL to skip): z_samples[n_rays][n_fine] (unsorted), inds int32 [n_rays][n_fine]
 * (searchsorted(cdf, u, right) result), cdf_out[n_rays][n_coarse-1].
 * cdf_in (optional): use this cdf instead of computing it ("bit-exact indices given the same cdf"). */
int32_t nerfb200_sample_pdf_merge(const float* z_coarse, const float* weights_coarse, const float* u,
                                  const float* cdf_in, int64_t n_rays, int32_t n_coarse, int32_t n_fine,
                                  float* z_fine, float* z_samples, int32_t* inds, float* cdf_out, void* stream);

/* Backward of nerfb200_mlp_fwd w.r.t. the parameters.  d_raw[n_points][4]; stash from the forward (same impl).
 * gstash: scratch fp32[nerfb200_bwd_scratch_floats(arch, n_points, impl)] (impl 0: the per-layer gradient stash;
 * impl 1: the L2-resident gradient blob the fused kernel reduces its weight-gradient tiles into; -1 where the
 * backward refuses the impl, reason in nerfb200_last_error()).
 * flat_grad: fp32[flat_param_count], ACCUMULATED into (zero it first).  Gradients w.r.t. rays / z are not
 * produced (the reference detaches the fine depths, train_utils.py:103, and rays are data). */
int64_t nerfb200_bwd_scratch_floats(const nerfb200_arch_t* arch, int64_t n_points, int32_t impl);
int32_t nerfb200_mlp_bwd(const nerfb200_arch_t* arch, const float* blob, const float* rays, int32_t ray_stride,
                         const float* z, int64_t n_rays, int32_t n_samples, const float* d_raw,
                         const float* stash, float* gstash, float* flat_grad, int32_t impl, void* stream);
/* The two halves of nerfb200_mlp_bwd as separate calls (autograd's accumulation of nn.Linear backward,
 * nerf/models.py:233-256 replayed in reverse): dgrad walks the chain backwards and fills `gstash` with the
 * pre-activation gradients; wgrad reduces dW = dY^T X over all points into `flat_grad` (+=).  impl 0 only: the
 * wgmma backward is one fused kernel that never writes the gradients out (NERFB200_ERR_UNSUPPORTED). */
int32_t nerfb200_mlp_dgrad(const nerfb200_arch_t* arch, const float* blob, const float* d_raw, const float* stash,
                           float* gstash, int64_t n_points, int32_t impl, void* stream);
int32_t nerfb200_mlp_wgrad(const nerfb200_arch_t* arch, const float* rays, int32_t ray_stride, const float* z,
                           int64_t n_rays, int32_t n_samples, const float* d_raw, const float* stash,
                           const float* gstash, float* flat_grad, int32_t impl, void* stream);

/* ---- caller-given samples (run_network, nerf/train_utils.py:8-25; volume_render_radiance_field,
 * nerf/volume_rendering_utils.py:6-53) ----------------------------------------------------------------
 * The same kernels as the stage entry points above, on points and depths the caller chose instead of the stratified /
 * hierarchical samples of a ray row.  Ray r's view direction is the 3 floats at dirs + r * dir_stride (dir_stride >= 0,
 * in floats; 0 broadcasts one direction), so the last three columns of any ray row can be read in place.
 *
 * mlp_fwd_pts: nerfb200_mlp_fwd with the points given: pts[n_rays][n_samples][3]; sample s of row r takes row r's view
 *   direction.  dirs must be NULL iff the architecture has no view directions (NERFB200_ERR_INVALID otherwise).  impl
 *   codes, stash and refusals exactly as nerfb200_mlp_fwd (with n_samples the samples per row).
 * mlp_bwd_pts: its backward w.r.t. the parameters (impl 0 or 1), as nerfb200_mlp_bwd: it reads the encodings from the
 *   stash, so it takes no points; impl 1 reads the view directions again.  No gradient w.r.t. points or directions. */
int32_t nerfb200_mlp_fwd_pts(const nerfb200_arch_t* arch, const float* blob, const float* pts, const float* dirs,
                             int32_t dir_stride, int64_t n_rays, int32_t n_samples, float* raw, float* stash,
                             int32_t impl, void* stream);
int32_t nerfb200_mlp_bwd_pts(const nerfb200_arch_t* arch, const float* blob, const float* dirs, int32_t dir_stride,
                             int64_t n_rays, int32_t n_samples, const float* d_raw, const float* stash, float* gstash,
                             float* flat_grad, int32_t impl, void* stream);
/* volume_render_fwd: nerfb200_composite_fwd with the directions through (dirs, dir_stride): raw[n_rays][n_samples][4],
 *   z[n_rays][n_samples], 1 <= n_samples <= 1024, noise unit normals [n_rays][n_samples] or NULL.
 *   out[n_rays][8] = [r g b disp acc depth 0 0]; weights[n_rays][n_samples] may be NULL.
 * volume_render_bwd: its backward w.r.t. raw, taking every output: g_out[n_rays][8] = dL/d[r g b disp acc depth . .]
 *   (the depth slot included, unlike nerfb200_composite_bwd) and g_weights[n_rays][n_samples] = dL/dweights or NULL.
 *   Writes d_raw[n_rays][n_samples][4]. */
int32_t nerfb200_volume_render_fwd(const float* raw, const float* z, const float* dirs, int32_t dir_stride,
                                   const float* noise, int64_t n_rays, int32_t n_samples, float noise_std,
                                   int32_t white_bkgd, float* out, float* weights, void* stream);
int32_t nerfb200_volume_render_bwd(const float* raw, const float* z, const float* dirs, int32_t dir_stride,
                                   const float* noise, const float* g_out, const float* g_weights, int64_t n_rays,
                                   int32_t n_samples, float noise_std, int32_t white_bkgd, float* d_raw, void* stream);

/* ---- whole-path entry points ------------------------------------------------------------------- */

/* Workspace (device bytes) needed by nerfb200_render_fwd for n_rays rays; training adds the stashes. */
int64_t nerfb200_render_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                        const nerfb200_render_opts_t* opts, int64_t n_rays, int32_t training);

/* Byte offsets of the named sections inside the render workspace (test / debugging hook), in the
 * order z_coarse, raw_coarse, weights_coarse, z_fine, raw_fine, stash_coarse, stash_fine, gstash, d_raw. */
int32_t nerfb200_render_workspace_layout(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                         const nerfb200_render_opts_t* opts, int64_t n_rays, int32_t training,
                                         int64_t* offsets9);

/* ---- random numbers of the render path ---------------------------------------------------------
 * predict_and_render_radiance has four random inputs, in the reference's draw order (SURVEY.md section 5):
 *   stream 0 t_rand [n][nc]     uniform [0, 1), used when perturb is set
 *   stream 1 noise_c[n][nc]     unit normal,    used when noise_std > 0
 *   stream 2 u      [n][nf]     uniform [0, 1), used when perturb is set and n_fine > 0
 *   stream 3 noise_f[n][nc+nf]  unit normal,    used when noise_std > 0 and n_fine > 0
 * With perturb off the fine pass resamples at the det=True torch.linspace(0,1,nf), computed in the kernel.
 * Each input comes from a tensor the caller drew, or from the seeded stream: a pure function of (seed, step, stream,
 * global ray, sample), generated inside the kernels that use it.  That stream is Philox4x32-10 keyed by the seed,
 * counter (sample / 4, stream + 4 * step, global ray low 32 bits, high 32 bits).  Uniforms are (w >> 8) * 2^-24 in
 * [0, 1); normals are Box-Muller on word pairs with u1 = ((w >> 8) + 1) * 2^-24 (the exact definition is in
 * csrc/common.cuh).  A ray's numbers do not depend on how the batch is chunked or sharded. */
typedef struct nerfb200_rng {
  uint64_t seed;
  uint64_t step;      /* training step (< 2^30) */
  int64_t ray_offset; /* global index of the call's first ray (>= 0) */
} nerfb200_rng_t;

/* Materialises stream `stream_id` (0..3) for rays ray_offset .. ray_offset + n_rays - 1, samples 0 .. per_ray - 1:
 * out[n_rays][per_ray], uniforms for streams 0 and 2, unit normals for 1 and 3.  The numbers the render kernels use,
 * through the same device function: a render call given *rng equals one given these tensors. */
int32_t nerfb200_random_fill(const nerfb200_rng_t* rng, int32_t stream_id, int64_t n_rays, int32_t per_ray, float* out,
                             void* stream);

/* predict_and_render_radiance for one ray chunk (train_utils.py:28-127), and its backward.
 * Random inputs (streams above): rng non-NULL generates every one in-kernel, and then every random tensor pointer
 * must be NULL.  rng NULL reads the tensors t_rand, noise_c, u, noise_f, each only when the options use it: t_rand and
 * u must then be given, a noise tensor left NULL means no noise.  render_bwd needs the noise again for the sigma ReLU gate: pass it the same *rng,
 * or the same noise tensors, as the render_fwd call that filled the workspace (seeded, it reads no noise tensor).
 * render_fwd: out_coarse/out_fine[n][8] = [r g b disp acc depth 0 0] (out_fine NULL when n_fine == 0).
 *   impl: the MLP kernels as in nerfb200_mlp_fwd (0 fp32 CUDA cores, 1 wgmma, 3 single-pass fp16 wgmma; any other
 *   code is NERFB200_ERR_INVALID); impl 3 renders only: training = 1 is refused with NERFB200_ERR_UNSUPPORTED.
 *   Both calls check every network they will run before their first launch, so a refusal writes nothing.
 *   workspace: nerfb200_render_workspace_bytes(...) bytes; keeps z/raw/stash for render_bwd.
 * render_bwd: g_coarse/g_fine[n][8] upstream grads (g_fine NULL when no fine pass); accumulates into flat_grad_c /
 *   flat_grad_f (may alias different ranges of one buffer).  parts: bit 0 = the fine network's backward, bit 1 = the
 *   coarse network's (3 = both, fine first).  Two calls (1, then 2) let the host start the all-reduce of the fine
 *   network's gradient while the coarse backward runs. */
int32_t nerfb200_render_fwd(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                            const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                            const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                            const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                            float* out_coarse, float* out_fine, void* workspace, int32_t training, int32_t impl,
                            void* stream);
int32_t nerfb200_render_bwd(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                            const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                            const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                            const float* noise_c, const float* noise_f, const float* g_coarse, const float* g_fine,
                            void* workspace, float* flat_grad_c, float* flat_grad_f, int32_t impl, int32_t parts,
                            void* stream);

/* Fused Adam over a flat vector (torch.optim.Adam semantics, train_nerf.py:136-141,261-270):
 * p, m, v updated in place from g; step is the 1-based step count AFTER this update; grad_scale
 * multiplies g first (1/world_size after a summed all-reduce). */
int32_t nerfb200_adam_step(float* p, const float* g, float* m, float* v, int64_t n, int32_t step, float lr,
                           float beta1, float beta2, float eps, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERFB200_H_ */
