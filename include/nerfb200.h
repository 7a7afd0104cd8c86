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

/* ---- occupancy grid: inference renders that skip the MLP in empty space ---------------------------------------
 * A bitfield over the axis-aligned box [lo, hi) in the coordinates the MLP encodes (world space, or NDC for forward-facing
 * scenes), res[0] x res[1] x res[2] cells.  The cell of a point x, per axis c, all in fp32 with round-to-nearest:
 *     scale_c = (float)res[c] / (hi[c] - lo[c]);   t_c = (x_c - lo[c]) * scale_c
 * x is inside the box iff 0 <= t_c < res[c] on every axis (a NaN coordinate is outside); then i_c = (int)t_c and the
 * cell's index is  idx = (i_2 * res[1] + i_1) * res[0] + i_0  (x fastest).  The bitfield is uint32
 * words[nerfb200_grid_words(grid)], cell idx at bit (idx & 31) of word idx >> 5 (least significant bit first); a set bit
 * is an occupied cell.  A sample inside the box whose cell bit is clear is skipped; a sample outside the box is always
 * evaluated. */
typedef struct nerfb200_grid {
  float lo[3];
  float hi[3];
  int32_t res[3]; /* cells per axis, 1 .. 4096 */
} nerfb200_grid_t;
#define NERFB200_GRID_MAX_RES 4096

/* uint32 words of the grid's bitfield; -1 for an invalid descriptor (res outside 1 .. 4096, hi <= lo, non-finite). */
int64_t nerfb200_grid_words(const nerfb200_grid_t* grid);
/* Host restatement of the cell rule above (test hook): cell_out[i] = the cell index of point xyz_host[i][3], or -1 when
 * the point lies outside the box.  Host memory only. */
int32_t nerfb200_grid_locate(const nerfb200_grid_t* grid, const float* xyz_host, int64_t n, int64_t* cell_out);

/* Sample compaction of one pass (stage entry point and test hook).  For every sample s of ray r, the point
 * o + d z[r][s] is formed as the MLP forward forms it and looked up in the grid:
 *   - a skipped sample gets raw[r][s] = [0 0 0 -inf]: the compositing then gives it alpha = 0 and weight 0 exactly, with
 *     or without noise (-inf + noise * std = -inf, ReLU -> sigma 0, exp(-0 * delta) = 1);
 *   - the evaluated samples, in (ray, sample) order, become the rows of map[]: rays are taken in groups of 10
 *     consecutive rays (the most one 64-row MLP block may touch), each group's evaluated samples fill whole 64-row
 *     blocks, and the rows after a group's last sample up to its block's end hold -1 (padding).  map[row] = r * n_samples
 *     + s.  blocks[2 b], blocks[2 b + 1] = the first and last ray block b touches.
 * *n_blocks (device int32) = the number of blocks written, *n_evaluated (device int64, may be NULL) = evaluated samples.
 * Sizes: map int32[64 * nerfb200_grid_max_blocks(n_rays, n_samples)], blocks int32[2 * that];
 * scratch int32[nerfb200_grid_scratch_ints(n_rays, n_samples)].  Prefix sums throughout: the same inputs give the
 * same map.  No host synchronisation: the counts stay in device memory. */
int64_t nerfb200_grid_max_blocks(int64_t n_rays, int32_t n_samples);
int64_t nerfb200_grid_scratch_ints(int64_t n_rays, int32_t n_samples);
int32_t nerfb200_grid_compact(const nerfb200_grid_t* grid, const uint32_t* bits, const float* rays, int32_t ray_stride,
                              const float* z, int64_t n_rays, int32_t n_samples, float* raw, int32_t* map,
                              int32_t* blocks, int32_t* n_blocks, int64_t* n_evaluated, int32_t* scratch, void* stream);

/* nerfb200_render_fwd for inference (training = 0) with an occupancy grid: after each pass's depths, the compaction above
 * decides which samples run the MLP; the wgmma forward runs over the map only (impl 1 or 3; impl 0 is refused with
 * NERFB200_ERR_UNSUPPORTED) and writes raw[point] of each evaluated point, bit for bit what render_fwd computes for it.
 * The random inputs are those of render_fwd.  With every cell occupied the six outputs equal render_fwd's bit for bit.
 * workspace: nerfb200_render_grid_workspace_bytes(...) bytes; its first sections are those of render_fwd's inference
 * workspace (nerfb200_render_workspace_layout with training = 0).  n_evaluated: device int64[2] receiving the evaluated
 * samples of the coarse and the fine pass, or NULL. */
int64_t nerfb200_render_grid_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                             const nerfb200_render_opts_t* opts, int64_t n_rays);
int32_t nerfb200_render_fwd_grid(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                 const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                 const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                                 const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                                 const nerfb200_grid_t* grid, const uint32_t* bits, float* out_coarse, float* out_fine,
                                 void* workspace, int32_t impl, int64_t* n_evaluated, void* stream);

/* ---- early ray termination: inference renders that stop a ray's last pass once it is opaque ----------------------
 * nerfb200_render_fwd_early_stop is render_fwd for inference (impl 1 or 3), with or without an occupancy grid (grid and
 * bits both NULL: no grid), and a threshold t = stop_transmittance, 0 <= t < 1.
 *   - Only the last pass terminates: the fine pass when n_fine > 0, else the coarse pass.  The coarse pass of a two-pass
 *     render runs as render_fwd / render_fwd_grid run it, so its outputs, weights and the fine depths are bit-identical.
 *   - Rounds.  In the last pass a ray's evaluated samples are those the grid keeps (all of them without a grid).  They
 *     run the MLP in rounds, in sample order: round k takes evaluated samples k K .. k K + K - 1 (K = NERFB200_STOP_ROUND)
 *     of every ray still live, compacted as nerfb200_grid_compact compacts (groups of 10 rays, 64-row blocks).
 *   - Termination.  After each round in which a ray evaluated samples, its transmittance T is the fp32 product, in sample
 *     order, of the compositing's q = (1 - alpha) + 1e-10 over its samples evaluated so far, alpha from the same sigma
 *     gate, noise, delta and |d| as the compositing.  The ray stops when T < t (strict) and it has samples left to
 *     evaluate; each of those gets raw = [0 0 0 -inf].  With t = 0 no ray stops.
 *   - Outputs.  The last pass is composited as render_fwd composites it, over the full raw.  An evaluated sample's raw is
 *     bit for bit render_fwd's (a row's MLP result does not depend on its block).
 *   - Guarantee.  A ray that never stops gets render_fwd's outputs (render_fwd_grid's with a grid) bit for bit.  For a
 *     ray that stops, the weights left out sum to at most its T at the stop, which is below t: without a white
 *     background rgb and acc can only drop, by at most t, and depth by at most t * max z; with a white background rgb
 *     can only rise, by at most t.
 * stop_sample (device int32[n_rays], may be NULL): one past the last sample the ray evaluated when it stopped, so every
 * sample from there on that it would have evaluated was skipped by termination; n_samples of the pass if it never
 * stopped.  n_evaluated (device int64[2], may be NULL): the MLP rows each pass ran (the coarse pass of a two-pass render
 * without a grid runs all n_rays * n_coarse).  No host synchronisation: rounds after every ray has finished run empty.
 * Refused before any launch: impl 0 (NERFB200_ERR_UNSUPPORTED); t outside [0, 1) or NaN, an invalid grid, a grid without
 * bits or bits without a grid (NERFB200_ERR_INVALID); an architecture the wgmma inference forward refuses (its reason).
 * workspace: nerfb200_render_early_stop_workspace_bytes(...) bytes; its first sections are those of render_fwd's
 * inference workspace. */
#define NERFB200_STOP_ROUND 32
/* NERFB200_STOP_ROUND, for bindings that do not read this header */
int32_t nerfb200_render_early_stop_round(void);
int64_t nerfb200_render_early_stop_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                                   const nerfb200_render_opts_t* opts, int64_t n_rays);
int32_t nerfb200_render_fwd_early_stop(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                       const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                       const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                                       const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                                       const nerfb200_grid_t* grid, const uint32_t* bits, float stop_transmittance,
                                       float* out_coarse, float* out_fine, void* workspace, int32_t impl,
                                       int64_t* n_evaluated, int32_t* stop_sample, void* stream);

/* ---- meshes: marching cubes over a lattice of values -------------------------------------------------------------
 * The box is a nerfb200_grid_t read as res[c] cubes per axis; its lattice is the (res[0] + 1) x (res[1] + 1) x
 * (res[2] + 1) cube corners, point (i_0, i_1, i_2) at linear index (i_2 * n_1 + i_1) * n_0 + i_0 with n_c = res[c] + 1
 * (x fastest), at coordinates, per axis c, in fp32 with round-to-nearest and no contraction:
 *     p_c(i) = lo[c] + ((hi[c] - lo[c]) * (float)i) / (float)res[c]
 * volume[n_2][n_1][n_0] holds one fp32 value per lattice point.  A point is inside when its value exceeds `level` (NaN is
 * outside).  The lattice edge (q, a) runs from point q to its +1 neighbour along axis a; it crosses when exactly one of
 * its ends is inside, and then carries one vertex, at t = (level - v0) / (v1 - v0) from q:
 *     coordinate a = p_a(q_a) + t * (p_a(q_a + 1) - p_a(q_a)),  the other two = those of q   (fp32, each op rounded)
 * Vertex ids follow lattice-edge order: the crossing edges sorted by (linear index of q, a).  Each cube (named by its low
 * corner) takes its triangles from the face-consistent case table csrc/mc_table.cuh (generated by tools/gen_mc_table.py,
 * which states the corner and edge numbering): every face of a cube carries segments chosen by that face's four corner
 * signs alone (on a face with two diagonal inside corners the inside corners stay apart), so two cubes sharing a face
 * agree on it and the mesh is closed wherever the surface stays inside the lattice.  Faces are int32 vertex-id triples,
 * counter-clockwise seen from outside (the normal by the right-hand rule points from inside to outside), cube by cube in
 * linear order and, within a cube, in table order.  Prefix sums throughout, no atomics: the mesh is a function of the
 * volume and the level.
 *
 * mesh_lattice_points: pts[nz][n_1][n_0][3] = the lattice points of planes i_2 = z0 .. z0 + nz - 1 (the points a caller
 *   evaluates its field at; they depend on the lattice index alone, not on how the planes are split into calls).
 * mesh_workspace_bytes: device bytes of the workspace mesh_count fills and mesh_emit reads; -1 for an invalid box or
 *   more than 2^31 lattice points.
 * mesh_count: classify every lattice point (its crossing edges, and its cube's case) and scan: totals[0] = vertices,
 *   totals[1] = faces (device int64[2]).  The counts stay in device memory; a caller sizing the outputs reads them once.
 * mesh_emit: with the workspace of mesh_count on the same volume and level, writes vertices[V][3] and faces[F][3]
 *   (V, F = the totals; max_vertices, max_faces bound every write).  view_dirs[V][3] (may be NULL) receives, per vertex,
 *   the direction of a ray reaching it head-on from outside: the normalised density gradient, i.e. -n for the outward
 *   normal n.  The gradient at lattice point i is, per axis c, (v[i_hi] - v[i_lo]) / (h_c * (float)(i_hi - i_lo)) with
 *   i_lo = max(i_c - 1, 0), i_hi = min(i_c + 1, res[c]) (central differences, one-sided at the lattice's faces) and
 *   h_c = (hi[c] - lo[c]) / (float)res[c]; along the edge g = g0 + t * (g1 - g0) per component;
 *   s = (gx * gx + gy * gy) + gz * gz; dir = g / sqrt(s) when 0 < s < inf, else (0, 0, 1).  All fp32, each op rounded. */
int64_t nerfb200_mesh_workspace_bytes(const nerfb200_grid_t* box);
int32_t nerfb200_mesh_lattice_points(const nerfb200_grid_t* box, int32_t z0, int32_t nz, float* pts, void* stream);
int32_t nerfb200_mesh_count(const nerfb200_grid_t* box, const float* volume, float level, void* workspace,
                            int64_t* totals, void* stream);
int32_t nerfb200_mesh_emit(const nerfb200_grid_t* box, const float* volume, float level, const void* workspace,
                           int64_t max_vertices, int64_t max_faces, float* vertices, int32_t* faces, float* view_dirs,
                           void* stream);

/* ---- sparse meshes: marching cubes over the bricks an occupancy grid calls occupied ------------------------------
 * The lattice, its values, the vertex rule, the case table and the winding are those of "meshes" above; only the cubes
 * that are marched, and so the numbering, differ.  A lattice point depends on its index alone, so the sparse path
 * evaluates exactly the points (and gets exactly the values) the dense path would at the same indices.
 *   - Bricks.  Brick (b_0, b_1, b_2), b_c = 0 .. ceil(res[c] / B) - 1 with B = NERFB200_MESH_BRICK, holds the cubes
 *     whose low corner q has floor(q_c / B) = b_c; its corner points are the lattice points i with b_c B <= i_c <=
 *     min(b_c B + B, res[c]) (bricks on the box's upper faces are partial).  Brick index (b_2 * nb_1 + b_1) * nb_0 + b_0,
 *     x fastest.  Brick indices are int32 (at most 512^3 bricks).
 *   - Activity.  A brick is active when one of its corner points, at the fp32 coordinates p_c(i) of "meshes", lies
 *     outside the grid's box or in an occupied cell under the cell rule of "occupancy grid" (a point outside the box is
 *     always evaluated by renders too).  The cell rule is separable per axis, so the library tests each distinct cell
 *     the corners' axis cells combine to; the result is exactly that of the point rule.
 *   - Output.  The faces are those of the dense mesh over the same values and level restricted to the cubes of active
 *     bricks; the vertices are the crossing edges those cubes use, with bit-identical coordinates (and view
 *     directions).  Each crossing edge carries one vertex, owned by the lowest-index active brick with a cube using the
 *     edge.  Vertex ids run by owning brick, then by (linear lattice index of q, a) within it; faces by brick, then by
 *     cube linear index, then in table order.  Prefix sums throughout, no atomics: the mesh is a function of the values,
 *     the level and the grid.  If no face of the dense mesh lies in a cube of an inactive brick, the sparse mesh is the
 *     dense mesh up to this renumbering.
 *   - Values are brick-major over the active bricks in slot order: slot s holds P = p1^3 values, p1 = B + 1 + 2 halo,
 *     corner point l (0 .. B per axis, lattice index b B + l) at s * P + ((l_2 + halo) * p1 + l_1 + halo) * p1 + l_0 + halo.
 *     halo = 1 adds the points one outside the brick, which the view directions' central differences read; there a
 *     lattice index outside 0 .. res[c] is clamped onto the lattice (those values are never read).
 *   - Memory.  brick_map and the brick list are int32 per brick of the box; the scratch of mesh_sparse_bricks is
 *     three axis tables of 4097 int32 and 20 bytes per 256 bricks; everything else is per active brick: P values and
 *     mesh_sparse_workspace_bytes (392 bytes per brick).
 *
 * mesh_brick: B.  mesh_sparse_brick_count: bricks of the box (-1 for an invalid box).
 * mesh_sparse_bricks: the activity test and its compaction.  brick_map[brick] = the brick's slot (its rank among the
 *   active bricks, in brick order) or -1; bricks[slot] = brick (int32[mesh_sparse_brick_count], the first *n_active
 *   written); *n_active (device int64) = the count.  scratch: mesh_sparse_scratch_bytes(box) device bytes.
 * mesh_sparse_bricks_host: the activity test on the host (test hook): active[brick] = 0 / 1, host memory only.
 * mesh_sparse_points: pts[count * P][3] = the lattice points of slots first .. first + count - 1 in value order.
 * mesh_sparse_count / _emit: mesh_count / mesh_emit over the active bricks' values.  totals[0] = vertices, totals[1] =
 *   faces (device int64[2]).  view_dirs (may be NULL; needs halo = 1) as in mesh_emit; edge_keys (int64[V], may be
 *   NULL) = q * 3 + a of each vertex's lattice edge, q its low end's linear lattice index.
 * Refused before any launch: an invalid box or grid, a null pointer, halo other than 0 / 1, a non-finite level, an
 * active count outside 0 .. the box's bricks. */
#define NERFB200_MESH_BRICK 8
int32_t nerfb200_mesh_brick(void);
int64_t nerfb200_mesh_sparse_brick_count(const nerfb200_grid_t* box);
int64_t nerfb200_mesh_sparse_scratch_bytes(const nerfb200_grid_t* box);
int64_t nerfb200_mesh_sparse_workspace_bytes(const nerfb200_grid_t* box, int64_t n_active);
int32_t nerfb200_mesh_sparse_bricks(const nerfb200_grid_t* box, const nerfb200_grid_t* grid, const uint32_t* bits,
                                    int32_t* brick_map, int32_t* bricks, int64_t* n_active, void* scratch,
                                    void* stream);
int32_t nerfb200_mesh_sparse_bricks_host(const nerfb200_grid_t* box, const nerfb200_grid_t* grid,
                                         const uint32_t* bits_host, uint8_t* active_host);
int32_t nerfb200_mesh_sparse_points(const nerfb200_grid_t* box, const int32_t* bricks, int64_t first, int64_t count,
                                    int32_t halo, float* pts, void* stream);
int32_t nerfb200_mesh_sparse_count(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                   int64_t n_active, const float* values, int32_t halo, float level, void* workspace,
                                   int64_t* totals, void* stream);
int32_t nerfb200_mesh_sparse_emit(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                  int64_t n_active, const float* values, int32_t halo, float level,
                                  const void* workspace, int64_t max_vertices, int64_t max_faces, float* vertices,
                                  int32_t* faces, float* view_dirs, int64_t* edge_keys, void* stream);

/* ---- density gradient: sigma and its gradient w.r.t. the points (normals, field probes) -------------------------
 * density_grad: out[P][4] = (sigma_raw, d sigma_raw / dx, d / dy, d / dz) at pts[P][3], P >= 1 and < 2^31.  sigma_raw is
 *   the network's sigma output before the ReLU (fc_alpha, or column 3 of fc_out without view directions), bit for bit
 *   what nerfb200_mlp_fwd_pts with impl 1 writes to raw[p][3] at the same point; sigma reads no view direction, so none
 *   is taken.  The gradient is w.r.t. the coordinates the MLP encodes (world space for Blender scenes, NDC for LLFF):
 *   the exact chain rule of the trunk (layer1 without, the other trunk layers with their ReLU; a ReLU's derivative is
 *   1 where its output is nonzero) and of the positional encoding (d sin(f x) = f cos(f x), d cos(f x) = -f sin(f x), the
 *   argument f x rounded to fp32 as the forward rounds it), each product in the forward's three-term fp16 split with
 *   fp32 accumulation.  Inference only (no backward); impl 1 alone: impl 0 and 3 are refused.  An operand out of the
 *   fp16 range gives inf / NaN, not a clamped value.
 * density_grad_supported: NERFB200_OK if density_grad runs this architecture with `impl`, else the reason (the last
 *   error), without touching a device.
 * The surface normal of a level set of sigma is -grad / |grad| (outward: toward lower density).  "NDC scenes" below maps
 * an NDC gradient to world space. */
int32_t nerfb200_density_grad_supported(const nerfb200_arch_t* arch, int32_t impl);

/* ---- normal maps: the composited surface normal of an inference render's last pass ------------------------------
 * render_fwd_normals: render_fwd for inference (training = 0) -- with an occupancy grid when grid / bits are given, and
 *   with early ray termination of the last pass when stop_transmittance >= 0 (negative: none; NaN is refused) -- whose
 *   out_coarse / out_fine are bit for bit those of nerfb200_render_fwd, _fwd_grid or _fwd_early_stop on the same
 *   inputs, plus normals[n_rays][3] of the last pass (the fine pass, or the coarse pass of a coarse-only network):
 *     n_i = -g_i / |g_i| at the last pass's sample i, g_i = density_grad's gradient at the point o + d z_i formed as the
 *         MLP forms it; |g| = sqrt((gx * gx + gy * gy) + gz * gz), n_i = 0 where that is 0 (fp32, each op rounded);
 *     N = sum over the samples with w_i != 0, in sample order, of w_i * n_i (fp32, each op rounded), w_i the weights the
 *         render's own compositing of that pass computed (with its noise, when noise_std > 0).
 *   N is not renormalised: |N| <= acc up to rounding, and N = 0 for a ray whose weights are all 0.  The gradient is
 *   evaluated at the samples with a nonzero weight alone, compacted on the device (no host read); with a grid or early
 *   stopping every such sample ran the MLP.  impl 1 alone (density_grad's refusal for impl 0 and 3), before any launch.
 * render_normals_workspace_bytes: bytes of the workspace render_fwd_normals takes (-1 on invalid arguments); its first
 *   sections are laid out as nerfb200_render_workspace_layout(..., training = 0). */
int64_t nerfb200_render_normals_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                                const nerfb200_render_opts_t* opts, int64_t n_rays);
int32_t nerfb200_render_fwd_normals(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                    const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                    const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                                    const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                                    const nerfb200_grid_t* grid, const uint32_t* bits, float stop_transmittance,
                                    float* out_coarse, float* out_fine, float* normals, void* workspace, int32_t impl,
                                    void* stream);
int32_t nerfb200_density_grad(const nerfb200_arch_t* arch, const float* blob, const float* pts, int64_t n_points,
                              float* out, int32_t impl, void* stream);

/* ---- NDC scenes: world-space geometry of forward-facing scenes --------------------------------------------------
 * A forward-facing (LLFF) scene's MLP encodes NDC points: ray generation with ndc != 0 applies ndc_rays(H, W, focal,
 * 1.0, ...) (nerf_helpers.py:170-197), which maps a world point p with p_z < 0 to the point q the MLP encodes,
 *     N(p):  q_x = (sw * p_x) / p_z,   q_y = (sh * p_y) / p_z,   q_z = 1 + 2 / p_z,
 * with sw = fp32(-1 / (W / (2 focal))) and sh = fp32(-1 / (H / (2 focal))) evaluated in double and rounded once,
 * exactly as nerfb200_gen_rays / pack_rays compute them (W, H the image's width and height as integers, focal the fp32
 * focal length).  Every formula below is fp32 with round-to-nearest, each op rounded, in the order written (no
 * contraction):
 *   - inverse (defined for q_z < 1; q_z = 1 is the far plane at infinity):
 *         p_z = 2 / (q_z - 1),   p_x = (q_x * p_z) / sw,   p_y = (q_y * p_z) / sh;
 *   - gradient: the world gradient of a field sigma(N(p)) is J^T(q) g for its NDC gradient g,
 *         s = (q_z - 1) * 0.5,   G_x = s * (sw * g_x),   G_y = s * (sh * g_y),
 *         G_z = s * (-((q_x * g_x) + (q_y * g_y)) - ((q_z - 1) * g_z));
 *     s = 1 / p_z is negative inside the frustum, so it flips the direction as well as scaling it;
 *   - orientation: det J = -2 sw sh / p_z^4 < 0, so N reverses orientation.  N is projective, so a straight edge stays
 *     straight and a triangle mesh extracted in NDC is exactly a triangle mesh in world space once each face's second
 *     and third vertex ids are swapped (faces stay counter-clockwise seen from outside).
 * The unit world direction of a vector v is the rule of mesh_emit's view directions: l = (v_x * v_x + v_y * v_y) +
 * v_z * v_z; v / sqrt(l) when 0 < l < inf, else (0, 0, 1).
 *
 * ndc_mesh_to_world: one pass over a mesh extracted in NDC (mesh_emit / mesh_sparse_emit): world_vertices[i] =
 *   N^-1(vertices[i]); world_faces[f] = (faces[f][0], faces[f][2], faces[f][1]); world_dirs[i] = the unit world direction
 *   of J^T(vertices[i]) view_dirs[i] (view_dirs / world_dirs both NULL, or both given).  Each output may be its input.
 * ndc_from_world: q[i] = N(p[i]) for p[n][3] (p_z < 0 for a meaningful result; not checked on the device).
 * ndc_grad_to_world: rows[n][4] = (sigma, g_x, g_y, g_z) as density_grad writes them at the NDC points q[n][3];
 *   out[n][4] = (sigma, J^T(q) g), sigma copied.  out may be rows.
 * render_fwd_normals_ndc: render_fwd_normals of an NDC render (rays from gen_rays / pack_rays with ndc != 0 and this
 *   H, W, focal) with the normal map in world space: each sample's gradient g_i is replaced by J^T(q_i) g_i at the
 *   sample's NDC point q_i = o + d z_i BEFORE it is normalised and weighted; the sums, outputs, refusals and workspace are
 *   render_fwd_normals'.
 * Refused before any launch: a null ndc, height or width <= 0, focal not finite and > 0, a null pointer where one is
 * needed, a negative count (NERFB200_ERR_INVALID).  No atomics, no host synchronisation. */
typedef struct nerfb200_ndc {
  int32_t height;
  int32_t width;
  float focal;
} nerfb200_ndc_t;
int32_t nerfb200_ndc_mesh_to_world(const nerfb200_ndc_t* ndc, const float* vertices, const int32_t* faces,
                                   const float* view_dirs, int64_t n_vertices, int64_t n_faces, float* world_vertices,
                                   int32_t* world_faces, float* world_dirs, void* stream);
int32_t nerfb200_ndc_from_world(const nerfb200_ndc_t* ndc, const float* p, int64_t n, float* q, void* stream);
int32_t nerfb200_ndc_grad_to_world(const nerfb200_ndc_t* ndc, const float* q, const float* rows, int64_t n, float* out,
                                   void* stream);
int32_t nerfb200_render_fwd_normals_ndc(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                        const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                        const float* rays, int32_t ray_stride, int64_t n_rays,
                                        const nerfb200_rng_t* rng, const float* t_rand, const float* noise_c,
                                        const float* u, const float* noise_f, const nerfb200_grid_t* grid,
                                        const uint32_t* bits, float stop_transmittance, const nerfb200_ndc_t* ndc,
                                        float* out_coarse, float* out_fine, float* normals, void* workspace,
                                        int32_t impl, void* stream);

/* ---- baked fields: a trained network sampled once on the bricks of a lattice, rendered without the MLP ------------
 * The box and its lattice are those of "meshes"; the bricks, their activity under an occupancy grid, their slots and the
 * point order inside a brick are those of "sparse meshes" with halo = 0 (P = 9^3 = 729 points per brick, corner point l
 * of slot s at row s * 729 + (l_2 * 9 + l_1) * 9 + l_0, lattice index b B + l clamped onto 0 .. res).  The field lives in
 * the coordinates the MLP encodes (world space for Blender scenes, NDC for LLFF scenes).
 *   - Directions.  D = NERFB200_BAKE_DIRS = 64 on a spherical Fibonacci lattice: for i = 0 .. 63, z = 1 - (2 i + 1) / 64,
 *     r = sqrt(1 - z^2), phi = i pi (3 - sqrt 5), d_i = (r cos phi, r sin phi, z), in fp64, rounded once to fp32.
 *   - Basis.  Real spherical harmonics of degree <= 2, 9 functions of a unit vector (x, y, z):
 *       Y_0 = 0.28209479177387814,
 *       Y_1 = -0.4886025119029199 y,  Y_2 = 0.4886025119029199 z,  Y_3 = -0.4886025119029199 x,
 *       Y_4 = 1.0925484305920792 x y,  Y_5 = -1.0925484305920792 y z,  Y_6 = 0.31539156525252005 (2 z^2 - x^2 - y^2),
 *       Y_7 = -1.0925484305920792 x z,  Y_8 = 0.5462742152960396 (x^2 - y^2).
 *     (Y_1..Y_3 carry the Condon-Shortley sign of the complex harmonics they are made from.)  The projection
 *     M = (Y^T Y)^-1 Y^T (9 x 64), Y[i][j] = Y_j(d_i) in fp64 at the fp32 directions, is computed in fp64 by the
 *     library and rounded once to fp32.  bake_basis returns the directions and M.
 *   - Values.  values[slot][729][32] fp32 (128 B per lattice point, NERFB200_BAKE_CHANNELS):
 *       [0]          sigma_raw: the bits nerfb200_mlp_fwd_pts with impl 1 writes to raw[p][3] at that point;
 *       [1 + 9 c + j] the coefficient of Y_j of colour channel c's PRE-sigmoid logit: acc = 0, then for d = 0 .. 63 in
 *                    order acc = fmaf(M[j][d], logit_c(d), acc), logit_c(d) the bits mlp_fwd_pts with impl 1 writes to
 *                    raw[p][c] at the point with view direction d_d.  Without view directions coefficient 0 is
 *                    logit_c / Y_0 (fp32) and the others are 0;
 *       [28 .. 31]   0.
 *   - Rendering (baked_render).  Rays are rows [o(3) d(3) near far (viewdir(3))] as gen_rays / pack_rays write them.
 *     All fp32 with round-to-nearest, each op rounded, no contraction unless fmaf is named.
 *       interval  [t_a, t_b] = [near, far] intersected with the box's slab interval (per axis (lo - o) / d and
 *                 (hi - o) / d, fminf / fmaxf order).  An axis with d_c = +-0 has x_c = o_c at every sample: it leaves
 *                 the interval as it is when lo_c <= o_c < hi_c and makes the ray empty otherwise (o_c NaN included);
 *                 h = min over c of (hi_c - lo_c) / res_c, |d| = sqrt((dx dx + dy dy) + dz dz),
 *                 dt = (0.5 h) / |d|; sample k is t_k = t_a + (k + 0.5) dt for every k with t_k < t_b.
 *       lookup    x = o + d t_k, per axis as the MLP forms its points; its cube i is the cell of x under the cell rule of
 *                 "occupancy grid" applied to the box (t_c = (x_c - lo_c) scale_c, i_c = (int) t_c), f_c = t_c - i_c; the
 *                 brick floor(i / 8) and brick_map give the slot.  A sample outside the box, or in a brick whose slot is
 *                 -1, has sigma_raw = 0 and colour 0.
 *       interp    channels 0 .. 27 trilinear over the cube's 8 corners k = 0 .. 7 (corner offset (k & 1, k >> 1 & 1,
 *                 k >> 2), point l + offset of the brick), weight w_k = (w_x w_y) w_z with w_c = f_c for offset 1 and
 *                 1 - f_c for 0; v = 0, then v = fmaf(w_k, value_k, v) for k = 0 .. 7.
 *       colour    with view directions s_c = sum over j = 0 .. 8 of Y_j(viewdir) coef_cj (acc = 0, acc = fmaf(Y_j, coef_cj,
 *                 acc), Y_j in fp32 from the constants above as written, x x etc. rounded), without them s_c = Y_0 coef_c0;
 *                 rgb_c = 1 / (1 + exp(-s_c)).
 *       composite alpha and q = (1 - alpha) + 1e-10 as the library's compositing (volume_render_radiance_field) forms
 *                 them with noise 0 and z_next = t_k + dt for every sample (no 1e10 last interval).  Samples go in rounds
 *                 of 32; in a round, lane L's transmittance is T_round times the exclusive product scan of q over the
 *                 round's lanes (Hillis-Steele order), w = alpha T, and T_next = (T_lane 31) q_31.  rgb, acc = sum w and
 *                 depth = sum w t are summed in sample order; disp = 1 / max(1e-10, depth / acc) (NaN when acc = 0, as
 *                 composite_fwd); a white background adds 1 - acc to rgb.  out[n_rays][8] = [r g b disp acc depth 0 0].
 *       stopping  stop_transmittance t in [0, 1): after each round the ray stops once T < t.  t = 0 never stops, and a ray
 *                 that does not stop gets the t = 0 outputs bit for bit; for a ray that stops the weights left out sum
 *                 to less than t.
 *
 * bake_basis: dirs_host[64][3], proj_host[9][64] (host memory).
 * bake_supported: NERFB200_OK if bake runs this architecture, else the reason (the last error), without a device.  The
 *   wgmma inference forward's refusals apply (NERFB200_ERR_UNSUPPORTED); hidden 128 or 256, with or without view
 *   directions.
 * bake: the values of slots first .. first + count - 1 (bricks from mesh_sparse_bricks) into values + slot * 729 * 32.
 *   logits (test hook, may be NULL): logits[(slot - first) * 729 + l][64][3] = logit_c(d).  count * 729 < 2^31.
 * baked_render: the rendering above; brick_map from mesh_sparse_bricks over the same box, values from bake.
 *   ray_stride >= 11 with view directions, >= 8 without.
 * Refused before any launch: an invalid box, a null pointer, a count or range outside the box's bricks, an architecture
 * bake_supported refuses, t outside [0, 1) or NaN.  No atomics, no host synchronisation. */
#define NERFB200_BAKE_DIRS 64
#define NERFB200_BAKE_SH 9
#define NERFB200_BAKE_CHANNELS 32
int32_t nerfb200_bake_basis(float* dirs_host, float* proj_host);
int32_t nerfb200_bake_supported(const nerfb200_arch_t* arch);
int32_t nerfb200_bake(const nerfb200_arch_t* arch, const float* blob, const nerfb200_grid_t* box, const int32_t* bricks,
                      int64_t first, int64_t count, float* values, float* logits, void* stream);
int32_t nerfb200_baked_render(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                              int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                              int32_t white_background, float stop_transmittance, float* out, void* stream);

/* ---- baked fields: gradients and fine-tuning -------------------------------------------------------------------------
 * The gradient of baked_render (stop_transmittance 0) with respect to the values, the tie that keeps every stored copy
 * of a lattice point equal, and an Adam step over the values, so a baked field can be fine-tuned on images through its
 * own renderer (as PlenOctrees / SNeRG fine-tune theirs).  All fp32, each op rounded, no contraction.
 *   - Backward (baked_render_bwd).  One warp per ray re-marches the ray exactly as baked_render does (interval, t_k,
 *     lookup, interp, colour, alpha, q, T in rounds of 32).  out is the forward's [n][8] rows, g_out the upstream
 *     gradient rows in the same layout [g_r g_g g_b g_disp g_acc g_depth - -].  Per ray:
 *       G_acc = g_acc, G_depth = g_depth; a white background adds -(g_r + g_g + g_b) to G_acc; when g_disp != 0 and
 *       ratio = depth / acc is > 1e-10 or NaN, disp = 1 / ratio, G_depth += g_disp (-disp disp) / acc and G_acc +=
 *       g_disp (disp disp) depth / (acc acc) (the compositing backward's rule, one shared device function);
 *       E = (((g_r r' + g_g g') + g_b b') + G_acc acc) + G_depth depth from the forward's totals, r' = r - (1 - acc) etc.
 *       with a white background.
 *     Per sample (c its rgb, w = alpha T): v = (((g_r c_r + g_g c_g) + g_b c_b) + G_acc) + G_depth t;
 *       P = the running sum of w v in sample order, this sample included (one fp32 add per sample, lane order);
 *       dL/dalpha = T v - (E - P) / q;  dsigma_raw = gate ? (dL/dalpha delta) exp(-sigma delta) : 0;
 *       d s_c = ((w g_c) c_c) (1 - c_c);  d coef_cj = d s_c Y_j with view directions; without them d coef_c0 = d s_c Y_0
 *       and the other coefficients receive 0.
 *     S = E - P stands for the suffix sum over later samples that composite_bwd forms by a reverse pass (the baked
 *     renderer stores no samples).  It carries the rounding of E and of the prefix's adds, a few ulps of E, where the true
 *     suffix of a saturated ray is ~0; dsigma sees that error times delta exp(-sigma delta) / q <= delta.  Corner k of
 *     the sample's cube receives fp32(w_k x) of each of the 28 channel gradients x, added into d_values (layout of
 *     values; channels 28 .. 31 receive nothing) with vector fp32 reductions, seven float4 per corner, which flush
 *     subnormal sums to zero as every fp32 atomic add on sm_90 does.  A sample outside the box, in an inactive brick, or
 *     with a closed gate and w = 0 adds nothing.  The order of the reductions is the order the hardware runs them in:
 *     the raw gradients may differ in the last bits between runs (bit-reproducible baked gradients are not offered); the
 *     tie below keeps the field's copies equal whatever those bits are.  d_values is added into, so chunks of rays
 *     accumulate; zero it first.
 *   - Tie (baked_tie).  A lattice point on a brick face is stored once per active brick holding it, and on the box's upper
 *     faces the clamp of b B + l onto 0 .. res stores it again under several l of one brick.  Along one axis the copies
 *     of lattice index q are, in ascending brick order: for q < res, (q / 8 - 1, l = 8) when q is a positive multiple of
 *     8, then (q / 8, q mod 8); for q = res, (nb - 1, l) for l = res - 8 (nb - 1) .. 8.  A point's stored copies are the
 *     products of its three axes' lists (z outer, then y, then x) whose brick is active.  d_tied[copy] = 0, then += each
 *     copy's d_values in that order; channels 28 .. 31 are written 0.  Every copy of a point sums the same terms in the
 *     same order, so every copy gets the same bits; an elementwise optimiser (baked_adam_step_dev, torch.optim.Adam) then
 *     keeps copies that start bit-equal (as the bake writes them) bit-equal.  Out of place: d_values must not overlap
 *     d_tied.
 *   - Adam (baked_adam_step_dev).  adam_step_dev's update of step *step_dev + 1 with grad_scale 1 over values[n_active]
 *     [729][32]: channel 0 (sigma_raw) at rate lr_schedule(lr_sigma), channels 1 .. 27 at rate lr_schedule(lr_sh), the
 *     same lr_decay / lr_decay_factor: on each channel group the bits adam_step_dev gives at that rate.  Channels 28 .. 31
 *     of values, m and v are not touched.  The step counter is not advanced (step_advance does that).
 * Refused before any launch: an invalid box, a null pointer, n_rays <= 0, ray_stride < 11 with view directions (< 8
 * without), n_active outside 1 .. the box's bricks (tie; <= 0 for Adam), d_values overlapping d_tied, rates or a
 * schedule adam_step_dev refuses.  No host synchronisation. */
int32_t nerfb200_baked_render_bwd(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                  int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                  int32_t white_background, const float* out, const float* g_out, float* d_values,
                                  void* stream);
int32_t nerfb200_baked_tie(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks, int64_t n_active,
                           const float* d_values, float* d_tied, void* stream);
int32_t nerfb200_baked_adam_step_dev(float* values, const float* g, float* m, float* v, int64_t n_active,
                                     const int64_t* step_dev, double lr_sigma, double lr_sh, double lr_decay,
                                     double lr_decay_factor, float beta1, float beta2, float eps, void* stream);

/* ---- baked fields: pruning ------------------------------------------------------------------------------------------
 * Which active bricks a baked field's renders use, so that the others can be dropped (as PlenOctrees prunes voxels
 * whose largest rendering weight over the training rays is small).  Dropping bricks is host-side compaction of the
 * field (brick_map, bricks, values); the library supplies each brick's peak weight over a set of rays.
 *   - Peak weights (baked_max_weights).  One warp per ray re-marches the ray exactly as baked_render does with
 *     stop_transmittance 0: the same interval, t_k, lookup, alpha, q and T in rounds of 32 with the same Hillis-Steele
 *     scan.  For every sample whose slot is >= 0, max_w[slot] = max(max_w[slot], w), w = alpha T the bits the renderer
 *     forms for that sample; a NaN w is recorded as +inf, so that brick survives any finite threshold.  w depends on
 *     sigma_raw alone, so only channel 0 is interpolated: the 8 corners in the same order through the same fmaf chain as
 *     the renderer's interp, which gives the renderer's sigma_raw bits while reading 4 B of each 128-B point; no colour
 *     or SH is formed.  A ray is marched to t_b (no stop at T = 0: a NaN later in the ray must still be seen).
 *     max_w is fp32[n_active] and max-accumulated: zero it once and pass it to every chunk of rays.  A max is exact, so
 *     the result is the same bits for every chunking, ray order and run.
 *   - Transparent bricks.  A brick every stored sigma_raw of which is <= 0 (-0 included) and whose channels 0 .. 27 are
 *     all finite can be dropped (its brick_map entry set to -1) leaving every render bit for bit the same, from any ray,
 *     with or without a white background or early stopping.  Every sample in such a brick interpolates sigma_raw <= 0
 *     (non-negative weights times non-positive values), so sigma = 0, alpha = +0 and q = (1 - 0) + 1e-10 = 1 exactly
 *     (1e-10 is below half an ulp of 1): T passes unchanged, w = +0, and w rgb and w t are +-0, which leave every sum
 *     (each starts at +0) unchanged.  A dropped sample is a miss, which has the same alpha, q and w, and a round whose
 *     lanes all miss (skipped by the renderer) is equivalent to one in which they hit such a brick.  Normal maps
 *     (baked_render_normals) stay the same bits too: such samples have w = +0 and are skipped by the normal sum, as
 *     they add nothing to the colour sums ("baked fields: normal maps and point queries").
 *   - Unseen bricks.  A brick with max_w == 0 over a set of rays can be dropped leaving the renders of those rays bit
 *     for bit the same (with or without early stopping: the march agrees at every round).  A dropped sample had w = +0,
 *     so either alpha = 0 (q = 1 as for a miss) or T = 0 before it; T is a product of factors q in [1e-10, 1], so once
 *     it is 0 it stays 0 when the dropped q becomes 1, and every later sample keeps w = +0.  The one exception is a
 *     product that rounds to 0 exactly at the fp32 underflow boundary: alpha > 0 and T > 0 with alpha T (or a partial
 *     product of the scan) below 2^-150, so 0 under one association and not under the other.  T is then subnormal and
 *     the later weights that can differ are below 2^-126.
 *   - Non-finite fields.  Both statements hold for finite fields only.  A NaN or infinite coefficient in a brick whose
 *     samples have w = 0 still makes the render NaN (0 NaN and 0 inf are NaN), and dropping that brick changes it; the
 *     transparency rule therefore asks that channels 0 .. 27 be finite, and a NaN w keeps its brick through +inf.
 * baked_max_weights: box, brick_map, values, rays and ray_stride as baked_render; max_w[n_active] fp32.
 * Refused before any launch: an invalid box, a null pointer, n_rays <= 0, ray_stride < 11 with view directions (< 8
 * without).  No host synchronisation; the only atomics are integer atomicMax on the bits of non-negative floats (which
 * order as unsigned integers): per round the lanes are grouped by slot (__match_any_sync), each group's largest weight
 * found by __reduce_max_sync, and one lane per group issues the atomic; w = 0 is skipped, as max_w starts at 0. */
int32_t nerfb200_baked_max_weights(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                   int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                   float* max_w, void* stream);

/* ---- baked fields: half precision ----------------------------------------------------------------------------------
 * A baked field whose values are stored in IEEE binary16, at half the bytes of the fp32 field, for fields that are kept,
 * saved, rendered and pruned (PlenOctrees and SNeRG ship their fields in half precision).  Fine-tuning stays fp32: the
 * fp16 entry points have no gradient, tie, Adam or regulariser twins; fine-tune the widened field and convert it back.
 *   - Layout.  values[slot][729][32] binary16 (64 B per lattice point), the bits as uint16_t; the channels mean what they
 *     mean in the fp32 field ("baked fields"), channels 28 .. 31 are 0.
 *   - Conversion rule, fp32 -> fp16 channel by channel: a finite x with |x| > 65504 saturates to +-65504, then every
 *     finite value is rounded to nearest even; +-inf and NaN stay +-inf and NaN (the NaN payload is not specified).  No
 *     finite value becomes an infinity the fp32 field did not have (a -inf corner would make the trilinear sum -inf or
 *     NaN).  In torch: torch.where(x.isfinite(), x.clamp(-65504, 65504), x).half(), the same bits.
 *   - Rendering and peak weights (baked_render_f16, baked_max_weights_f16).  Each value is widened exactly to fp32 as it
 *     is gathered; every other op is the fp32 rule of "baked fields" and "baked fields: pruning": the same corners in the
 *     same order through the same fmaf chain.  An fp16 field therefore renders, and gives peak weights, bit for bit like
 *     the fp32 field holding its widened values.  A corner's channels 0 .. 27 are three 16-B loads and one 8-B load (56
 *     of its 64 B); the peak weights read sigma_raw alone, 2 B per corner.
 *   - Bake (bake_f16).  The fp32 bake's values with the conversion rule applied at the store: bit-equal to converting
 *     bake's output (NaN compared as a class).  The logits test hook stays fp32.
 * bake_f16, baked_render_f16, baked_max_weights_f16: the arguments of bake, baked_render and baked_max_weights, values
 *   binary16.  Refused before any launch: whatever their fp32 twins refuse (the same checks), and a values pointer that
 *   is not 16-B aligned. */
int32_t nerfb200_bake_f16(const nerfb200_arch_t* arch, const float* blob, const nerfb200_grid_t* box,
                          const int32_t* bricks, int64_t first, int64_t count, uint16_t* values, float* logits,
                          void* stream);
int32_t nerfb200_baked_render_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                  int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                  int32_t white_background, float stop_transmittance, float* out, void* stream);
int32_t nerfb200_baked_max_weights_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                       int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                       float* max_w, void* stream);

/* ---- baked fields: regularisers -------------------------------------------------------------------------------------
 * Squared total variation of the density and of the SH coefficients over the lattice, and a Cauchy sparsity term on the
 * density (as Plenoxels regularises its voxels), with their gradient in the tie's convention, so that fine-tuning can
 * trade fitting the training views for a smoother, emptier field.
 *   - Lattice points.  The points q of 0 .. res (per axis) with at least one stored copy in an active brick, the copies
 *     enumerated as the tie enumerates them ("baked fields: gradients and fine-tuning").  P is their number.
 *   - Canonical copy.  A point's first copy in the tie's order (z outer, then y, then x, bricks ascending) whose brick is
 *     active.  Every value read below is read at the canonical copy of its point, so the result does not depend on which
 *     copy a thread holds, even if copies differ.
 *   - Edges.  The pairs (q, q + e_c) with q_c + 1 <= res_c such that an active brick holds both points: brick q_c / 8
 *     along c (the only brick whose points 8 b .. min(8 b + 8, res) hold q_c and q_c + 1) and, along each other axis a,
 *     any brick of q_a's copy list (at most two distinct bricks, so at most 4 candidates in brick_map).  The clamped
 *     repeats on the upper faces are one point and never form an edge.
 *   - Loss.  With v_ch channel ch of a point, sigma = v_0 and sigma+ = max(sigma, 0):
 *       L = (1 / P) [ l_sigma sum_edges (d sigma)^2 + l_sh sum_edges sum_{ch = 1 .. 27} (d v_ch)^2
 *                     + l_s sum_points log(1 + 2 sigma+^2) ],
 *     squared TV on sigma_raw, squared TV on the 27 coefficients and a Cauchy sparsity term on the density at the
 *     lattice points.  Dividing by P keeps a weight meaningful across resolutions and prunes.
 *   - Gradient.  Written for every stored copy as dL / d(the copy's lattice point), the convention of the tied gradient
 *     of baked_render_bwd + baked_tie.  fp32, each op rounded, no contraction:
 *       S_ch = 0, then S_ch += (v_p - v_n) over the point's edges in the order -x, +x, -y, +y, -z, +z;
 *       g_ch = a_ch S_ch with a_0 = fp32(2 l_sigma / P) and a_1..27 = fp32(2 l_sh / P), each formed in fp64 and rounded
 *       once; channel 0 then adds (b sigma+) / (1 + 2 (sigma+ sigma+)) with b = fp32(4 l_s / P) formed the same way;
 *       d[copy][ch] += g_ch for ch = 0 .. 27 (added into the caller's buffer); channels 28 .. 31 are not touched.
 *     Every copy of a point computes the same terms in the same order, so every copy gets the same bits, and a d whose
 *     copies were bit-equal (the tie's output) stays so.
 *   - Value.  partials[slot] = (sum over the slot's stored points that are canonical copies of l_sigma (sum of the
 *     point's +x / +y / +z edges' (d sigma)^2) + l_sh (the same over channels 1 .. 27) + l_s log1p(2 sigma+^2)) / P, in
 *     fp64 (differences of the fp32 values, exact in fp64), each point's edges and sparsity term counted once; the
 *     per-point sums are reduced over the slot in a fixed order, so the partials are the same bits every run.  L is
 *     their sum.
 * baked_lattice_count: *count = P (int64, device memory; one memset and one launch, integer atomics).
 * baked_regularizer: reads P from *count when it runs (no host synchronisation), adds the gradient into d (layout of
 *   values; may be NULL) and writes partials fp64[n_active] (may be NULL, not both).  One CTA per slot.
 * Refused before any launch: an invalid box, a null pointer where one is needed (d and partials both NULL included),
 * n_active outside 1 .. the box's bricks, a weight that is negative, NaN or infinite, d overlapping values. */
int32_t nerfb200_baked_lattice_count(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                     int64_t n_active, int64_t* count, void* stream);
int32_t nerfb200_baked_regularizer(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                   int64_t n_active, const float* values, const int64_t* count, double tv_sigma,
                                   double tv_sh, double sparsity, float* d, double* partials, void* stream);

/* ---- baked fields: subdivision --------------------------------------------------------------------------------------
 * The field on the box (lo, hi, 2 res) that holds the same trilinear function as a field on (lo, hi, res), so that a
 * field can be trained coarse to fine (as Plenoxels upsamples its grid): train, prune, subdivide, train again.
 *   - Child bricks.  Per axis, parent brick pb has the children 2 pb + delta, delta in {0, 1}, that exist in the child
 *     box (8 (2 pb + delta) < 2 res, i.e. 2 pb + delta < the child box's bricks along that axis); a partial parent brick
 *     on an upper face can have only delta = 0 along that axis.  The child field's active bricks are the children of
 *     every active parent brick, in ascending child-brick order (so its bricks are sorted and its brick_map is their
 *     rank, as mesh_sparse_bricks produces them).  The caller forms this list; the library fills its values.
 *   - Values.  Child corner point l of child brick b' holds the child lattice index q' = min(8 b' + l, 2 res) per axis,
 *     which lies at the parent half-index q' / 2.  Along an axis where q' is even it uses the parent point q' / 2 with
 *     weight 1; where q' is odd it uses (q' - 1) / 2 and (q' + 1) / 2 with weight 1/2 each.  With m the number of odd
 *     axes, the value is over the 2^m parent points:
 *       m = 0: the parent point's bits (a copy: -0, inf and NaN payloads included);
 *       m >= 1: the points visited in the renderer's corner order (k = 0 .. 7, offset (k & 1, k >> 1 & 1, k >> 2))
 *               skipping those with offset 1 along an even axis; each term is w v with w = 2^-m, acc = the first term,
 *               then acc = acc + term.  fp32, each op rounded, no contraction, no flush to zero (w v is exact unless it
 *               is subnormal).
 *     Every parent point is read from its copy in parent brick floor(b' / 2) (local points 4 delta .. 4 delta + 4 per
 *     axis), so child copies are bit-equal wherever the parent's copies are, as they are after a bake and after every
 *     tied update.  All 28 channels go through the rule; channels 28 .. 31 are written 0.  A child whose parent brick's
 *     brick_map entry is -1 (or not below n_active) is written as all zeros.
 *   - Why the function is preserved.  The cell rule's scale = (float) res / (hi - lo) doubles exactly, so the child
 *     cell coordinate is exactly twice the parent's, and a trilinear function restricted to a sub-cube is its
 *     interpolation of the sub-cube's corner values.  The child field therefore renders the parent's continuous
 *     sigma_raw and SH field up to the fp32 rounding of the new lattice values; only the renderer's sample spacing,
 *     half the smallest cube side, halves.
 * baked_subdivide: box, brick_map and values[n_active][729][32] the parent field (fp32); child_bricks[n_child] the child
 *   box's active bricks as above; child_values[n_child][729][32] fp32 receives the child field.  One CTA per child slot
 *   staging the 5 x 5 x 5 parent points it reads in shared memory; offsets in 64 bits.  n_child 0 launches nothing.
 * Refused before any launch: an invalid box or 2 res > 4096 on any axis, a null pointer, n_active outside 0 .. the
 * parent box's bricks, n_child outside 0 .. the child box's bricks, child_values overlapping values.  No atomics, no host
 * synchronisation.  fp16 fields have no subdivision: subdivide the widened field. */
int32_t nerfb200_baked_subdivide(const nerfb200_grid_t* box, const int32_t* brick_map, int64_t n_active,
                                 const float* values, const int32_t* child_bricks, int64_t n_child,
                                 float* child_values, void* stream);

/* ---- baked fields: meshes -------------------------------------------------------------------------------------------
 * The level set of a baked field's own density as a triangle mesh, with the normals and colours the field itself gives
 * (as Plenoxels / PlenOctrees export meshes of their fitted grids), without a network.  All fp32 with round-to-nearest,
 * each op rounded, no contraction unless fmaf is named.
 *   - Values.  Marching cubes runs over sigma_raw itself (channel 0, widened exactly to fp32 from an fp16 field), not
 *     over relu(sigma_raw): mesh_sparse_count / mesh_sparse_emit with halo = 0 on the field's box, brick_map and bricks,
 *     the field's layout being that of "sparse meshes" with halo = 0.  Along a lattice edge the renderer's density is
 *     relu of a linear function, so for level >= 0 its crossing is the crossing of sigma_raw itself; relu'd values would
 *     move the vertex wherever an endpoint is negative (endpoints -100 and 100 at level 50: t = 0.75 on sigma_raw, 0.5 on
 *     relu values, a quarter of a cube off the renderer's surface).  For level >= 0 the inside / outside classification
 *     is relu's, so the faces and the vertex numbering are those of the sparse mesh of relu(sigma_raw) (extract_mesh of
 *     the baked network over the same grid); vertices differ only on edges with a negative endpoint.  A negative level
 *     is refused by the library's Python interface: the density is never negative.
 *   - Direction and normal (baked_mesh_dirs).  Vertex i's lattice edge (q, a) is edge_keys[i] = q * 3 + a (mesh_sparse_
 *     emit's keys); t = (level - v0) / (v1 - v0) on the endpoints' sigma_raw.  The gradient at each endpoint is
 *     mesh_emit's (central differences, one-sided at the lattice's faces) over sigma_raw read at each point's canonical
 *     copy ("baked fields: regularisers"); a lattice point no active brick holds reads 0, the renderer's miss.  dir is
 *     mesh_emit's view-direction rule on those gradients: -n, or (0, 0, 1) where the interpolated gradient vanishes or is
 *     not finite; normal = -dir, or (0, 0, 0) where the rule fell back.  On a field whose every brick is active, dir is
 *     bit for bit mesh_sparse_emit's view_dirs with halo = 1 over the same sigma_raw.
 *   - Colour (baked_mesh_colors).  Channels 0 .. 27 at the vertex from the edge's two endpoints' canonical copies by the
 *     renderer's fmaf chain restricted to those two corners: v = 0, v = fmaf(1 - t, v0, v), v = fmaf(t, v1, v); then the
 *     renderer's colour with Y_j(dirs[i]) (Y_0 alone without view directions): the colour the renderer gives that point
 *     seen head-on from outside, as extract_mesh(colors=True) gives for a network.
 *   - NDC.  A field baked from a forward-facing scene lives in NDC: the NDC vertices, faces and dirs go through
 *     ndc_mesh_to_world; the colours are formed with the WORLD direction (the baked SH were fitted to world view
 *     directions); the normals are -(world dir), or 0 where the NDC rule fell back.
 *   - Copies.  Every lookup reads canonical copies, so the attributes do not depend on which copy a thread holds.  The
 *     vertex positions come from the copy the marching brick holds, and agree with t whenever the field's copies are
 *     bit-equal, which holds for every field the library produces (bake, tie, subdivide, prune, half).
 *   - Transparent prune.  Dropping transparent bricks ("baked fields: pruning") leaves the faces and the vertices (ids
 *     included) the same bits at level >= 0: such a brick holds no endpoint of a crossing edge (sigma_raw <= 0 <= level at
 *     all its points), so it owns no vertex.  Normals and colours are the same bits at every vertex whose gradient
 *     stencil keeps a copy of every point; a stencil point stored only in a dropped brick then reads 0 instead of its
 *     sigma_raw <= 0.  This is the one place where pruning a transparent brick changes what is read, while renders stay
 *     the same bits.
 *   - Robustness.  A key off the lattice's edges, or an endpoint no active brick holds, reads nothing out of bounds and
 *     writes NaN for that vertex.  Keys are meant to come from mesh_sparse_emit over the same field and level; the device
 *     does not check that.
 * baked_mesh_dirs: dirs[n_vertices][3], normals[n_vertices][3] (may be NULL).
 * baked_mesh_colors: colors[n_vertices][3]; dirs[n_vertices][3] is read with view directions (may be NULL without).
 * _f16: values binary16 ("baked fields: half precision"), each value widened exactly as it is read.
 * One thread per vertex, offsets in 64 bits, no atomics, no host synchronisation; n_vertices 0 launches nothing.
 * Refused before any launch: an invalid box, a null pointer where one is needed, n_vertices < 0, a non-finite level,
 * an fp16 values pointer that is not 16-B aligned. */
int32_t nerfb200_baked_mesh_dirs(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                 float level, const int64_t* edge_keys, int64_t n_vertices, float* dirs,
                                 float* normals, void* stream);
int32_t nerfb200_baked_mesh_dirs_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                     float level, const int64_t* edge_keys, int64_t n_vertices, float* dirs,
                                     float* normals, void* stream);
int32_t nerfb200_baked_mesh_colors(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                   int32_t use_viewdirs, float level, const int64_t* edge_keys, const float* dirs,
                                   int64_t n_vertices, float* colors, void* stream);
int32_t nerfb200_baked_mesh_colors_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                       int32_t use_viewdirs, float level, const int64_t* edge_keys, const float* dirs,
                                       int64_t n_vertices, float* colors, void* stream);

/* ---- baked fields: 8-bit values -------------------------------------------------------------------------------------
 * A baked field whose values are stored as one byte per channel with a per-channel scale and offset, at a quarter of
 * the bytes of the fp32 field and half of the fp16 one, for fields that are kept, saved, rendered, pruned and meshed
 * (SNeRG ships its baked grids as 8-bit values).  Fine-tuning, the regularisers and subdivision stay fp32: dequantise
 * the field, work on it, and quantise it again.
 *   - Layout.  values[slot][729][32] uint8 codes (32 B per lattice point, one 32-B sector); channels 28 .. 31 hold 0
 *     and are never read.  dequant[2][28] fp32 in device memory: row 0 the scale s_c of channel c, row 1 its offset o_c.
 *   - Quantisation (done by the library's Python interface, BakedField.quantize), for c = 0 .. 27, every op rounded to
 *     fp32: lo_c = min(0, min v) and hi_c = max(0, max v) over every stored value of channel c (every slot and lattice
 *     point), so the range holds 0; s_c = (hi_c - lo_c) / 255, or 1 where that is 0; z_c = clamp(rint(-lo_c / s_c), 0,
 *     255), an integer held as +0 when it is 0 (never -0), so o_c = -(z_c s_c) is -0 for z_c = 0; q = clamp(rint((v -
 *     o_c) / s_c), 0, 255), rint rounding half to even.  Every division is correctly rounded (not a multiplication by
 *     a rounded reciprocal), so the codes and the table are the same bits on every device.  A field with a non-finite
 *     value in channels 0 .. 27, or whose range hi_c - lo_c overflows fp32, is refused.
 *   - Dequantisation.  v' = fl(fl(q s_c) + o_c): two rounded ops, no contraction (in torch q.float() * s + o).  Zero is
 *     exact: v'(z_c) = fl(z_c s_c) - fl(z_c s_c) = +0, so a sigma_raw <= 0 gets a code <= z_0 and dequantises to <= 0,
 *     and a transparent brick ("baked fields: pruning") stays transparent.  Equal values get equal codes, so the stored
 *     copies of a lattice point stay bit-equal and the mesh rule of "baked fields: meshes" ("Copies") still holds.  The
 *     scales are per channel, not per brick, for that reason.
 *   - Rendering, peak weights and meshes (baked_render_u8, baked_max_weights_u8, baked_mesh_dirs_u8,
 *     baked_mesh_colors_u8).  Each code is dequantised as it is gathered; every other op is the fp32 rule of "baked
 *     fields", "baked fields: pruning" and "baked fields: meshes": the same corners in the same order through the same
 *     fmaf chain.  A uint8 field therefore renders, gives peak weights and meshes bit for bit like the fp32 field holding
 *     its dequantised values.  A corner's channels 0 .. 27 are two 16-B loads; the peak weights and the mesh's sigma_raw
 *     reads are one byte per point.  The 56 table entries are copied into each CTA's shared memory once.
 * baked_render_u8, baked_max_weights_u8, baked_mesh_dirs_u8, baked_mesh_colors_u8: the arguments of baked_render,
 *   baked_max_weights, baked_mesh_dirs and baked_mesh_colors, values uint8 codes followed by dequant.  Refused before any
 *   launch: whatever their fp32 twins refuse (the same checks), a values pointer that is not 16-B aligned, and a null
 *   dequant. */
int32_t nerfb200_baked_render_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                 const float* dequant, int32_t use_viewdirs, const float* rays, int32_t ray_stride,
                                 int64_t n_rays, int32_t white_background, float stop_transmittance, float* out,
                                 void* stream);
int32_t nerfb200_baked_max_weights_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                      const float* dequant, int32_t use_viewdirs, const float* rays, int32_t ray_stride,
                                      int64_t n_rays, float* max_w, void* stream);
int32_t nerfb200_baked_mesh_dirs_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                    const float* dequant, float level, const int64_t* edge_keys, int64_t n_vertices,
                                    float* dirs, float* normals, void* stream);
int32_t nerfb200_baked_mesh_colors_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                      const float* dequant, int32_t use_viewdirs, float level, const int64_t* edge_keys,
                                      const float* dirs, int64_t n_vertices, float* colors, void* stream);

/* ---- baked fields: normal maps and point queries ---------------------------------------------------------------------
 * The geometry probes a trained network has (normal maps of a render, raw outputs and the density gradient at caller-
 * given points), for a baked field without its network.  All fp32 with round-to-nearest, each op rounded, no
 * contraction unless fmaf is named, as in every baked section.
 *   - Gradient at a point x.  The renderer's lookup of x ("baked fields": the cell rule, the cube, the fractions f, the
 *     brick slot).  For each axis c: g_c = 0, then for the corners k = 0 .. 7 in the renderer's order g_c =
 *     fmaf(s_kc * p_kc, v_k, g_c), then g_c = g_c * scale_c.  v_k is corner k's sigma_raw (channel 0, read as the
 *     renderer reads it); s_kc is +1 where the corner's offset on axis c is 1 and -1 where it is 0 (exact); p_kc is the
 *     product of the other two axes' trilinear weights in axis order (w_y w_z, w_x w_z, w_x w_y); scale_c = res_c / (hi_c -
 *     lo_c) of the cell rule.  This is the exact gradient of the trilinear sigma_raw inside the cube; on a cube face it
 *     is one-sided, the gradient of the cube the lookup picked.  A point outside the box or in an inactive brick has
 *     sigma_raw = 0 and gradient 0.  It is the gradient of sigma_raw, not of relu(sigma_raw); wherever a sample has a
 *     nonzero weight sigma_raw > 0 and the two agree.
 *   - Normal map (baked_render_normals).  The march of baked_render (interval, t_k, rounds of 32, scan, early stopping,
 *     outputs): out[n][8] is bit for bit what baked_render writes for the same inputs.  normals[n][3] = N: per sample,
 *     the gradient above at the sample's point x = o + d t_k formed as the lookup forms it; with a camera ndc, g is
 *     first replaced by J^T(x) g ("NDC scenes", ndc_grad_to_world); n = -g / |g| with |g| = sqrt((g_x g_x + g_y g_y) +
 *     g_z g_z), n = 0 where |g| = 0 (render_fwd_normals' rule).  N = 0, then N += w n in sample order over the samples
 *     with w != 0, broadcast across the round's lanes as the colour sums are; skipping w == 0 keeps a NaN gradient out
 *     of rays that never reach it.  A stopped ray sums the samples before its stop.  N is not renormalised: |N| <= acc
 *     up to rounding.  The gradient reads the sigma_raw corners the interp already loads.
 *   - Point query (baked_query).  At pts[P][3], in the field's own frame: raw[P][4] = (s_r, s_g, s_b, sigma_raw),
 *     run_network's raw layout (pre-sigmoid logits, then sigma_raw), each channel the renderer's interp at the point
 *     and s_c the renderer's logit with Y_j(dirs[p]) (dirs taken as given, not normalised) or Y_0 alone without view
 *     directions; (0, 0, 0, 0) outside the box or in an inactive brick.  grad[P][3] = the gradient above.  At a point
 *     whose fractions are exactly 0 the channels are the stored values bit for bit (the lattice points of a box whose
 *     cell rule puts them at f = 0, e.g. a power-of-two box).
 *   - Formats.  fp16 values and uint8 codes go through the one per-format point reader of "baked fields: half
 *     precision" / "baked fields: 8-bit values": such a field gives normals, raw values and gradients bit for bit like
 *     its widened fp32 field.
 *   - Transparent prune.  Dropping transparent bricks ("baked fields: pruning") leaves normal maps the same bits: their
 *     samples have w = +0 and are skipped, exactly as for the colour sums.
 * baked_render_normals: the arguments of baked_render plus ndc (NULL: normals in the field's frame; else the NDC camera
 *   the rays were generated with, for world-space normals) and normals[n_rays][3].
 * baked_query: dirs[P][3] is read with view directions when raw is given (may be NULL otherwise); raw and grad may each
 *   be NULL, not both.  One thread per point; n_points 0 launches nothing.
 * _f16 / _u8: values binary16, or uint8 codes followed by dequant, as baked_render_f16 / baked_render_u8.
 * Refused before any launch: whatever baked_render refuses (the same checks), a null normals, an ndc make_ndc_map
 * refuses ("NDC scenes"), n_points < 0, raw and grad both NULL, view directions with raw and no dirs.  No atomics, no
 * host synchronisation. */
int32_t nerfb200_baked_render_normals(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                      int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                      int32_t white_background, float stop_transmittance, const nerfb200_ndc_t* ndc,
                                      float* out, float* normals, void* stream);
int32_t nerfb200_baked_render_normals_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                          int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                          int32_t white_background, float stop_transmittance,
                                          const nerfb200_ndc_t* ndc, float* out, float* normals, void* stream);
int32_t nerfb200_baked_render_normals_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                         const float* dequant, int32_t use_viewdirs, const float* rays,
                                         int32_t ray_stride, int64_t n_rays, int32_t white_background,
                                         float stop_transmittance, const nerfb200_ndc_t* ndc, float* out,
                                         float* normals, void* stream);
int32_t nerfb200_baked_query(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                             int32_t use_viewdirs, const float* pts, const float* dirs, int64_t n_points, float* raw,
                             float* grad, void* stream);
int32_t nerfb200_baked_query_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                 int32_t use_viewdirs, const float* pts, const float* dirs, int64_t n_points,
                                 float* raw, float* grad, void* stream);
int32_t nerfb200_baked_query_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                const float* dequant, int32_t use_viewdirs, const float* pts, const float* dirs,
                                int64_t n_points, float* raw, float* grad, void* stream);

/* Fused Adam over a flat vector (torch.optim.Adam semantics, train_nerf.py:136-141,261-270):
 * p, m, v updated in place from g; step is the 1-based step count AFTER this update; grad_scale
 * multiplies g first (1/world_size after a summed all-reduce). */
int32_t nerfb200_adam_step(float* p, const float* g, float* m, float* v, int64_t n, int32_t step, float lr,
                           float beta1, float beta2, float eps, float grad_scale, void* stream);

/* ---- a training step with no host work between its launches (one CUDA graph per step) ------------------
 * A captured graph freezes kernel arguments, so the one value that changes between replays is a step counter in device
 * memory: step_dev (int64) holds the number of optimisation steps done before this one, and every entry point below
 * that depends on the step reads it there when it runs.  nerfb200_step_advance adds 1 after the step's updates.
 *
 * random_fill_dev: nerfb200_random_fill with rng->step replaced by *step_dev (rng->step must be 0); the same device
 *   function, so the render kernels fed these tensors give the bits of a render call given the rng at that step.
 *   *step_dev >= 2^30 writes NaN (its counters would alias another step's).
 * draw_pixels: from (seed, *step_dev), *image_out = one image uniformly out of n_images and ids_out[n] = n distinct
 *   pixel ids out of n_pixels, uniform without replacement (the reference's two np.random.choice calls): each pixel gets a
 *   64-bit Philox key and the n smallest (key, id) pairs are taken, in ascending key order.  Exact and deterministic;
 *   its Philox counters never coincide with the render streams' (csrc/common.cuh).  n > n_pixels: NERFB200_ERR_INVALID.
 *   workspace: nerfb200_draw_workspace_bytes(n_pixels) bytes (-1: n_pixels outside 1 .. 2^31 - 1).
 * gen_rays_posed: nerfb200_gen_rays with the pose read on the device: the top 3 x 4 block of poses[*image] of a
 *   [n_images][pose_rows][4] table (pose_rows 3 or 4); the same rows as gen_rays given that pose, bit for bit.
 * gather_rows: out[k][0..2] = src[*image * rows_per_image + ids[k]][0..2] (targets, or a ray pool's rows).
 * mse_loss: *loss = mse(out_coarse[:, :3], target) + mse(out_fine[:, :3], target) (the coarse term alone when out_fine is
 *   NULL), out_* the [n][8] rows of render_fwd, target [n][3]; g_coarse / g_fine [n][8] receive the upstream gradients
 *   render_bwd takes, bit for bit what autograd of torch's mean mse_loss gives: fp32(fp32(2 / 3n) * fp32(x - t)) in
 *   columns 0..2, zero elsewhere.  The loss sums the squares in fp64 and rounds each mean once.
 * lr_schedule: lr_out[i] = the rate parallel.FusedAdam uses for the step after done[i] steps, lr0 * lr_decay_factor **
 *   (max(done[i] - 1, 0) / (lr_decay * 1000)) in fp64 rounded once to fp32 (lr0 when lr_decay is 0).
 * adam_step_dev: nerfb200_adam_step for step *step_dev + 1 at rate lr_schedule(*step_dev); same bits as adam_step given
 *   that step and rate. */
int32_t nerfb200_random_fill_dev(const nerfb200_rng_t* rng, const int64_t* step_dev, int32_t stream_id, int64_t n_rays,
                                 int32_t per_ray, float* out, void* stream);
int64_t nerfb200_draw_workspace_bytes(int64_t n_pixels);
int32_t nerfb200_draw_pixels(uint64_t seed, const int64_t* step_dev, int32_t n_images, int64_t n_pixels, int64_t n,
                             int64_t* image_out, int64_t* ids_out, void* workspace, void* stream);
int32_t nerfb200_gen_rays_posed(const float* poses, int32_t pose_rows, const int64_t* image, int32_t height,
                                int32_t width, float focal, const int64_t* pixel_ids, int64_t n, int32_t ndc, float near,
                                float far, int32_t use_viewdirs, int32_t out_stride, float* out, void* stream);
int32_t nerfb200_gather_rows(const float* src, int64_t rows_per_image, const int64_t* image, const int64_t* ids,
                             int64_t n, float* out, void* stream);
int32_t nerfb200_mse_loss(const float* out_coarse, const float* out_fine, const float* target, int64_t n, float* loss,
                          float* g_coarse, float* g_fine, void* stream);
int32_t nerfb200_lr_schedule(const int64_t* done, int64_t n, double lr0, double lr_decay, double lr_decay_factor,
                             float* lr_out, void* stream);
int32_t nerfb200_adam_step_dev(float* p, const float* g, float* m, float* v, int64_t n, const int64_t* step_dev,
                               double lr0, double lr_decay, double lr_decay_factor, float beta1, float beta2, float eps,
                               float grad_scale, void* stream);
int32_t nerfb200_step_advance(int64_t* step_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERFB200_H_ */
