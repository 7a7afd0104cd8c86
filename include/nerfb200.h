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
