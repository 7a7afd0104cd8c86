// common.cuh -- shared declarations for the nerfb200 CUDA library (sm_90a).
//
// The "plan" is the host-built description of one FlexibleNeRFModel (nerf/models.py:185-256 of the
// reference) as a chain of GEMM layers (outputs of 64*NJ columns, evaluated tile-by-tile) and up
// to two narrow "heads" (fc_alpha: 1 output, fc_rgb: 3, fc_out: 4) that are evaluated as dot
// products.  It is passed by value to every kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nerfb200.h"

namespace nerfb200 {

constexpr int kMaxGemm = 20;
constexpr int kTileRows = 128;   // points per CTA tile
constexpr int kThreads = 256;    // threads per CTA in the MLP kernels

struct GemmLayer {
  int k_h;       // input columns taken from the previous activation (0 for layer1, else hidden)
  int k_enc;     // padded (multiple of 8) encoded-input columns appended after k_h (0 if none)
  int enc_real;  // real encoded columns (63 / 27 / ...)
  int enc_sel;   // 0: xyz encoding, 1: direction encoding
  int n;         // output features (hidden or hidden/2), multiple of 64
  int relu;      // ReLU after the bias (layer1 has none: models.py:238)
  int wt_off;    // blob offset of Wt[k_h + k_enc][n]   (forward operand)
  int wh_off;    // blob offset of Wh[n][k_h]           (dgrad operand; h-part only)
  int b_off;     // blob offset of bias[n]
  int cum_n;     // sum of n over previous gemm layers: stash slice = base + n_points * cum_n
  int flat_w;    // offset of weight[n][k_h + enc_real] in the flat (torch-layout) vector
  int flat_b;    // offset of bias[n] in the flat vector
  int src;       // gemm index whose output is this layer's h-input (-1 for layer1)
  // wgmma operand copy (mlp_tc.cu): k_tc = K the tensor-core path contracts over (the direction
  // encoding of layers_dir[0] is hoisted out per ray, so k_tc = k_h there); per k-step of 16 the blob
  // holds [hi slab0 | hi slab1 | lo slab0 | lo slab1], slab = [n][8 fp16] (the wgmma canonical K-major,
  // no swizzle: 8-row core matrices 128 B apart, the two K halves one slab apart); fp16 x 2 split with a
  // 2^11-scaled residual (tc_common.cuh split_f16x2).
  int k_tc;
  int tc_off;
  // dgrad operand copy: Wt[k < k_h][n] as K-major slabs over the reduction index n, hi|lo per 16 n
  int tcd_off;
  int mask_cum;  // ReLU bit-mask words (uint32, one bit per output) per point before this layer's
};

struct HeadLayer {
  int k;        // input features
  int n_out;    // 1, 3 or 4
  int out_col;  // first column of raw[...,4] it produces
  int w_off;    // blob offset of W[n_out][k] (torch layout), 4-float aligned
  int b_off;    // blob offset of bias[4]
  int src;      // gemm index whose output it reads
  int flat_w, flat_b;
};

struct Plan {
  int n_gemm;
  int n_trunk;  // gemm layers 0..n_trunk-1 are layer1 + layers_xyz
  int n_head;
  int hidden;
  int sum_n;  // floats stashed per point: every gemm layer's output + the two padded encodings + the mask words
  int enc_cum[2];  // stash slice of the xyz / direction encoding: base + n_points * enc_cum[sel], width enc_tile_w / dim_dir_pad
  int mask_base;   // stash slice of the ReLU bit masks: base + n_points * (mask_base + g.mask_cum), n/32 words per point
  int dim_xyz, dim_xyz_pad, dim_dir, dim_dir_pad;
  int enc_tile_w;  // dim_xyz padded to 16: width of the xyz-encoding operand tile of the wgmma path (tc_common.cuh)
  int n_freq_xyz, n_freq_dir, inc_xyz, inc_dir;
  int blob_floats, flat_floats;
  int use_viewdirs;
  GemmLayer g[kMaxGemm];
  HeadLayer h[2];  // viewdirs: h[0] = fc_alpha (after trunk), h[1] = fc_rgb (after dir layer); else h[0] = fc_out
  float freq_xyz[NERFB200_MAX_FREQS];
  float freq_dir[NERFB200_MAX_FREQS];
};

// ---------------------------------------------------------------------------------------------
// Random inputs of the render kernels.  Each one comes either from a tensor the host drew (the reference's
// torch.rand / torch.randn order) or from the seeded counter-based stream defined below (nerfb200_rng_t).
//
// The seeded stream is Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011):
//   key     = (seed & 0xffffffff, seed >> 32)
//   counter = (sample >> 2, stream + 4 * step, ray & 0xffffffff, ray >> 32)
// with ray the GLOBAL ray index (ray_offset + the ray's row in the call) and stream 0 t_rand, 1 noise_c, 2 u, 3 noise_f.
// One call yields the four 32-bit words w[0..3] of samples 4b .. 4b + 3 of one ray in one stream.
//   uniform (t_rand, u):     sample j = 4b + i is (w[i] >> 8) * 2^-24, in [0, 1) (torch's 24-bit construction)
//   normal (noise_c, noise_f): Box-Muller on the pairs (w[0], w[1]) -> samples 4b, 4b + 1 and (w[2], w[3]) -> 4b + 2,
//                            4b + 3: u1 = ((w[2p] >> 8) + 1) * 2^-24 in (0, 1], u2 = (w[2p + 1] >> 8) * 2^-24,
//                            r = sqrt(-2 ln u1), sample 4b + 2p = r cos(2 pi u2), sample 4b + 2p + 1 = r sin(2 pi u2),
//                            evaluated in fp64 and rounded once to fp32.
// So every random number is a pure function of (seed, step, stream, global ray, sample): a ray gets the same numbers
// whatever the chunking of the batch or its sharding across GPUs.  step < 2^30 keeps stream + 4 * step in 32 bits.
//
// The pixel draw of a training step (step.cu, nerfb200_draw_pixels) uses the same key and reserves a counter word:
//   counter = (q, step & 0xffffffff, purpose, 0x80000000)
// purpose 0: the 64-bit keys of pixels 2q (words 0, 1) and 2q + 1 (words 2, 3); purpose 1, q = 0: the image (words 0, 1).
// The render streams' last word is the high half of a global ray index >= 0 and < 2^63, so its top bit is never set:
// the draw's counters cannot coincide with any render stream's, for any step.  (A fifth render stream id instead would
// be stream + 4 * step = 4 + 4 * step, which is stream 0 of the next step.)
// ---------------------------------------------------------------------------------------------
enum RandStream { kRandTRand = 0, kRandNoiseC = 1, kRandU = 2, kRandNoiseF = 3 };

struct RandSrc {
  const float* ptr;    // tensor source [ray][stride], or nullptr
  int64_t stride;      // floats per ray in ptr
  int seeded;          // ptr == nullptr and seeded: generate from the stream below; neither: no source
  uint32_t key0, key1; // the seed
  uint32_t ctr1;       // stream + 4 * step
  int64_t ray_offset;  // global index of the call's first ray

  __host__ __device__ bool present() const { return ptr != nullptr || seeded; }
#ifdef __CUDACC__
  __device__ __forceinline__ float uniform(int64_t ray, int j) const;
  __device__ __forceinline__ float normal(int64_t ray, int j) const;
#endif
};

inline RandSrc rand_none() { return RandSrc{nullptr, 0, 0, 0, 0, 0, 0}; }
inline RandSrc rand_tensor(const float* p, int64_t stride) { return RandSrc{p, stride, 0, 0, 0, 0, 0}; }
inline RandSrc rand_seeded(const nerfb200_rng_t& r, int stream) {
  return RandSrc{nullptr, 0, 1, (uint32_t)r.seed, (uint32_t)(r.seed >> 32), (uint32_t)stream + 4u * (uint32_t)r.step,
                 r.ray_offset};
}

// Where the MLP forwards read a sample's position and its ray's view direction.  The render path forms the point
// o + d z from the ray row and the depth (train_utils.py:67); a caller that chose its own points gives them as pts.
// Ray r's view direction is the 3 floats at dirs + r * dir_stride: rays + 8 and ray_stride on the render path.
struct PointSrc {
  const float* rays;  // [n_rays][ray_stride] = [o(3) d(3) ...], read when pts is null
  int ray_stride;
  const float* z;     // [n_points], read when pts is null
  const float* pts;   // [n_points][3], or null: the point is o + d z
  const float* dirs;  // null without view directions
  int dir_stride;
};

// host side (api.cu)
int build_plan(const nerfb200_arch_t* arch, Plan* plan);  // 0 or NERFB200_ERR_*
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
void count_launch();  // one call per kernel launched (nerfb200_launch_count)
int device_sms();     // SM count of the current device (grid sizes of persistent / grid-stride kernels)

// launchers (one per .cu), all return NERFB200_OK or an error code
int launch_pack(const Plan& p, const float* flat, float* blob, cudaStream_t s);
int launch_sample_coarse(const float* rays, int ray_stride, int64_t n_rays, const RandSrc& t_rand, int n_coarse,
                         int perturb, int lindisp, float* z, cudaStream_t s);
// materialises n_rays x per_ray numbers of a seeded stream (uniform for t_rand / u, normal for noise_c / noise_f)
int launch_random_fill(const RandSrc& src, int stream_id, int64_t n_rays, int per_ray, float* out, cudaStream_t s);
int launch_gen_rays(const float* c2w12_host, int height, int width, float focal, const int64_t* pix, int64_t n, int ndc,
                    float near, float far, int use_viewdirs, int out_stride, float* out, cudaStream_t s);
int launch_pack_rays(const float* ro, const float* rd, int64_t n, int height, int width, float focal, int ndc, float near,
                     float far, int use_viewdirs, int out_stride, float* out, cudaStream_t s);
int launch_encode(const Plan& p, int which, const float* x, int64_t n, float* out, cudaStream_t s);
// compositing: ray r's direction (its norm scales the sample spacing) is the 3 floats at dirs + r * dir_stride
int launch_composite_fwd(const float* raw, const float* z, const float* dirs, int dir_stride, const RandSrc& noise,
                         int64_t n_rays, int n_samples, float noise_std, int white_bkgd, float* out,
                         float* weights, cudaStream_t s);
// sample_grads: also take the upstream gradient of depth (g_out[r][5]) and of the weights (g_w[n_rays][n_samples],
// may be null); the render path's backward takes neither
int launch_composite_bwd(const float* raw, const float* z, const float* dirs, int dir_stride, const RandSrc& noise,
                         const float* g_out, const float* g_w, bool sample_grads, int64_t n_rays, int n_samples,
                         float noise_std, int white_bkgd, float* d_raw, cudaStream_t s);
// u: a tensor [n_rays][n_fine], the seeded stream, or none (the det=True linspace)
int launch_sample_pdf_merge(const float* z_coarse, const float* weights_coarse, const RandSrc& u,
                            const float* cdf_in, int64_t n_rays, int n_coarse, int n_fine, float* z_fine,
                            float* z_samples, int32_t* inds, float* cdf_out, cudaStream_t s);
int launch_adam(float* p, const float* g, float* m, float* v, int64_t n, int step, float lr, float b1, float b2,
                float eps, float grad_scale, cudaStream_t s);

// ---- a training step whose step count lives in device memory (step.cu; nerfb200.h "a training step ...") ----
// the learning-rate schedule of parallel.FusedAdam: lr0 * factor ** (max(done - 1, 0) / (decay * 1000)); decay <= 0: lr0
struct LrSchedule {
  double lr0, decay, factor;
};
int launch_random_fill_dev(const RandSrc& src, const int64_t* step, int stream_id, int64_t n_rays, int per_ray,
                           float* out, cudaStream_t s);
int launch_gen_rays_posed(const float* poses, int pose_rows, const int64_t* image, int height, int width, float focal,
                          const int64_t* pix, int64_t n, int ndc, float near, float far, int use_viewdirs, int out_stride,
                          float* out, cudaStream_t s);
int launch_lr_schedule(const int64_t* done, int64_t n, const LrSchedule& sch, float* out, cudaStream_t s);
int launch_adam_dev(float* p, const float* g, float* m, float* v, int64_t n, const int64_t* done, const LrSchedule& sch,
                    float b1, float b2, float eps, float grad_scale, cudaStream_t s);

// The MLP kernel families.  Each file's predicate says whether its kernels take a plan (NERFB200_OK, else the reason
// in the last error, prefixed with `what`); api.cu's check_impl maps an impl code to them, and its mlp_forward /
// mlp_backward pick the launchers, which do not check again.
// fp32 CUDA cores (mlp_simt.cu), impl 0: the forward, then the backward's two halves (dgrad fills the gradient stash
// `gstash`, wgrad reduces it into flat_grad)
int simt_supported(const Plan& p, const char* what);
int launch_mlp_fwd_simt(const Plan& p, const float* blob, const PointSrc& src, int64_t n_rays, int n_samples, float* raw,
                        float* stash, cudaStream_t s);
int launch_dgrad_simt(const Plan& p, const float* blob, const float* d_raw, const float* stash, float* gstash,
                      int64_t P, cudaStream_t s);
int launch_wgrad_simt(const Plan& p, const float* rays, int ray_stride, const float* z, int n_samples,
                      const float* d_raw, const float* stash, const float* gstash, int64_t P, float* flat_grad,
                      cudaStream_t s);
// wgmma forward (mlp_tc.cu), impl 1 and 3: training writes the stash (hidden 128 only); fast is the single-pass
// fp16 inference forward (impl 3, no stash)
int tc_supported(const Plan& p, int n_samples, bool training, const char* what);
int launch_mlp_fwd_tc(const Plan& p, const float* blob, const PointSrc& src, int64_t n_rays, int n_samples, float* raw,
                      float* stash, bool fast, cudaStream_t s);
// density gradient (mlp_tc.cu, nerfb200.h "density gradient"), impl 1 only: sigma_raw and its gradient w.r.t. the points;
// grad_tc_supported checks what it needs beyond tc_supported(training = false)
int grad_tc_supported(const Plan& p, const char* what);
int launch_density_grad_tc(const Plan& p, const float* blob, const float* pts, int64_t n_points, float* out,
                           const int* n_dev, cudaStream_t s);
// ---- normal maps of a render's last pass (normals.cu; nerfb200.h "normal maps") ----
// The samples with nonzero compositing weight, compacted: count[r], first[r] (their first slot), *total; pts[slot][3] =
// o + d z as the MLP forms it
struct NormalState {
  int* count;
  int* first;
  int* total;
  float* pts;
  float* grad;  // [slot][4], density_grad's output
};
int launch_normal_compact(const float* rays, int ray_stride, const float* z, const float* weights, int64_t n_rays,
                          int n_samples, const NormalState& ns, cudaStream_t s);
// ---- NDC scenes (ndc.cu; nerfb200.h "NDC scenes"): the map N of ndc_rays and its Jacobian ----
// sw, sh of the header, as raygen.cu's finish_ray computes them
struct NdcMap {
  float sw, sh;
};
// NERFB200_ERR_INVALID (reason prefixed with `what`) for a null or malformed camera
int make_ndc_map(const nerfb200_ndc_t* ndc, NdcMap* m, const char* what);
// q = N(p)
__device__ __forceinline__ void ndc_forward(const NdcMap& m, const float p[3], float q[3]) {
  q[0] = __fdiv_rn(__fmul_rn(m.sw, p[0]), p[2]);
  q[1] = __fdiv_rn(__fmul_rn(m.sh, p[1]), p[2]);
  q[2] = __fadd_rn(1.0f, __fdiv_rn(2.0f, p[2]));
}
// p = N^-1(q)
__device__ __forceinline__ void ndc_inverse(const NdcMap& m, const float q[3], float p[3]) {
  p[2] = __fdiv_rn(2.0f, __fsub_rn(q[2], 1.0f));
  p[0] = __fdiv_rn(__fmul_rn(q[0], p[2]), m.sw);
  p[1] = __fdiv_rn(__fmul_rn(q[1], p[2]), m.sh);
}
// G = J^T(q) g: the world gradient of a field whose NDC gradient at q is g
__device__ __forceinline__ void ndc_grad_to_world(const NdcMap& m, const float q[3], const float g[3], float G[3]) {
  const float qz1 = __fsub_rn(q[2], 1.0f);
  const float s = __fmul_rn(qz1, 0.5f);
  const float t = __fadd_rn(__fmul_rn(q[0], g[0]), __fmul_rn(q[1], g[1]));
  G[0] = __fmul_rn(s, __fmul_rn(m.sw, g[0]));
  G[1] = __fmul_rn(s, __fmul_rn(m.sh, g[1]));
  G[2] = __fmul_rn(s, __fsub_rn(-t, __fmul_rn(qz1, g[2])));
}
int launch_ndc_mesh_to_world(const NdcMap& m, const float* vertices, const int32_t* faces, const float* view_dirs,
                             int64_t n_vertices, int64_t n_faces, float* world_vertices, int32_t* world_faces,
                             float* world_dirs, cudaStream_t s);
int launch_ndc_from_world(const NdcMap& m, const float* p, int64_t n, float* q, cudaStream_t s);
int launch_ndc_grad_to_world(const NdcMap& m, const float* q, const float* rows, int64_t n, float* out, cudaStream_t s);
// world: each gradient is mapped by J^T at its point ns.pts[slot] before it is normalised (nerfb200.h "NDC scenes")
int launch_normal_sum(const float* weights, int64_t n_rays, int n_samples, const NormalState& ns, float* normals,
                      cudaStream_t s, const NdcMap* world = nullptr);
// wgmma backward (mlp_tc_bwd.cu), impl 1: data-gradient chain + every weight gradient in one kernel; `scratch` holds
// the L2-resident fixed-point gradient blob (bwd_tc_scratch_floats) the weight-gradient tiles are reduced into.
// bwd_tc_supported checks what it needs beyond tc_supported(training = true).
int bwd_tc_supported(const Plan& p, const char* what);
int launch_mlp_bwd_tc(const Plan& p, const float* blob, const float* dirs, int dir_stride, int64_t n_rays, int n_samples,
                      const float* d_raw, const float* stash, float* scratch, float* flat_grad, cudaStream_t s);
int64_t bwd_tc_scratch_floats(const Plan& p);

// ---- occupancy grid (occupancy.cu; nerfb200.h "occupancy grid") ----
// The rows the wgmma forward runs when a grid decides which samples are evaluated: map[row] = point (-1: padding), in
// 64-row blocks; blocks[b] = (first ray, last ray) of block b; *n_blocks blocks, read by the kernel from device memory.
constexpr int kGridGroupRays = 10;  // rays per compaction group: at most this many per 64-row block (tc kMaxRaysPerTile)
struct RowMap {
  const int* map;
  const int2* blocks;
  const int* n_blocks;
};
int64_t grid_max_blocks(int64_t n_rays, int n_samples);
int64_t grid_scratch_ints(int64_t n_rays, int n_samples);
int check_grid(const nerfb200_grid_t* g, const char* what);
int launch_grid_compact(const nerfb200_grid_t& g, const uint32_t* bits, const float* rays, int ray_stride, const float* z,
                        int64_t n_rays, int n_samples, float* raw, int* map, int* blocks, int* n_blocks,
                        int64_t* n_evaluated, int* scratch, cudaStream_t s);
// ---- early ray termination of an inference render's last pass (nerfb200.h "early ray termination") ----
// Per-ray state in device memory: order[r][i] = the sample of the ray's i-th evaluated sample, n_eval[r] = its evaluated
// count (cut to what it ran when it stops), T[r] = its transmittance; counts[g] = the rows of group g in the next round.
constexpr int kStopRound = NERFB200_STOP_ROUND;
struct StopState {
  int* order;
  int* n_eval;
  float* T;
  int* stop;  // stop_sample, or null
  int* counts;
};
// the 64-row blocks one round can fill
int64_t stop_round_max_blocks(int64_t n_rays, int n_samples);
// marks the pass's samples (grid lookup when bits is non-null, skipped ones get raw = [0 0 0 -inf]), fills order /
// n_eval / T / stop and round 0's counts; *other_rows = other_value when other_rows is non-null
int launch_stop_mark(const nerfb200_grid_t& g, const uint32_t* bits, const float* rays, int ray_stride, const float* z,
                     int64_t n_rays, int n_samples, float* raw, const StopState& st, int64_t* other_rows,
                     int64_t other_value, cudaStream_t s);
// round k's row map from the counts and the first blocks grid_scan_kernel made of them (RowMap format)
int launch_stop_scatter(const StopState& st, const int* first_block, int64_t n_rays, int n_samples, int round, int* map,
                        int* blocks, cudaStream_t s);
// after round k's MLP: T of every ray that ran rows, the stop test, raw = [0 0 0 -inf] for a stopped ray's remaining
// samples, round k + 1's counts; *n_evaluated (if non-null) gets round k's rows added (round 0: set)
int launch_stop_update(float* raw, const float* z, const float* dirs, int dir_stride,
                       const RandSrc& noise, float noise_std, int64_t n_rays, int n_samples, int round, float threshold,
                       const StopState& st, const int64_t* round_rows, int64_t* n_evaluated, cudaStream_t s);
// grid_scan_kernel (occupancy.cu) alone: first blocks, block count and row total of per-group row counts
int launch_grid_scan(const int* counts, int64_t n_groups, int* first_block, int* n_blocks, int64_t* n_rows,
                     cudaStream_t s);
// the wgmma inference forward (impl 1, or fast: impl 3) over a RowMap of the points o + d z of the ray rows; max_blocks
// bounds *n_blocks (the grid size is chosen on the host)
int launch_mlp_fwd_tc_map(const Plan& p, const float* blob, const float* rays, int ray_stride, const float* z,
                          int64_t n_rays, int n_samples, const RowMap& m, int64_t max_blocks, float* raw, bool fast,
                          cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__

// Stash row swizzle.  The activation / gradient stashes ([points][n] fp32, workspace private to this library) keep
// every 16-byte chunk of a row at chunk index (q ^ (point & 7)) inside its 128-byte segment.  Global access
// patterns are unchanged (a permutation inside each 128 B line), and a 128-row tile of the stash is byte-identical
// to a bank-conflict-free shared-memory tile.  The fp32 kernels use it; the tensor-core kernels stash operand tiles
// instead (tc_common.cuh "Operand tiles"), written from the epilogue registers.
__device__ __forceinline__ int swz_col(int col, int64_t point) { return (((col >> 2) ^ (int)(point & 7)) << 2) | (col & 3); }

// Positional encoding of one scalar coordinate (nerf_helpers.py:113-157): writes x (if include) and
// sin/cos(x * f_i) at the reference's channel positions for coordinate c of 3:
//   [x y z | sin(f0 xyz) | cos(f0 xyz) | sin(f1 xyz) | ...]
// `row` points at the start of this point's encoding.  x * f is rounded to fp32 first, as the
// reference evaluates `tensor * freq` before sin/cos (nerf_helpers.py:149-151).
__device__ __forceinline__ void encode_coord(float x, int c, int include, int f_begin, int f_end,
                                             const float* __restrict__ freqs, float* __restrict__ row) {
  const int base = include ? 3 : 0;
  if (include && f_begin == 0) row[c] = x;
  for (int f = f_begin; f < f_end; ++f) {
    float s, co;
    sincosf(__fmul_rn(x, freqs[f]), &s, &co);
    row[base + 6 * f + c] = s;
    row[base + 6 * f + 3 + c] = co;
  }
}

// Philox4x32-10: ten rounds, the key bumped by the Weyl constants between rounds (Random123's philox4x32_R(10, ...)).
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

__device__ __forceinline__ uint4 rand_block(const RandSrc& s, int64_t ray, int j) {
  const uint64_t g = (uint64_t)(s.ray_offset + ray);
  return philox4x32_10(make_uint4((uint32_t)j >> 2, s.ctr1, (uint32_t)g, (uint32_t)(g >> 32)), s.key0, s.key1);
}

__device__ __forceinline__ float RandSrc::uniform(int64_t ray, int j) const {
  if (ptr) return ptr[ray * stride + j];
  const uint4 w = rand_block(*this, ray, j);
  const uint32_t x = (j & 2) ? ((j & 1) ? w.w : w.z) : ((j & 1) ? w.y : w.x);
  return (float)(x >> 8) * 0x1p-24f;
}

__device__ __forceinline__ float RandSrc::normal(int64_t ray, int j) const {
  if (ptr) return ptr[ray * stride + j];
  const uint4 w = rand_block(*this, ray, j);
  const uint32_t a = (j & 2) ? w.z : w.x, b = (j & 2) ? w.w : w.y;
  const double u1 = (double)((a >> 8) + 1) * 0x1p-24, u2 = (double)(b >> 8) * 0x1p-24;
  const double r = sqrt(-2.0 * log(u1));
  double sn, cs;
  sincospi(2.0 * u2, &sn, &cs);
  return (float)(r * ((j & 1) ? sn : cs));
}

// torch.linspace(0, 1, n)[q] as torch's CUDA kernel evaluates it: the stratified sampler's grid (train_utils.py:45)
// and the det=True u of sample_pdf (nerf_helpers.py:272-276)
__device__ __forceinline__ float linspace01(int q, int n) {
  if (n == 1) return 0.f;
  const float step = __fdiv_rn(1.0f, (float)(n - 1));
  if (q < n / 2) return __fmul_rn(step, (float)q);
  return __fmaf_rn(-step, (float)(n - q - 1), 1.0f);
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned sa = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

#endif  // __CUDACC__

}  // namespace nerfb200
