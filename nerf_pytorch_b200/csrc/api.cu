// api.cu -- the extern "C" surface declared in include/nerfb200.h: argument checking, plan
// building, workspace carving and kernel orchestration for the whole per-ray path
// (predict_and_render_radiance, nerf/train_utils.py:28-127 of the reference).
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <atomic>

#include "common.cuh"

#define NB_TRY(expr)                    \
  do {                                  \
    int _rc = (expr);                   \
    if (_rc != NERFB200_OK) return _rc; \
  } while (0)

namespace nerfb200 {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int device_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  return sms;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return NERFB200_OK;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return NERFB200_ERR_CUDA;
}

static inline int pad8(int x) { return (x + 7) & ~7; }
static inline int pad4(int x) { return (x + 3) & ~3; }

int build_plan(const nerfb200_arch_t* a, Plan* p) {
  if (!a || !p) {
    set_error("build_plan: null argument");
    return NERFB200_ERR_INVALID;
  }
  memset(p, 0, sizeof(*p));
  if (a->hidden != 128 && a->hidden != 256) {
    set_error("unsupported hidden_size %d (kernels implement 128 and 256)", a->hidden);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (a->num_layers < 1 || a->num_layers > 16) {
    set_error("unsupported num_layers %d (1..16)", a->num_layers);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (a->skip_every <= 0) {
    set_error("skip_connect_every must be > 0 (got %d)", a->skip_every);
    return NERFB200_ERR_INVALID;
  }
  if (a->n_freq_xyz < 0 || a->n_freq_xyz > NERFB200_MAX_FREQS || a->n_freq_dir < 0 ||
      a->n_freq_dir > NERFB200_MAX_FREQS) {
    set_error("number of encoding functions out of range (max %d)", NERFB200_MAX_FREQS);
    return NERFB200_ERR_UNSUPPORTED;
  }
  const int H = a->hidden;
  p->hidden = H;
  p->use_viewdirs = a->use_viewdirs ? 1 : 0;
  p->n_freq_xyz = a->n_freq_xyz;
  p->n_freq_dir = a->n_freq_dir;
  p->inc_xyz = a->include_input_xyz ? 1 : 0;
  p->inc_dir = a->include_input_dir ? 1 : 0;
  p->dim_xyz = 3 * p->inc_xyz + 6 * a->n_freq_xyz;
  p->dim_dir = p->use_viewdirs ? 3 * p->inc_dir + 6 * a->n_freq_dir : 0;
  if (p->dim_xyz <= 0 || (p->use_viewdirs && p->dim_dir <= 0)) {
    set_error("empty encoding (dim_xyz %d, dim_dir %d)", p->dim_xyz, p->dim_dir);
    return NERFB200_ERR_UNSUPPORTED;
  }
  p->dim_xyz_pad = pad8(p->dim_xyz);
  p->dim_dir_pad = pad8(p->dim_dir);
  p->enc_tile_w = (p->dim_xyz + 15) & ~15;
  for (int i = 0; i < NERFB200_MAX_FREQS; ++i) {
    p->freq_xyz[i] = a->freq_xyz[i];
    p->freq_dir[i] = a->freq_dir[i];
  }

  int blob = 0, flat = 0, cum = 0, ng = 0;
  auto add_gemm = [&](int k_h, int enc_sel, int enc_real, int n, int relu, int src) {
    GemmLayer& g = p->g[ng];
    g.k_h = k_h;
    g.enc_sel = enc_sel;
    g.enc_real = enc_real;
    g.k_enc = pad8(enc_real);
    g.n = n;
    g.relu = relu;
    g.src = src;
    g.wt_off = blob;
    blob += (g.k_h + g.k_enc) * n;
    g.wh_off = blob;
    blob += n * g.k_h;
    g.b_off = blob;
    blob += n;
    g.k_tc = enc_sel == 1 ? k_h : k_h + g.k_enc;
    g.tc_off = blob;
    blob += 3 * ((g.k_tc + 15) & ~15) * n / 2;  // three fp16 copies (hs | h | l) of [K padded to 16][n]
    g.tcd_off = blob;
    blob += 3 * g.k_h * n / 2;                  // three fp16 copies of [n][k_h] for the dgrad chain
    g.cum_n = cum;
    cum += n;
    g.flat_w = flat;
    flat += n * (k_h + enc_real);
    g.flat_b = flat;
    flat += n;
    return ng++;
  };
  auto set_head = [&](int idx, int k, int n_out, int out_col, int src) {
    HeadLayer& h = p->h[idx];
    h.k = k;
    h.n_out = n_out;
    h.out_col = out_col;
    h.src = src;
    h.w_off = blob;
    blob += pad4(n_out * k);
    h.b_off = blob;
    blob += 4;
    h.flat_w = flat;
    flat += n_out * k;
    h.flat_b = flat;
    flat += n_out;
  };

  // trunk: layer1 (no activation, models.py:238) + layers_xyz (ReLU; wide iff allocated wide, :210-215)
  add_gemm(0, 0, p->dim_xyz, H, 0, -1);
  for (int i = 0; i < a->num_layers - 1; ++i) {
    const bool wide = (i % a->skip_every == 0) && i > 0 && i != a->num_layers - 1;
    add_gemm(H, 0, wide ? p->dim_xyz : 0, H, 1, ng - 1);
  }
  p->n_trunk = ng;
  if (p->use_viewdirs) {
    // flat order follows the canonical slot order: fc_feat, fc_alpha, layers_dir[0], fc_rgb
    const int feat = add_gemm(H, 0, 0, H, 1, p->n_trunk - 1);      // models.py:248
    set_head(0, H, 1, 3, p->n_trunk - 1);                          // fc_alpha, models.py:249
    const int dir = add_gemm(H, 1, p->dim_dir, H / 2, 1, feat);    // models.py:250-252
    set_head(1, H / 2, 3, 0, dir);                                 // fc_rgb, models.py:253
    p->n_head = 2;
  } else {
    set_head(0, H, 4, 0, p->n_trunk - 1);  // fc_out, models.py:256
    p->n_head = 1;
  }
  p->n_gemm = ng;
  p->enc_cum[0] = cum;
  cum += p->enc_tile_w;
  p->enc_cum[1] = cum;
  cum += p->dim_dir_pad;
  p->mask_base = cum;
  int mw = 0;
  for (int i = 0; i < ng; ++i) {
    p->g[i].mask_cum = mw;
    mw += p->g[i].n / 32;
  }
  cum += mw;
  p->sum_n = cum;
  p->blob_floats = blob;
  p->flat_floats = flat;
  return NERFB200_OK;
}

// slot -> (is_head, index)
static bool slot_lookup(const Plan& p, int slot, bool* is_head, int* idx) {
  const int nt = p.n_trunk;
  if (slot < 0) return false;
  if (slot < nt) {
    *is_head = false;
    *idx = slot;
    return true;
  }
  if (p.use_viewdirs) {
    switch (slot - nt) {
      case 0: *is_head = false; *idx = nt; return true;
      case 1: *is_head = true; *idx = 0; return true;
      case 2: *is_head = false; *idx = nt + 1; return true;
      case 3: *is_head = true; *idx = 1; return true;
      default: return false;
    }
  }
  if (slot == nt) {
    *is_head = true;
    *idx = 0;
    return true;
  }
  return false;
}

static inline int64_t align256(int64_t bytes) { return (bytes + 255) & ~int64_t(255); }

// activation stash of n points: whole 128-point tiles (the wgmma path stores tiles)
static inline int64_t stash_floats(const Plan& p, int64_t n) { return ((n + 127) & ~int64_t(127)) * p.sum_n; }

struct Workspace {
  int64_t z_c, raw_c, w_c, z_f, raw_f, stash_c, stash_f, gstash, d_raw, total;
};

// What a call needs of the MLP kernels it selects with `impl`.
enum Need {
  kInference,  // the forward alone: render_fwd(training = 0), mlp_fwd without a stash
  kStash,      // the forward that writes the activation stash a backward reads
  kBackward,   // the backward (its forward has run)
  kHalves,     // the backward as two calls, mlp_dgrad and mlp_wgrad: the fp32 kernels only
  kGradient,   // the density gradient at points (density_grad): the wgmma kernels only
};

// The one place that maps an impl code to the kernel families' predicates: 0 the fp32 CUDA cores, 1 wgmma, 3 the
// single-pass fp16 wgmma forward, which renders only.  Every other code is refused (2 is a query of impl_supported,
// not a family).  A refusal reads "<what> impl=N (<label>): <reason>".
static int check_impl(const Plan& p, int impl, int n_samples, Need need, const char* what) {
  char who[96];
  if (need == kGradient && (impl == 0 || impl == 3)) {
    set_error("%s impl=%d: the density gradient runs on the split-precision wgmma kernels only (impl=1); the %s is not "
              "differentiated", what, impl, impl == 0 ? "fp32 CUDA-core forward" : "single-pass fp16 forward");
    return NERFB200_ERR_UNSUPPORTED;
  }
  switch (impl) {
    case 0:
      snprintf(who, sizeof(who), "%s impl=0 (fp32 CUDA cores)", what);
      return simt_supported(p, who);
    case 1:
      if (need == kHalves) {
        set_error("%s: impl=1 (wgmma) fuses dgrad and wgrad into one kernel; call nerfb200_mlp_bwd", what);
        return NERFB200_ERR_UNSUPPORTED;
      }
      snprintf(who, sizeof(who), "%s impl=1 (wgmma)", what);
      NB_TRY(tc_supported(p, n_samples, /*training=*/need != kInference && need != kGradient, who));
      if (need == kGradient) return grad_tc_supported(p, who);
      return need == kBackward ? bwd_tc_supported(p, who) : NERFB200_OK;
    case 3:
      if (need != kInference) {
        set_error("%s: impl=3 (single-pass fp16 wgmma forward) is inference only; train with impl=0 or impl=1", what);
        return NERFB200_ERR_UNSUPPORTED;
      }
      snprintf(who, sizeof(who), "%s impl=3 (single-pass fp16 wgmma)", what);
      return tc_supported(p, n_samples, /*training=*/false, who);
    default:
      set_error("%s: unknown impl %d", what, impl);
      return NERFB200_ERR_INVALID;
  }
}

// The points of the render path: o + d z from the ray rows, view directions in columns 8..10.
static PointSrc ray_points(const float* rays, int ray_stride, const float* z) {
  return PointSrc{rays, ray_stride, z, nullptr, rays + 8, ray_stride};
}

// The MLP forward of one network on the kernels check_impl accepted; a non-null stash is written for the backward.
static int mlp_forward(const Plan& p, int impl, const float* blob, const PointSrc& src, int64_t n_rays, int n_samples,
                       float* raw, float* stash, cudaStream_t s) {
  if (impl == 0) return launch_mlp_fwd_simt(p, blob, src, n_rays, n_samples, raw, stash, s);
  return launch_mlp_fwd_tc(p, blob, src, n_rays, n_samples, raw, stash, /*fast=*/impl == 3, s);
}

// Its backward, accumulated into flat_grad.  gstash: impl 0 the gradient stash, impl 1 the gradient blob.  Both read
// the encodings from the stash; only the fused backward reads the view directions again.
static int mlp_backward(const Plan& p, int impl, const float* blob, const PointSrc& src, int64_t n_rays, int n_samples,
                        const float* d_raw, const float* stash, float* gstash, float* flat_grad, cudaStream_t s) {
  if (impl == 1)
    return launch_mlp_bwd_tc(p, blob, src.dirs, src.dir_stride, n_rays, n_samples, d_raw, stash, gstash, flat_grad, s);
  const int64_t P = n_rays * n_samples;
  NB_TRY(launch_dgrad_simt(p, blob, d_raw, stash, gstash, P, s));
  return launch_wgrad_simt(p, src.rays, src.ray_stride, src.z, n_samples, d_raw, stash, gstash, P, flat_grad, s);
}

static int check_opts(const nerfb200_render_opts_t* o) {
  if (!o) {
    set_error("null render options");
    return NERFB200_ERR_INVALID;
  }
  if (o->n_coarse < 2 || o->n_coarse > 1024 || o->n_fine < 0 || o->n_coarse + o->n_fine > 1024) {
    set_error("unsupported sample counts (n_coarse %d, n_fine %d; need 2 <= nc, nc + nf <= 1024)", o->n_coarse,
              o->n_fine);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (o->n_fine > 0 && o->n_coarse < 4) {
    set_error("hierarchical sampling needs n_coarse >= 4");
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

// What every render-family call starts from: the plans, the sample counts and the base workspace.
struct RenderSetup {
  Plan pc, pf;
  bool fine;  // a fine pass: n_fine > 0 and a fine arch
  int nc, ns;
  Workspace w;
};

// Builds the coarse plan, the fine plan when arch_f is given, checks the options and n_rays > 0 (refused with the
// text `empty`, or with none when it is NULL) and carves the base workspace.  The workspace queries pass arch_f as
// given, so that they refuse an invalid one even with n_fine = 0; the renders pass it only for a fine pass.
static int render_setup(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f, const nerfb200_render_opts_t* opts,
                        int64_t n, int training, const char* empty, RenderSetup* r) {
  NB_TRY(build_plan(arch_c, &r->pc));
  if (arch_f) NB_TRY(build_plan(arch_f, &r->pf));
  NB_TRY(check_opts(opts));
  if (n <= 0) {
    if (empty) set_error("%s", empty);
    return NERFB200_ERR_INVALID;
  }
  const Plan &pc = r->pc, &pf = r->pf;
  const bool fine = r->fine = arch_f && opts->n_fine > 0;
  const int64_t nc = r->nc = opts->n_coarse, ns = r->ns = opts->n_coarse + opts->n_fine;
  Workspace* w = &r->w;
  int64_t off = 0;
  auto take = [&](int64_t floats) {
    int64_t at = off;
    off += align256(floats * 4);
    return at;
  };
  w->z_c = take(n * nc);
  w->raw_c = take(n * nc * 4);
  w->w_c = take(n * nc);
  w->z_f = take(fine ? n * ns : 0);
  w->raw_f = take(fine ? n * ns * 4 : 0);
  if (training) {
    const int64_t sc = stash_floats(pc, n * nc);
    const int64_t sf = fine ? stash_floats(pf, n * ns) : 0;
    w->stash_c = take(sc);
    w->stash_f = take(sf);
    // backward scratch: the gradient stash of the CUDA-core path / the gradient blob of the wgmma path
    int64_t gs = sc > sf ? sc : sf;
    const int64_t bc = pc.hidden == 128 ? bwd_tc_scratch_floats(pc) : 0;
    const int64_t bf = (fine && pf.hidden == 128) ? bwd_tc_scratch_floats(pf) : 0;
    if (bc > gs) gs = bc;
    if (bf > gs) gs = bf;
    w->gstash = take(gs);
    w->d_raw = take(n * (fine ? ns : nc) * 4);
  } else {
    w->stash_c = w->stash_f = w->gstash = w->d_raw = off;
  }
  w->total = off;
  return NERFB200_OK;
}

}  // namespace nerfb200

using namespace nerfb200;

extern "C" {

int32_t nerfb200_version(void) { return NERFB200_VERSION; }
const char* nerfb200_last_error(void) { return g_err; }
int64_t nerfb200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
int64_t nerfb200_bwd_bytes_per_point(const nerfb200_arch_t* arch) {
  Plan p;
  if (build_plan(arch, &p) != NERFB200_OK) return -1;
  int64_t bytes = 16;  // d_raw
  for (int t = 0; t < p.n_gemm; ++t) {
    const GemmLayer& g = p.g[t];
    if (g.k_h > 0) bytes += 4 * g.k_h;                               // the layer input tile (hi + lo)
    if (g.k_enc > 0 && g.enc_sel == 0) bytes += 4 * p.enc_tile_w;    // the encoding tile
    if (g.relu) bytes += g.n / 8;                                    // ReLU bit mask
  }
  for (int h = 0; h < p.n_head; ++h) bytes += 4 * p.h[h].k;          // the heads' input tiles
  return bytes;
}

int32_t nerfb200_impl_supported(const nerfb200_arch_t* arch, int32_t n_samples, int32_t impl) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  if (impl == 2) return check_impl(p, 1, n_samples, kInference, "impl_supported");  // the wgmma forward alone
  return check_impl(p, impl, n_samples, impl == 3 ? kInference : kBackward, "impl_supported");
}

int64_t nerfb200_bwd_scratch_floats(const nerfb200_arch_t* arch, int64_t n_points, int32_t impl) {
  Plan p;
  if (build_plan(arch, &p) != NERFB200_OK || n_points < 0 ||
      check_impl(p, impl, 0, kBackward, "bwd_scratch_floats") != NERFB200_OK)
    return -1;
  return impl == 1 ? bwd_tc_scratch_floats(p) : stash_floats(p, n_points);
}

int64_t nerfb200_num_linear(const nerfb200_arch_t* arch) {
  Plan p;
  if (build_plan(arch, &p) != NERFB200_OK) return -1;
  return p.n_gemm + p.n_head;
}
int64_t nerfb200_flat_param_count(const nerfb200_arch_t* arch) {
  Plan p;
  if (build_plan(arch, &p) != NERFB200_OK) return -1;
  return p.flat_floats;
}
int64_t nerfb200_blob_floats(const nerfb200_arch_t* arch) {
  Plan p;
  if (build_plan(arch, &p) != NERFB200_OK) return -1;
  return p.blob_floats;
}
int64_t nerfb200_stash_floats(const nerfb200_arch_t* arch, int64_t n_points) {
  Plan p;
  if (build_plan(arch, &p) != NERFB200_OK || n_points < 0) return -1;
  return stash_floats(p, n_points);
}

int32_t nerfb200_flat_layout(const nerfb200_arch_t* arch, int32_t slot, int64_t* w_off, int64_t* b_off,
                             int32_t* in_features, int32_t* out_features) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  bool is_head;
  int idx;
  if (!slot_lookup(p, slot, &is_head, &idx)) {
    set_error("flat_layout: slot %d out of range", slot);
    return NERFB200_ERR_INVALID;
  }
  if (is_head) {
    if (w_off) *w_off = p.h[idx].flat_w;
    if (b_off) *b_off = p.h[idx].flat_b;
    if (in_features) *in_features = p.h[idx].k;
    if (out_features) *out_features = p.h[idx].n_out;
  } else {
    if (w_off) *w_off = p.g[idx].flat_w;
    if (b_off) *b_off = p.g[idx].flat_b;
    if (in_features) *in_features = p.g[idx].k_h + p.g[idx].enc_real;
    if (out_features) *out_features = p.g[idx].n;
  }
  return NERFB200_OK;
}

int32_t nerfb200_pack_weights(const nerfb200_arch_t* arch, const float* flat, float* blob, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  if (!flat || !blob) {
    set_error("pack_weights: null pointer");
    return NERFB200_ERR_INVALID;
  }
  return launch_pack(p, flat, blob, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_sample_coarse(const float* rays, int32_t ray_stride, int64_t n_rays, const float* t_rand,
                               int32_t n_coarse, int32_t perturb, int32_t lindisp, float* z, void* stream) {
  if (!rays || !z || n_rays <= 0 || n_coarse < 2 || ray_stride < 8 || (perturb && !t_rand)) {
    set_error("sample_coarse: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  return launch_sample_coarse(rays, ray_stride, n_rays, perturb ? rand_tensor(t_rand, n_coarse) : rand_none(), n_coarse,
                              perturb, lindisp, z, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_gen_rays(const float* c2w12_host, int32_t height, int32_t width, float focal, const int64_t* pixel_ids,
                          int64_t n, int32_t ndc, float near, float far, int32_t use_viewdirs, int32_t out_stride,
                          float* out, void* stream) {
  if (!c2w12_host || !out || n <= 0) {
    set_error("gen_rays: null pointer or empty batch");
    return NERFB200_ERR_INVALID;
  }
  return launch_gen_rays(c2w12_host, height, width, focal, pixel_ids, n, ndc, near, far, use_viewdirs, out_stride, out,
                         static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_pack_rays(const float* ro, const float* rd, int64_t n, int32_t height, int32_t width, float focal,
                           int32_t ndc, float near, float far, int32_t use_viewdirs, int32_t out_stride, float* out,
                           void* stream) {
  if (!ro || !rd || !out || n <= 0) {
    set_error("pack_rays: null pointer or empty batch");
    return NERFB200_ERR_INVALID;
  }
  return launch_pack_rays(ro, rd, n, height, width, focal, ndc, near, far, use_viewdirs, out_stride, out,
                          static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_encode(const nerfb200_arch_t* arch, int32_t which, const float* x, int64_t n, float* out,
                        void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  if (!x || !out || n <= 0 || which < 0 || which > 1 || (which == 1 && !p.use_viewdirs)) {
    set_error("encode: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  return launch_encode(p, which, x, n, out, static_cast<cudaStream_t>(stream));
}

static int check_mlp_args(const Plan& p, const void* blob, const float* rays, int ray_stride, const float* z,
                          int64_t n_rays, int n_samples) {
  if (!blob || !rays || !z || n_rays <= 0 || n_samples <= 0) {
    set_error("mlp: null pointer or empty input");
    return NERFB200_ERR_INVALID;
  }
  if (ray_stride < (p.use_viewdirs ? 11 : 8)) {
    set_error("mlp: ray_stride %d too small (need %d columns)", ray_stride, p.use_viewdirs ? 11 : 8);
    return NERFB200_ERR_INVALID;
  }
  if (n_rays * (int64_t)n_samples >= (int64_t(1) << 31)) {
    set_error("mlp: more than 2^31 points in one call; chunk the rays");
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

int32_t nerfb200_mlp_fwd(const nerfb200_arch_t* arch, const float* blob, const float* rays, int32_t ray_stride,
                         const float* z, int64_t n_rays, int32_t n_samples, float* raw, float* stash,
                         int32_t impl, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  NB_TRY(check_mlp_args(p, blob, rays, ray_stride, z, n_rays, n_samples));
  if (!raw) {
    set_error("mlp_fwd: null output");
    return NERFB200_ERR_INVALID;
  }
  NB_TRY(check_impl(p, impl, n_samples, stash ? kStash : kInference, "mlp_fwd"));
  return mlp_forward(p, impl, blob, ray_points(rays, ray_stride, z), n_rays, n_samples, raw, stash,
                     static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_mlp_bwd(const nerfb200_arch_t* arch, const float* blob, const float* rays, int32_t ray_stride,
                         const float* z, int64_t n_rays, int32_t n_samples, const float* d_raw,
                         const float* stash, float* gstash, float* flat_grad, int32_t impl, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  NB_TRY(check_mlp_args(p, blob, rays, ray_stride, z, n_rays, n_samples));
  if (!d_raw || !stash || !gstash || !flat_grad) {
    set_error("mlp_bwd: null pointer");
    return NERFB200_ERR_INVALID;
  }
  NB_TRY(check_impl(p, impl, n_samples, kBackward, "mlp_bwd"));
  return mlp_backward(p, impl, blob, ray_points(rays, ray_stride, z), n_rays, n_samples, d_raw, stash, gstash,
                      flat_grad, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_mlp_dgrad(const nerfb200_arch_t* arch, const float* blob, const float* d_raw, const float* stash,
                           float* gstash, int64_t n_points, int32_t impl, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  if (!blob || !d_raw || !stash || !gstash || n_points <= 0) {
    set_error("mlp_dgrad: null pointer or empty input");
    return NERFB200_ERR_INVALID;
  }
  NB_TRY(check_impl(p, impl, 0, kHalves, "mlp_dgrad"));
  return launch_dgrad_simt(p, blob, d_raw, stash, gstash, n_points, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_mlp_wgrad(const nerfb200_arch_t* arch, const float* rays, int32_t ray_stride, const float* z,
                           int64_t n_rays, int32_t n_samples, const float* d_raw, const float* stash,
                           const float* gstash, float* flat_grad, int32_t impl, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  if (!rays || !z || !d_raw || !stash || !gstash || !flat_grad || n_rays <= 0 || n_samples <= 0) {
    set_error("mlp_wgrad: null pointer or empty input");
    return NERFB200_ERR_INVALID;
  }
  NB_TRY(check_impl(p, impl, n_samples, kHalves, "mlp_wgrad"));
  return launch_wgrad_simt(p, rays, ray_stride, z, n_samples, d_raw, stash, gstash, n_rays * n_samples, flat_grad,
                           static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_composite_fwd(const float* raw, const float* z, const float* rays, int32_t ray_stride,
                               const float* noise, int64_t n_rays, int32_t n_samples, float noise_std,
                               int32_t white_bkgd, float* out, float* weights, void* stream) {
  if (!raw || !z || !rays || !out || n_rays <= 0 || n_samples <= 0 || n_samples > 1024 || ray_stride < 8) {
    set_error("composite_fwd: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  return launch_composite_fwd(raw, z, rays + 3, ray_stride, rand_tensor(noise, n_samples), n_rays, n_samples, noise_std,
                              white_bkgd, out, weights, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_composite_bwd(const float* raw, const float* z, const float* rays, int32_t ray_stride,
                               const float* noise, const float* g_out, int64_t n_rays, int32_t n_samples,
                               float noise_std, int32_t white_bkgd, float* d_raw, void* stream) {
  if (!raw || !z || !rays || !g_out || !d_raw || n_rays <= 0 || n_samples <= 0 || n_samples > 1024 ||
      ray_stride < 8) {
    set_error("composite_bwd: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  return launch_composite_bwd(raw, z, rays + 3, ray_stride, rand_tensor(noise, n_samples), g_out, nullptr,
                              /*sample_grads=*/false, n_rays, n_samples, noise_std, white_bkgd, d_raw,
                              static_cast<cudaStream_t>(stream));
}

static int check_pts_args(const Plan& p, const float* dirs, int dir_stride, int64_t n_rays, int n_samples,
                          const char* what) {
  if (n_rays <= 0 || n_samples <= 0) {
    set_error("%s: empty input", what);
    return NERFB200_ERR_INVALID;
  }
  if ((dirs != nullptr) != (p.use_viewdirs != 0) || dir_stride < 0) {
    set_error("%s: dirs must be given iff the architecture uses view directions (use_viewdirs %d, dirs %s, "
              "dir_stride %d >= 0)", what, p.use_viewdirs, dirs ? "given" : "NULL", dir_stride);
    return NERFB200_ERR_INVALID;
  }
  if (n_rays * (int64_t)n_samples >= (int64_t(1) << 31)) {
    set_error("%s: more than 2^31 points in one call; chunk the points", what);
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

int32_t nerfb200_mlp_fwd_pts(const nerfb200_arch_t* arch, const float* blob, const float* pts, const float* dirs,
                             int32_t dir_stride, int64_t n_rays, int32_t n_samples, float* raw, float* stash,
                             int32_t impl, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  NB_TRY(check_pts_args(p, dirs, dir_stride, n_rays, n_samples, "mlp_fwd_pts"));
  if (!blob || !pts || !raw) {
    set_error("mlp_fwd_pts: null pointer");
    return NERFB200_ERR_INVALID;
  }
  NB_TRY(check_impl(p, impl, n_samples, stash ? kStash : kInference, "mlp_fwd_pts"));
  return mlp_forward(p, impl, blob, PointSrc{nullptr, 0, nullptr, pts, dirs, dir_stride}, n_rays, n_samples, raw,
                     stash, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_density_grad_supported(const nerfb200_arch_t* arch, int32_t impl) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  return check_impl(p, impl, 0, kGradient, "density_grad");
}

int32_t nerfb200_density_grad(const nerfb200_arch_t* arch, const float* blob, const float* pts, int64_t n_points,
                              float* out, int32_t impl, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  if (!blob || !pts || !out || n_points <= 0) {
    set_error("density_grad: null pointer or empty input");
    return NERFB200_ERR_INVALID;
  }
  if (n_points >= (int64_t(1) << 31)) {
    set_error("density_grad: more than 2^31 points in one call; chunk the points");
    return NERFB200_ERR_UNSUPPORTED;
  }
  NB_TRY(check_impl(p, impl, 0, kGradient, "density_grad"));
  return launch_density_grad_tc(p, blob, pts, n_points, out, nullptr, static_cast<cudaStream_t>(stream));
}

// the bake runs the wgmma inference forward's trunk (impl 1) and its own direction loop
static int bake_check(const Plan& p) {
  NB_TRY(check_impl(p, 1, 0, kInference, "bake"));
  return bake_tc_supported(p, "bake impl=1 (wgmma)");
}

int32_t nerfb200_bake_supported(const nerfb200_arch_t* arch) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  return bake_check(p);
}

// the checks bake and bake_f16 share: the plan into *p, then the box, the pointers, the slot range, the architecture
static int check_bake(const char* what, const nerfb200_arch_t* arch, Plan* p, const float* blob,
                      const nerfb200_grid_t* box, const int32_t* bricks, int64_t first, int64_t count,
                      const void* values) {
  NB_TRY(build_plan(arch, p));
  NB_TRY(check_grid(box, what));
  const int64_t n_bricks = nerfb200_mesh_sparse_brick_count(box);
  if (!blob || !bricks || !values || first < 0 || count <= 0 || first + count > n_bricks) {
    set_error("%s: null pointer, or slots %lld .. %lld outside the box's %lld bricks", what, (long long)first,
              (long long)(first + count - 1), (long long)n_bricks);
    return NERFB200_ERR_INVALID;
  }
  if (count * kBakePts >= (int64_t(1) << 31)) {
    set_error("%s: %lld bricks are 2^31 lattice points or more in one call; split the slots", what, (long long)count);
    return NERFB200_ERR_UNSUPPORTED;
  }
  return bake_check(*p);
}

int32_t nerfb200_bake(const nerfb200_arch_t* arch, const float* blob, const nerfb200_grid_t* box, const int32_t* bricks,
                      int64_t first, int64_t count, float* values, float* logits, void* stream) {
  Plan p;
  NB_TRY(check_bake("bake", arch, &p, blob, box, bricks, first, count, values));
  BakeBasis basis;
  bake_basis(&basis);
  return launch_bake_tc(p, blob, *box, bricks, first, count, values, logits, basis, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_bake_f16(const nerfb200_arch_t* arch, const float* blob, const nerfb200_grid_t* box,
                          const int32_t* bricks, int64_t first, int64_t count, uint16_t* values, float* logits,
                          void* stream) {
  Plan p;
  NB_TRY(check_bake("bake_f16", arch, &p, blob, box, bricks, first, count, values));
  NB_TRY(check_f16_values("bake_f16", values));
  BakeBasis basis;
  bake_basis(&basis);
  return launch_bake_tc(p, blob, *box, bricks, first, count, values, logits, basis, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_mlp_bwd_pts(const nerfb200_arch_t* arch, const float* blob, const float* dirs, int32_t dir_stride,
                             int64_t n_rays, int32_t n_samples, const float* d_raw, const float* stash, float* gstash,
                             float* flat_grad, int32_t impl, void* stream) {
  Plan p;
  NB_TRY(build_plan(arch, &p));
  NB_TRY(check_pts_args(p, dirs, dir_stride, n_rays, n_samples, "mlp_bwd_pts"));
  if (!blob || !d_raw || !stash || !gstash || !flat_grad) {
    set_error("mlp_bwd_pts: null pointer");
    return NERFB200_ERR_INVALID;
  }
  NB_TRY(check_impl(p, impl, n_samples, kBackward, "mlp_bwd_pts"));
  return mlp_backward(p, impl, blob, PointSrc{nullptr, 0, nullptr, nullptr, dirs, dir_stride}, n_rays, n_samples,
                      d_raw, stash, gstash, flat_grad, static_cast<cudaStream_t>(stream));
}

static int check_volume_render_args(const float* raw, const float* z, const float* dirs, int dir_stride,
                                    int64_t n_rays, int n_samples, const char* what) {
  if (!raw || !z || !dirs || dir_stride < 0 || n_rays <= 0 || n_samples <= 0 || n_samples > 1024) {
    set_error("%s: invalid argument (null pointer, dir_stride < 0, or n_samples outside 1..1024)", what);
    return NERFB200_ERR_INVALID;
  }
  return NERFB200_OK;
}

int32_t nerfb200_volume_render_fwd(const float* raw, const float* z, const float* dirs, int32_t dir_stride,
                                   const float* noise, int64_t n_rays, int32_t n_samples, float noise_std,
                                   int32_t white_bkgd, float* out, float* weights, void* stream) {
  NB_TRY(check_volume_render_args(raw, z, dirs, dir_stride, n_rays, n_samples, "volume_render_fwd"));
  if (!out) {
    set_error("volume_render_fwd: null output");
    return NERFB200_ERR_INVALID;
  }
  return launch_composite_fwd(raw, z, dirs, dir_stride, rand_tensor(noise, n_samples), n_rays, n_samples, noise_std,
                              white_bkgd, out, weights, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_volume_render_bwd(const float* raw, const float* z, const float* dirs, int32_t dir_stride,
                                   const float* noise, const float* g_out, const float* g_weights, int64_t n_rays,
                                   int32_t n_samples, float noise_std, int32_t white_bkgd, float* d_raw, void* stream) {
  NB_TRY(check_volume_render_args(raw, z, dirs, dir_stride, n_rays, n_samples, "volume_render_bwd"));
  if (!g_out || !d_raw) {
    set_error("volume_render_bwd: null pointer");
    return NERFB200_ERR_INVALID;
  }
  return launch_composite_bwd(raw, z, dirs, dir_stride, rand_tensor(noise, n_samples), g_out, g_weights,
                              /*sample_grads=*/true, n_rays, n_samples, noise_std, white_bkgd, d_raw,
                              static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_sample_pdf_merge(const float* z_coarse, const float* weights_coarse, const float* u,
                                  const float* cdf_in, int64_t n_rays, int32_t n_coarse, int32_t n_fine,
                                  float* z_fine, float* z_samples, int32_t* inds, float* cdf_out, void* stream) {
  if (!z_coarse || (!weights_coarse && !cdf_in) || n_rays <= 0 || n_coarse < 4 || n_fine <= 0 ||
      n_coarse + n_fine > 1024) {
    set_error("sample_pdf_merge: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  // u NULL: no source, so the kernel resamples at the det=True linspace
  return launch_sample_pdf_merge(z_coarse, weights_coarse, rand_tensor(u, n_fine), cdf_in, n_rays, n_coarse, n_fine,
                                 z_fine, z_samples, inds, cdf_out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

namespace nerfb200 {

static int check_rng(const nerfb200_rng_t* rng, const char* what) {
  if (!rng) {
    set_error("%s: null rng", what);
    return NERFB200_ERR_INVALID;
  }
  if (rng->step >= (uint64_t(1) << 30) || rng->ray_offset < 0) {
    set_error("%s: rng step %llu must be < 2^30 and ray_offset %lld >= 0", what, (unsigned long long)rng->step,
              (long long)rng->ray_offset);
    return NERFB200_ERR_INVALID;
  }
  return NERFB200_OK;
}

// The four random inputs of one render call, rnd[kRandTRand], rnd[kRandNoiseC], rnd[kRandU], rnd[kRandNoiseF]: the
// seeded stream when rng is set, else the tensors.  An input the options do not use gets no source, so with perturb off
// the resampling kernel builds the det=True linspace for u.
static int render_randoms(const char* what, const nerfb200_render_opts_t& o, const nerfb200_rng_t* rng,
                          const float* const tensor[4], RandSrc rnd[4]) {
  if (rng) {
    NB_TRY(check_rng(rng, what));
    for (int s = 0; s < 4; ++s)
      if (tensor[s]) {
        set_error("%s: both an rng and a random tensor (stream %d) given", what, s);
        return NERFB200_ERR_INVALID;
      }
  }
  const bool fine = o.n_fine > 0, noise = o.noise_std > 0.f;
  const bool used[4] = {o.perturb != 0, noise, o.perturb && fine, noise && fine};
  const int64_t per_ray[4] = {o.n_coarse, o.n_coarse, o.n_fine, o.n_coarse + o.n_fine};
  for (int s = 0; s < 4; ++s)
    rnd[s] = !used[s] ? rand_none() : rng ? rand_seeded(*rng, s) : rand_tensor(tensor[s], per_ray[s]);
  return NERFB200_OK;
}

// An occupancy grid's sections, reused by both passes: the compaction scratch, the row map, its blocks and the live
// block count.
struct GridWorkspace {
  int64_t scratch, map, blocks, n_blocks, total;
};
static GridWorkspace carve_grid(int64_t base, int64_t n_rays, int n_samples) {
  GridWorkspace g;
  const int64_t mb = grid_max_blocks(n_rays, n_samples);
  g.scratch = base;
  g.map = g.scratch + align256(grid_scratch_ints(n_rays, n_samples) * 4);
  g.blocks = g.map + align256(mb * 64 * 4);
  g.n_blocks = g.blocks + align256(mb * 8);
  g.total = g.n_blocks + 256;
  return g;
}

// The sections of an early-stopping last pass: its per-ray state (StopState), the groups' first blocks, one round's row
// map, its blocks, block count and row total.
struct StopWorkspace {
  int64_t order, n_eval, T, counts, first_block, map, blocks, n_blocks, rows, total;
};
static StopWorkspace carve_stop(int64_t base, int64_t n_rays, int n_samples) {
  StopWorkspace sw;
  const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
  const int64_t mb = stop_round_max_blocks(n_rays, n_samples);
  sw.order = base;
  sw.n_eval = sw.order + align256(n_rays * n_samples * 4);
  sw.T = sw.n_eval + align256(n_rays * 4);
  sw.counts = sw.T + align256(n_rays * 4);
  sw.first_block = sw.counts + align256(groups * 4);
  sw.map = sw.first_block + align256(groups * 4);
  sw.blocks = sw.map + align256(mb * 64 * 4);
  sw.n_blocks = sw.blocks + align256(mb * 8);
  sw.rows = sw.n_blocks + 256;
  sw.total = sw.rows + 256;
  return sw;
}

// A normal map's sections: the last pass's weights, the compaction's count / first / total, the compacted points and
// their density_grad output.
struct NormalWorkspace {
  int64_t weights, count, first, total, pts, grad, end;
};
static NormalWorkspace carve_normal(int64_t base, int64_t n_rays, int n_samples) {
  NormalWorkspace nw;
  const int64_t P = n_rays * n_samples;
  nw.weights = base;
  nw.count = nw.weights + align256(P * 4);
  nw.first = nw.count + align256(n_rays * 4);
  nw.total = nw.first + align256(n_rays * 4);
  nw.pts = nw.total + 256;
  nw.grad = nw.pts + align256(P * 12);
  nw.end = nw.grad + align256(P * 16);
  return nw;
}

// The sections the inference variants add after the base workspace, in this order.  The grid's are sized for the
// larger pass it compacts: the fine pass, unless that pass stops early (then the stop rounds compact it).  The stop
// sections are sized for the last pass.  The normal map's follow the layout without early stopping, the larger of the
// two, so that their offsets do not depend on it.
struct ExtraWorkspace {
  GridWorkspace grid;
  StopWorkspace stop;
  NormalWorkspace normal;
};
static ExtraWorkspace carve_extras(const RenderSetup& r, int64_t n_rays, bool stop) {
  const int n_last = r.fine ? r.ns : r.nc;
  const GridWorkspace g = carve_grid(r.w.total, n_rays, stop ? r.nc : n_last);
  const StopWorkspace widest = carve_stop(carve_grid(r.w.total, n_rays, n_last).total, n_rays, n_last);
  return {g, carve_stop(g.total, n_rays, n_last), carve_normal(widest.total, n_rays, n_last)};
}

// A render_fwd-family call: render_fwd's arguments, then what the inference variants add to them.  Those are an
// occupancy grid (grid != NULL), early ray termination of the last pass below transmittance stop_t with its optional
// stop_sample output, the last pass's weights written to last_weights (normal maps), and the evaluated samples of each
// pass counted into n_evaluated.
struct RenderCall {
  const nerfb200_arch_t *arch_c, *arch_f;
  const nerfb200_render_opts_t* opts;
  const float *blob_c, *blob_f, *rays;
  int32_t ray_stride;
  int64_t n_rays;
  const nerfb200_rng_t* rng;
  const float* tensor[4];  // t_rand, noise_c, u, noise_f
  float *out_coarse, *out_fine;
  void* workspace;
  int32_t training, impl;
  void* stream;
  const nerfb200_grid_t* grid;
  const uint32_t* bits;
  bool stop;
  float stop_t;
  int32_t* stop_sample;
  float* last_weights;
  int64_t* n_evaluated;
};

static int check_grid_bits(const char* what, const nerfb200_grid_t* grid, const uint32_t* bits) {
  if ((grid == nullptr) == (bits == nullptr)) return NERFB200_OK;
  set_error("%s: a grid descriptor and its bits come together (descriptor %s, bits %s)", what, grid ? "given" : "NULL",
            bits ? "given" : "NULL");
  return NERFB200_ERR_INVALID;
}

// The refusals of a render_fwd-family call after its setup, in order and before any launch; rnd receives the call's
// random sources.
static int check_forward(const char* what, const RenderCall& a, const RenderSetup& r, RandSrc rnd[4]) {
  const nerfb200_render_opts_t& o = *a.opts;
  NB_TRY(render_randoms(what, o, a.rng, a.tensor, rnd));
  if (o.n_fine > 0 && (!a.arch_f || !a.blob_f || !a.out_fine)) {
    set_error("%s: fine pass requested but fine model / output missing", what);
    return NERFB200_ERR_INVALID;
  }
  if (!a.rays || !a.out_coarse || !a.workspace || !a.blob_c) {
    set_error("%s: null pointer or empty batch", what);
    return NERFB200_ERR_INVALID;
  }
  if (o.perturb && (!rnd[kRandTRand].present() || (r.fine && !rnd[kRandU].present()))) {
    set_error("%s: perturb set but t_rand or u missing", what);
    return NERFB200_ERR_INVALID;
  }
  if (a.grid) {
    NB_TRY(check_grid(a.grid, what));
    if (!a.bits) {
      set_error("%s: null grid bitfield", what);
      return NERFB200_ERR_INVALID;
    }
    if (a.training || a.impl == 0) {
      set_error("%s: the occupancy grid renders only (training = 0), on the wgmma inference forward: impl 1 or 3, not "
                "impl=%d", what, a.impl);
      return NERFB200_ERR_UNSUPPORTED;
    }
    if (grid_max_blocks(a.n_rays, r.ns) * 64 >= (int64_t(1) << 31)) {
      set_error("%s: more than 2^31 map rows in one call; chunk the rays", what);
      return NERFB200_ERR_UNSUPPORTED;
    }
  }
  if (a.stop) {
    if (a.training || a.impl == 0) {
      set_error("%s: early ray termination renders only (training = 0), on the wgmma inference forward: impl 1 or 3, "
                "not impl=%d", what, a.impl);
      return NERFB200_ERR_UNSUPPORTED;
    }
    if (!(a.stop_t >= 0.f && a.stop_t < 1.f)) {
      set_error("%s: stop_transmittance %g must be in [0, 1)", what, a.stop_t);
      return NERFB200_ERR_INVALID;
    }
  }
  const char* base = static_cast<const char*>(a.workspace);
  const Need need = a.training ? kStash : kInference;
  NB_TRY(check_mlp_args(r.pc, a.blob_c, a.rays, a.ray_stride, reinterpret_cast<const float*>(base + r.w.z_c), a.n_rays,
                        r.nc));
  NB_TRY(check_impl(r.pc, a.impl, r.nc, need, what));
  if (!r.fine) return NERFB200_OK;
  NB_TRY(check_mlp_args(r.pf, a.blob_f, a.rays, a.ray_stride, reinterpret_cast<const float*>(base + r.w.z_f), a.n_rays,
                        r.ns));
  return check_impl(r.pf, a.impl, r.ns, need, what);
}

// The passes of a checked render_fwd-family call.  Without extras the launches are exactly render_fwd's; with a grid
// (inference only) the MLP runs over each pass's compacted samples.
static int render_forward(const RenderCall& a, const RenderSetup& r, const RandSrc rnd[4]) {
  const nerfb200_render_opts_t& o = *a.opts;
  const int64_t n_rays = a.n_rays;
  const float* rays = a.rays;
  const int ray_stride = a.ray_stride, nc = r.nc;
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](int64_t off) { return reinterpret_cast<float*>(base + off); };
  auto I = [&](int64_t off) { return reinterpret_cast<int*>(base + off); };
  cudaStream_t s = static_cast<cudaStream_t>(a.stream);
  const ExtraWorkspace e = carve_extras(r, n_rays, a.stop);
  // the last pass with early ray termination: one marking launch, then rounds of compaction, MLP and the per-ray
  // transmittance update.  Rounds after every ray has finished have no blocks.
  auto stop_rounds = [&](bool is_fine, const Plan& p, const float* blob, int n, const float* z, float* raw) {
    const StopWorkspace& sw = e.stop;
    const int64_t groups = (n_rays + kGridGroupRays - 1) / kGridGroupRays;
    const StopState st{I(sw.order), I(sw.n_eval), F(sw.T), a.stop_sample, I(sw.counts)};
    int* nb = I(sw.n_blocks);
    int64_t* rows = reinterpret_cast<int64_t*>(base + sw.rows);
    // the coarse pass of a two-pass render without a grid ran every sample
    int64_t* coarse_rows = (is_fine && !a.grid && a.n_evaluated) ? a.n_evaluated : nullptr;
    NB_TRY(launch_stop_mark(a.grid ? *a.grid : nerfb200_grid_t{}, a.bits, rays, ray_stride, z, n_rays, n, raw, st,
                            coarse_rows, n_rays * nc, s));
    const RowMap m{I(sw.map), reinterpret_cast<const int2*>(base + sw.blocks), nb};
    const int64_t mb = stop_round_max_blocks(n_rays, n);
    for (int k = 0; k * kStopRound < n; ++k) {
      NB_TRY(launch_grid_scan(I(sw.counts), groups, I(sw.first_block), nb, rows, s));
      NB_TRY(launch_stop_scatter(st, I(sw.first_block), n_rays, n, k, I(sw.map), I(sw.blocks), s));
      NB_TRY(launch_mlp_fwd_tc_map(p, blob, rays, ray_stride, z, n_rays, n, m, mb, raw, a.impl == 3, s));
      NB_TRY(launch_stop_update(raw, z, rays + 3, ray_stride, rnd[is_fine ? kRandNoiseF : kRandNoiseC], o.noise_std,
                                n_rays, n, k, a.stop_t, st, rows, a.n_evaluated ? a.n_evaluated + is_fine : nullptr, s));
    }
    return NERFB200_OK;
  };
  // the MLP of one pass: every sample, or with a grid the compacted samples (skipped ones get raw = [0 0 0 -inf]), or
  // in the last pass of an early-stopping render the rounds above
  auto mlp = [&](bool is_fine, const Plan& p, const float* blob, int n, const float* z, float* raw, float* stash) {
    if (a.stop && is_fine == r.fine) return stop_rounds(is_fine, p, blob, n, z, raw);
    if (!a.grid)
      return mlp_forward(p, a.impl, blob, ray_points(rays, ray_stride, z), n_rays, n, raw, a.training ? stash : nullptr,
                         s);
    const GridWorkspace& gw = e.grid;
    int* nb = I(gw.n_blocks);
    NB_TRY(launch_grid_compact(*a.grid, a.bits, rays, ray_stride, z, n_rays, n, raw, I(gw.map), I(gw.blocks), nb,
                               a.n_evaluated ? a.n_evaluated + is_fine : nullptr, I(gw.scratch), s));
    const RowMap m{I(gw.map), reinterpret_cast<const int2*>(base + gw.blocks), nb};
    return launch_mlp_fwd_tc_map(p, blob, rays, ray_stride, z, n_rays, n, m, grid_max_blocks(n_rays, n), raw,
                                 a.impl == 3, s);
  };

  // one pass: depths -> MLP -> compositing.  The coarse pass (train_utils.py:45-94) takes stratified depths, the fine
  // pass (:96-125) resamples the coarse weights' pdf and merges the two sets.
  auto pass = [&](bool is_fine, const Plan& p, const float* blob, int n, float* z, float* raw, float* stash,
                  float* out, float* weights) {
    if (is_fine)
      NB_TRY(launch_sample_pdf_merge(F(r.w.z_c), F(r.w.w_c), rnd[kRandU], nullptr, n_rays, nc, o.n_fine, z, nullptr,
                                     nullptr, nullptr, s));
    else
      NB_TRY(launch_sample_coarse(rays, ray_stride, n_rays, rnd[kRandTRand], nc, o.perturb, o.lindisp, z, s));
    NB_TRY(mlp(is_fine, p, blob, n, z, raw, stash));
    return launch_composite_fwd(raw, z, rays + 3, ray_stride, rnd[is_fine ? kRandNoiseF : kRandNoiseC], n_rays, n,
                                o.noise_std, o.white_bkgd, out, weights, s);
  };
  // last_weights (normal maps): the last pass's compositing also writes its weights there
  NB_TRY(pass(false, r.pc, a.blob_c, nc, F(r.w.z_c), F(r.w.raw_c), F(r.w.stash_c), a.out_coarse,
              r.fine || !a.last_weights ? F(r.w.w_c) : a.last_weights));
  if (!r.fine) return NERFB200_OK;
  return pass(true, r.pf, a.blob_f, r.ns, F(r.w.z_f), F(r.w.raw_f), F(r.w.stash_f), a.out_fine, a.last_weights);
}

// render_fwd, render_fwd_grid and render_fwd_early_stop: the setup, the checks, then the passes
static int render_forward_call(const char* what, const RenderCall& a) {
  char empty[96];
  snprintf(empty, sizeof(empty), "%s: null pointer or empty batch", what);
  RenderSetup r;
  NB_TRY(render_setup(a.arch_c, a.opts && a.opts->n_fine > 0 ? a.arch_f : nullptr, a.opts, a.n_rays, a.training, empty,
                      &r));
  RandSrc rnd[4];
  NB_TRY(check_forward(what, a, r, rnd));
  return render_forward(a, r, rnd);
}

// render_fwd_normals, and with `world` its NDC render's world-space normal map (nerfb200.h "NDC scenes")
static int render_normals(const char* what, RenderCall a, float* normals, const NdcMap* world) {
  NB_TRY(check_grid_bits(what, a.grid, a.bits));
  if (a.stop_t != a.stop_t) {
    set_error("%s: stop_transmittance is NaN (negative: no early stopping)", what);
    return NERFB200_ERR_INVALID;
  }
  if (!normals || !a.workspace) {
    set_error("%s: null normals or workspace", what);
    return NERFB200_ERR_INVALID;
  }
  NB_TRY(check_opts(a.opts));
  const bool fine = a.opts->n_fine > 0;
  Plan pl;
  NB_TRY(build_plan(fine ? a.arch_f : a.arch_c, &pl));
  NB_TRY(check_impl(pl, a.impl, 0, kGradient, what));  // impl 1 alone, before any launch
  RenderSetup r;
  NB_TRY(render_setup(a.arch_c, fine ? a.arch_f : nullptr, a.opts, a.n_rays, /*training=*/0,
                      "render_fwd_normals: empty batch", &r));
  a.stop = a.stop_t >= 0.f;
  const NormalWorkspace nw = carve_extras(r, a.n_rays, a.stop).normal;
  char* base = static_cast<char*>(a.workspace);
  a.last_weights = reinterpret_cast<float*>(base + nw.weights);
  RandSrc rnd[4];
  NB_TRY(check_forward(what, a, r, rnd));
  NB_TRY(render_forward(a, r, rnd));
  const int64_t n_rays = a.n_rays;
  const int n_last = fine ? r.ns : r.nc;
  const float* z_last = reinterpret_cast<const float*>(base + (fine ? r.w.z_f : r.w.z_c));
  const NormalState st{reinterpret_cast<int*>(base + nw.count), reinterpret_cast<int*>(base + nw.first),
                       reinterpret_cast<int*>(base + nw.total), reinterpret_cast<float*>(base + nw.pts),
                       reinterpret_cast<float*>(base + nw.grad)};
  cudaStream_t s = static_cast<cudaStream_t>(a.stream);
  NB_TRY(launch_normal_compact(a.rays, a.ray_stride, z_last, a.last_weights, n_rays, n_last, st, s));
  NB_TRY(launch_density_grad_tc(pl, fine ? a.blob_f : a.blob_c, st.pts, n_rays * n_last, st.grad, st.total, s));
  return launch_normal_sum(a.last_weights, n_rays, n_last, st, normals, s, world);
}

}  // namespace nerfb200

extern "C" {

int64_t nerfb200_render_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                        const nerfb200_render_opts_t* opts, int64_t n_rays, int32_t training) {
  RenderSetup r;
  if (render_setup(coarse, fine, opts, n_rays, training, nullptr, &r) != NERFB200_OK) return -1;
  return r.w.total;
}

/* Byte offsets of the named sections of the render workspace (test hook): order
 * z_coarse, raw_coarse, weights_coarse, z_fine, raw_fine, stash_coarse, stash_fine, gstash, d_raw. */
int32_t nerfb200_render_workspace_layout(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                         const nerfb200_render_opts_t* opts, int64_t n_rays, int32_t training,
                                         int64_t* offsets9) {
  RenderSetup r;
  NB_TRY(render_setup(coarse, fine, opts, n_rays, training, "workspace_layout: invalid argument", &r));
  if (!offsets9) {
    set_error("workspace_layout: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  const Workspace& w = r.w;
  const int64_t v[9] = {w.z_c, w.raw_c, w.w_c, w.z_f, w.raw_f, w.stash_c, w.stash_f, w.gstash, w.d_raw};
  for (int i = 0; i < 9; ++i) offsets9[i] = v[i];
  return NERFB200_OK;
}

int32_t nerfb200_render_fwd(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                            const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                            const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                            const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                            float* out_coarse, float* out_fine, void* workspace, int32_t training, int32_t impl,
                            void* stream) {
  return render_forward_call("render_fwd", {arch_c, arch_f, opts, blob_c, blob_f, rays, ray_stride, n_rays, rng,
                                            {t_rand, noise_c, u, noise_f}, out_coarse, out_fine, workspace, training,
                                            impl, stream});
}

int64_t nerfb200_render_grid_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                             const nerfb200_render_opts_t* opts, int64_t n_rays) {
  RenderSetup r;
  if (render_setup(coarse, fine, opts, n_rays, /*training=*/0, nullptr, &r) != NERFB200_OK) return -1;
  return carve_extras(r, n_rays, /*stop=*/false).grid.total;
}

int32_t nerfb200_render_fwd_grid(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                 const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                 const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                                 const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                                 const nerfb200_grid_t* grid, const uint32_t* bits, float* out_coarse, float* out_fine,
                                 void* workspace, int32_t impl, int64_t* n_evaluated, void* stream) {
  if (!grid) {
    set_error("render_fwd_grid: null grid descriptor");
    return NERFB200_ERR_INVALID;
  }
  return render_forward_call("render_fwd_grid", {arch_c, arch_f, opts, blob_c, blob_f, rays, ray_stride, n_rays, rng,
                                                 {t_rand, noise_c, u, noise_f}, out_coarse, out_fine, workspace,
                                                 /*training=*/0, impl, stream, grid, bits, false, 0.f, nullptr,
                                                 nullptr, n_evaluated});
}

int32_t nerfb200_render_early_stop_round(void) { return kStopRound; }

int64_t nerfb200_render_early_stop_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                                   const nerfb200_render_opts_t* opts, int64_t n_rays) {
  RenderSetup r;
  if (render_setup(coarse, fine, opts, n_rays, /*training=*/0, nullptr, &r) != NERFB200_OK) return -1;
  return carve_extras(r, n_rays, /*stop=*/true).stop.total;
}

int32_t nerfb200_render_fwd_early_stop(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                       const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                       const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                                       const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                                       const nerfb200_grid_t* grid, const uint32_t* bits, float stop_transmittance,
                                       float* out_coarse, float* out_fine, void* workspace, int32_t impl,
                                       int64_t* n_evaluated, int32_t* stop_sample, void* stream) {
  NB_TRY(check_grid_bits("render_fwd_early_stop", grid, bits));
  return render_forward_call("render_fwd_early_stop", {arch_c, arch_f, opts, blob_c, blob_f, rays, ray_stride, n_rays,
                                                       rng, {t_rand, noise_c, u, noise_f}, out_coarse, out_fine,
                                                       workspace, /*training=*/0, impl, stream, grid, bits, true,
                                                       stop_transmittance, stop_sample, nullptr, n_evaluated});
}

int64_t nerfb200_render_normals_workspace_bytes(const nerfb200_arch_t* coarse, const nerfb200_arch_t* fine,
                                                const nerfb200_render_opts_t* opts, int64_t n_rays) {
  RenderSetup r;
  if (render_setup(coarse, fine, opts, n_rays, /*training=*/0, "render_fwd_normals: empty batch", &r) != NERFB200_OK)
    return -1;
  return carve_extras(r, n_rays, /*stop=*/false).normal.end;
}

int32_t nerfb200_render_fwd_normals(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                    const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                    const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                                    const float* t_rand, const float* noise_c, const float* u, const float* noise_f,
                                    const nerfb200_grid_t* grid, const uint32_t* bits, float stop_transmittance,
                                    float* out_coarse, float* out_fine, float* normals, void* workspace, int32_t impl,
                                    void* stream) {
  return render_normals("render_fwd_normals", {arch_c, arch_f, opts, blob_c, blob_f, rays, ray_stride, n_rays, rng,
                                               {t_rand, noise_c, u, noise_f}, out_coarse, out_fine, workspace,
                                               /*training=*/0, impl, stream, grid, bits, false, stop_transmittance},
                        normals, nullptr);
}

int32_t nerfb200_render_fwd_normals_ndc(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                                        const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                                        const float* rays, int32_t ray_stride, int64_t n_rays,
                                        const nerfb200_rng_t* rng, const float* t_rand, const float* noise_c,
                                        const float* u, const float* noise_f, const nerfb200_grid_t* grid,
                                        const uint32_t* bits, float stop_transmittance, const nerfb200_ndc_t* ndc,
                                        float* out_coarse, float* out_fine, float* normals, void* workspace,
                                        int32_t impl, void* stream) {
  NdcMap m;
  NB_TRY(make_ndc_map(ndc, &m, "render_fwd_normals_ndc"));
  return render_normals("render_fwd_normals_ndc", {arch_c, arch_f, opts, blob_c, blob_f, rays, ray_stride, n_rays, rng,
                                                   {t_rand, noise_c, u, noise_f}, out_coarse, out_fine, workspace,
                                                   /*training=*/0, impl, stream, grid, bits, false,
                                                   stop_transmittance},
                        normals, &m);
}

int32_t nerfb200_ndc_mesh_to_world(const nerfb200_ndc_t* ndc, const float* vertices, const int32_t* faces,
                                   const float* view_dirs, int64_t n_vertices, int64_t n_faces, float* world_vertices,
                                   int32_t* world_faces, float* world_dirs, void* stream) {
  NdcMap m;
  NB_TRY(make_ndc_map(ndc, &m, "ndc_mesh_to_world"));
  if (n_vertices < 0 || n_faces < 0 || (n_vertices > 0 && (!vertices || !world_vertices)) ||
      (n_faces > 0 && (!faces || !world_faces)) || ((view_dirs == nullptr) != (world_dirs == nullptr))) {
    set_error("ndc_mesh_to_world: a negative count, a null pointer, or view_dirs without world_dirs (or the reverse)");
    return NERFB200_ERR_INVALID;
  }
  return launch_ndc_mesh_to_world(m, vertices, faces, view_dirs, n_vertices, n_faces, world_vertices, world_faces,
                                  n_vertices > 0 ? world_dirs : nullptr, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_ndc_from_world(const nerfb200_ndc_t* ndc, const float* p, int64_t n, float* q, void* stream) {
  NdcMap m;
  NB_TRY(make_ndc_map(ndc, &m, "ndc_from_world"));
  if (n < 0 || (n > 0 && (!p || !q))) {
    set_error("ndc_from_world: a negative count or a null pointer");
    return NERFB200_ERR_INVALID;
  }
  return launch_ndc_from_world(m, p, n, q, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_ndc_grad_to_world(const nerfb200_ndc_t* ndc, const float* q, const float* rows, int64_t n, float* out,
                                   void* stream) {
  NdcMap m;
  NB_TRY(make_ndc_map(ndc, &m, "ndc_grad_to_world"));
  if (n < 0 || (n > 0 && (!q || !rows || !out))) {
    set_error("ndc_grad_to_world: a negative count or a null pointer");
    return NERFB200_ERR_INVALID;
  }
  return launch_ndc_grad_to_world(m, q, rows, n, out, static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_render_bwd(const nerfb200_arch_t* arch_c, const nerfb200_arch_t* arch_f,
                            const nerfb200_render_opts_t* opts, const float* blob_c, const float* blob_f,
                            const float* rays, int32_t ray_stride, int64_t n_rays, const nerfb200_rng_t* rng,
                            const float* noise_c, const float* noise_f, const float* g_coarse, const float* g_fine,
                            void* workspace, float* flat_grad_c, float* flat_grad_f, int32_t impl, int32_t parts,
                            void* stream) {
  RenderSetup r;
  NB_TRY(render_setup(arch_c, opts && opts->n_fine > 0 ? arch_f : nullptr, opts, n_rays, /*training=*/1,
                      "render_bwd: null pointer or empty batch", &r));
  const float* const tensor[4] = {nullptr, noise_c, nullptr, noise_f};
  RandSrc rnd[4];
  NB_TRY(render_randoms("render_bwd", *opts, rng, tensor, rnd));
  const bool fine = opts->n_fine > 0;
  if (fine && (!arch_f || !blob_f || !g_fine || !flat_grad_f)) {
    set_error("render_bwd: fine pass present but fine model / grads missing");
    return NERFB200_ERR_INVALID;
  }
  if (!rays || !g_coarse || !workspace || !blob_c || !flat_grad_c) {
    set_error("render_bwd: null pointer or empty batch");
    return NERFB200_ERR_INVALID;
  }
  if ((parts & 3) == 0) {
    set_error("render_bwd: parts must select the fine (1) and / or the coarse (2) backward");
    return NERFB200_ERR_INVALID;
  }
  const bool run_fine = fine && (parts & 1), run_coarse = parts & 2;
  if (run_fine) NB_TRY(check_impl(r.pf, impl, r.ns, kBackward, "render_bwd"));
  if (run_coarse) NB_TRY(check_impl(r.pc, impl, r.nc, kBackward, "render_bwd"));
  char* base = static_cast<char*>(workspace);
  auto F = [&](int64_t off) { return reinterpret_cast<float*>(base + off); };
  cudaStream_t s = static_cast<cudaStream_t>(stream);

  // one network's part: compositing backward into d_raw, then the MLP backward
  auto part = [&](const Plan& p, const float* blob, int n, const float* z, const float* raw, const float* stash,
                  const RandSrc& noise, const float* g, float* flat_grad) {
    NB_TRY(launch_composite_bwd(raw, z, rays + 3, ray_stride, noise, g, nullptr, /*sample_grads=*/false, n_rays, n,
                                opts->noise_std, opts->white_bkgd, F(r.w.d_raw), s));
    return mlp_backward(p, impl, blob, ray_points(rays, ray_stride, z), n_rays, n, F(r.w.d_raw), stash, F(r.w.gstash),
                        flat_grad, s);
  };
  if (run_fine)
    NB_TRY(part(r.pf, blob_f, r.ns, F(r.w.z_f), F(r.w.raw_f), F(r.w.stash_f), rnd[kRandNoiseF], g_fine, flat_grad_f));
  if (!run_coarse) return NERFB200_OK;
  // the coarse weights feed the resampler only through a detach (train_utils.py:103), so the
  // coarse net's gradient comes from rgb/disp/acc_coarse alone.
  return part(r.pc, blob_c, r.nc, F(r.w.z_c), F(r.w.raw_c), F(r.w.stash_c), rnd[kRandNoiseC], g_coarse, flat_grad_c);
}

int32_t nerfb200_random_fill(const nerfb200_rng_t* rng, int32_t stream_id, int64_t n_rays, int32_t per_ray, float* out,
                             void* stream) {
  NB_TRY(check_rng(rng, "random_fill"));
  if (!out || n_rays <= 0 || per_ray <= 0 || stream_id < 0 || stream_id > 3) {
    set_error("random_fill: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  return launch_random_fill(rand_seeded(*rng, stream_id), stream_id, n_rays, per_ray, out,
                            static_cast<cudaStream_t>(stream));
}

int32_t nerfb200_adam_step(float* p, const float* g, float* m, float* v, int64_t n, int32_t step, float lr,
                           float beta1, float beta2, float eps, float grad_scale, void* stream) {
  if (!p || !g || !m || !v || n <= 0 || step < 1) {
    set_error("adam_step: invalid argument");
    return NERFB200_ERR_INVALID;
  }
  return launch_adam(p, g, m, v, n, step, lr, beta1, beta2, eps, grad_scale, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
