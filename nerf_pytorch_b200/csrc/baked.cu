// baked.cu -- baked fields (include/nerfb200.h "baked fields"): the directions and the SH projection of a bake (host,
// fp64), and the renderer that marches a ray through the baked bricks without the MLP.
//   renderer  one warp per ray.  Each round the 32 lanes take 32 consecutive samples: the lane forms its point as the
//             MLP forms one, finds its cube and the cube's brick slot, gathers the cube's 8 corner points (128 B each:
//             sigma_raw and 27 SH coefficients) and interpolates them; sample_terms gives alpha and q as the library's
//             compositing forms them.  T is the warp's exclusive product scan of q; rgb, acc and depth are summed in
//             sample order by broadcasting each lane's terms.  A round whose lanes all miss (ballot) adds nothing and
//             skips its gathers.  No atomics, no shared memory.
#include <cmath>

#include "composite.cuh"

namespace nerfb200 {

void bake_basis(BakeBasis* b) {
  const double kPi = 3.14159265358979323846;
  double Y[kBakeDirs][kBakeSh];
  for (int i = 0; i < kBakeDirs; ++i) {
    const double z = 1.0 - (2.0 * i + 1.0) / kBakeDirs, r = std::sqrt(1.0 - z * z);
    const double phi = i * kPi * (3.0 - std::sqrt(5.0));
    const double d[3] = {r * std::cos(phi), r * std::sin(phi), z};
    for (int c = 0; c < 3; ++c) b->dir[i][c] = (float)d[c];
    const double x = b->dir[i][0], y = b->dir[i][1], w = b->dir[i][2];  // the fp32 directions the network sees
    Y[i][0] = 0.28209479177387814;
    Y[i][1] = -0.4886025119029199 * y;
    Y[i][2] = 0.4886025119029199 * w;
    Y[i][3] = -0.4886025119029199 * x;
    Y[i][4] = 1.0925484305920792 * x * y;
    Y[i][5] = -1.0925484305920792 * y * w;
    Y[i][6] = 0.31539156525252005 * (2.0 * w * w - x * x - y * y);
    Y[i][7] = -1.0925484305920792 * x * w;
    Y[i][8] = 0.5462742152960396 * (x * x - y * y);
  }
  // M = (Y^T Y)^-1 Y^T: Gauss-Jordan with partial pivoting on [Y^T Y | Y^T]
  double A[kBakeSh][kBakeSh + kBakeDirs];
  for (int j = 0; j < kBakeSh; ++j) {
    for (int k = 0; k < kBakeSh; ++k) {
      double s = 0.0;
      for (int i = 0; i < kBakeDirs; ++i) s += Y[i][j] * Y[i][k];
      A[j][k] = s;
    }
    for (int i = 0; i < kBakeDirs; ++i) A[j][kBakeSh + i] = Y[i][j];
  }
  for (int c = 0; c < kBakeSh; ++c) {
    int piv = c;
    for (int r = c + 1; r < kBakeSh; ++r)
      if (std::fabs(A[r][c]) > std::fabs(A[piv][c])) piv = r;
    for (int k = 0; k < kBakeSh + kBakeDirs; ++k) std::swap(A[c][k], A[piv][k]);
    const double inv = 1.0 / A[c][c];
    for (int k = 0; k < kBakeSh + kBakeDirs; ++k) A[c][k] *= inv;
    for (int r = 0; r < kBakeSh; ++r) {
      if (r == c) continue;
      const double f = A[r][c];
      for (int k = 0; k < kBakeSh + kBakeDirs; ++k) A[r][k] -= f * A[c][k];
    }
  }
  for (int j = 0; j < kBakeSh; ++j)
    for (int i = 0; i < kBakeDirs; ++i) b->proj[j][i] = (float)A[j][kBakeSh + i];
}

namespace {

constexpr int kBakedWarps = 4;
constexpr int kBakedVals = 1 + 3 * kBakeSh;  // interpolated channels: sigma_raw and the 27 coefficients
static_assert(kBakedVals == 28, "seven float4 per corner point");

struct BakedBox {
  nerfb200_grid_t g;
  int nb[3];      // bricks per axis
  float scale[3]; // the cell rule's res / (hi - lo)
  float h;        // the smallest cube side
};

// the SH basis at a unit direction (fp32, as the header writes it)
__device__ __forceinline__ void sh_basis(float x, float y, float z, float Y[kBakeSh]) {
  Y[0] = 0.28209479177387814f;
  Y[1] = __fmul_rn(-0.4886025119029199f, y);
  Y[2] = __fmul_rn(0.4886025119029199f, z);
  Y[3] = __fmul_rn(-0.4886025119029199f, x);
  Y[4] = __fmul_rn(__fmul_rn(1.0925484305920792f, x), y);
  Y[5] = __fmul_rn(__fmul_rn(-1.0925484305920792f, y), z);
  const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
  Y[6] = __fmul_rn(0.31539156525252005f, __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), xx), yy));
  Y[7] = __fmul_rn(__fmul_rn(-1.0925484305920792f, x), z);
  Y[8] = __fmul_rn(0.5462742152960396f, __fsub_rn(xx, yy));
}

__global__ void __launch_bounds__(kBakedWarps * 32)
baked_render_kernel(const BakedBox B, const int* __restrict__ brick_map, const float* __restrict__ values,
                    int use_viewdirs, const float* __restrict__ rays, int ray_stride, int64_t n_rays, int white_bkgd,
                    float stop_t, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kBakedWarps + (threadIdx.x >> 5);
  if (r >= n_rays) return;
  const float* rr = rays + r * ray_stride;
  float o[3], d[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = rr[c];
    d[c] = rr[3 + c];
  }
  // the interval: [near, far] and the box's slabs.  An axis with d_c = +-0 keeps x_c = o_c at every sample: it does not
  // restrict the interval when lo_c <= o_c < hi_c and empties the ray otherwise (its slab terms would be 0/0 or inf)
  float ta = rr[6], tb = rr[7];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (d[c] == 0.f) {
      if (!(o[c] >= B.g.lo[c] && o[c] < B.g.hi[c])) tb = -INFINITY;
      continue;
    }
    const float t0 = __fdiv_rn(__fsub_rn(B.g.lo[c], o[c]), d[c]), t1 = __fdiv_rn(__fsub_rn(B.g.hi[c], o[c]), d[c]);
    ta = fmaxf(ta, fminf(t0, t1));
    tb = fminf(tb, fmaxf(t0, t1));
  }
  const float dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
  const float dt = __fdiv_rn(__fmul_rn(0.5f, B.h), dnorm);
  float Y[kBakeSh];
  if (use_viewdirs) sh_basis(rr[8], rr[9], rr[10], Y);
  else Y[0] = 0.28209479177387814f;

  float T = 1.0f, ar = 0.f, ag = 0.f, ab = 0.f, aacc = 0.f, adepth = 0.f;
  // dt > 0 and finite, and sample indices exact in fp32: anything else is an empty ray
  const bool live = ta < tb && dt > 0.f && dt < INFINITY && __fdiv_rn(__fsub_rn(tb, ta), dt) < 16777216.f;
  for (int k0 = 0; live; k0 += 32) {
    const float t = __fadd_rn(ta, __fmul_rn(__fadd_rn((float)(k0 + lane), 0.5f), dt));
    if (!(__shfl_sync(0xffffffffu, t, 0) < tb)) break;  // t grows with k: no sample left
    const bool in_ray = t < tb;
    int slot = -1;
    float f[3];
    int l[3];
    if (in_ray) {
      bool inside = true;
      int bi[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float x = __fadd_rn(o[c], __fmul_rn(d[c], t));
        const float tc = __fmul_rn(__fsub_rn(x, B.g.lo[c]), B.scale[c]);
        inside = inside && tc >= 0.f && tc < (float)B.g.res[c];
        const int i = inside ? (int)tc : 0;
        f[c] = __fsub_rn(tc, (float)i);
        bi[c] = i >> 3;
        l[c] = i & 7;
      }
      if (inside) slot = brick_map[((int64_t)bi[2] * B.nb[1] + bi[1]) * B.nb[0] + bi[0]];
    }
    if (__ballot_sync(0xffffffffu, slot >= 0) == 0u) continue;  // q = 1 and w = 0 everywhere: T and the sums stay
    float v[kBakedVals];
#pragma unroll
    for (int ch = 0; ch < kBakedVals; ++ch) v[ch] = 0.f;
    if (slot >= 0) {
      const float4* base = reinterpret_cast<const float4*>(values + (int64_t)slot * kBakePts * kBakeCh);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
        const float wx = dx ? f[0] : __fsub_rn(1.0f, f[0]), wy = dy ? f[1] : __fsub_rn(1.0f, f[1]);
        const float wz = dz ? f[2] : __fsub_rn(1.0f, f[2]);
        const float w = __fmul_rn(__fmul_rn(wx, wy), wz);
        const float4* pv = base + (((l[2] + dz) * 9 + l[1] + dy) * 9 + l[0] + dx) * (kBakeCh / 4);
#pragma unroll
        for (int c4 = 0; c4 < kBakedVals / 4; ++c4) {
          const float4 a = __ldg(pv + c4);
          v[4 * c4] = fmaf(w, a.x, v[4 * c4]);
          v[4 * c4 + 1] = fmaf(w, a.y, v[4 * c4 + 1]);
          v[4 * c4 + 2] = fmaf(w, a.z, v[4 * c4 + 2]);
          v[4 * c4 + 3] = fmaf(w, a.w, v[4 * c4 + 3]);
        }
      }
    }
    float rgb[3] = {0.f, 0.f, 0.f};
    if (slot >= 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float s = 0.f;
        if (use_viewdirs) {
#pragma unroll
          for (int j = 0; j < kBakeSh; ++j) s = fmaf(Y[j], v[1 + kBakeSh * c + j], s);
        } else {
          s = __fmul_rn(Y[0], v[1 + kBakeSh * c]);
        }
        rgb[c] = sigmoidf_(s);
      }
    }
    const SampleTerms st = sample_terms(slot >= 0 ? v[0] : 0.f, 0.f, 0.f, false, t, __fadd_rn(t, dt), false, dnorm);
    const float Tl = __fmul_rn(T, warp_excl_prod(st.q, lane));
    const float w = __fmul_rn(st.alpha, Tl);
    const float cr = __fmul_rn(w, rgb[0]), cg = __fmul_rn(w, rgb[1]), cb = __fmul_rn(w, rgb[2]);
    const float cd = __fmul_rn(w, t);
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {  // in sample order
      ar = __fadd_rn(ar, __shfl_sync(0xffffffffu, cr, i));
      ag = __fadd_rn(ag, __shfl_sync(0xffffffffu, cg, i));
      ab = __fadd_rn(ab, __shfl_sync(0xffffffffu, cb, i));
      aacc = __fadd_rn(aacc, __shfl_sync(0xffffffffu, w, i));
      adepth = __fadd_rn(adepth, __shfl_sync(0xffffffffu, cd, i));
    }
    T = __shfl_sync(0xffffffffu, __fmul_rn(Tl, st.q), 31);
    if (T < stop_t) break;
  }
  if (lane == 0) {
    const float ratio = __fdiv_rn(adepth, aacc);
    const float disp = __fdiv_rn(1.0f, fmaxf(1e-10f, ratio));
    const float disp_out = (ratio != ratio) ? ratio : disp;  // fmaxf drops NaNs; keep it for empty rays
    if (white_bkgd) {
      const float bg = __fsub_rn(1.0f, aacc);
      ar = __fadd_rn(ar, bg);
      ag = __fadd_rn(ag, bg);
      ab = __fadd_rn(ab, bg);
    }
    float4* o4 = reinterpret_cast<float4*>(out + r * 8);
    o4[0] = make_float4(ar, ag, ab, disp_out);
    o4[1] = make_float4(aacc, adepth, 0.f, 0.f);
  }
}

}  // namespace
}  // namespace nerfb200

using namespace nerfb200;

extern "C" {

int32_t nerfb200_bake_basis(float* dirs_host, float* proj_host) {
  if (!dirs_host || !proj_host) {
    set_error("bake_basis: null pointer");
    return NERFB200_ERR_INVALID;
  }
  BakeBasis b;
  bake_basis(&b);
  for (int i = 0; i < kBakeDirs; ++i)
    for (int c = 0; c < 3; ++c) dirs_host[3 * i + c] = b.dir[i][c];
  for (int j = 0; j < kBakeSh; ++j)
    for (int i = 0; i < kBakeDirs; ++i) proj_host[kBakeDirs * j + i] = b.proj[j][i];
  return NERFB200_OK;
}

int32_t nerfb200_baked_render(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                              int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                              int32_t white_background, float stop_transmittance, float* out, void* stream) {
  if (int rc = check_grid(box, "baked_render")) return rc;
  if (!brick_map || !values || !rays || !out || n_rays <= 0 || ray_stride < (use_viewdirs ? 11 : 8)) {
    set_error("baked_render: null pointer, n_rays <= 0 or ray_stride %d too short", ray_stride);
    return NERFB200_ERR_INVALID;
  }
  if (!(stop_transmittance >= 0.f && stop_transmittance < 1.f)) {
    set_error("baked_render: stop_transmittance must lie in [0, 1), got %g", (double)stop_transmittance);
    return NERFB200_ERR_INVALID;
  }
  BakedBox B;
  B.g = *box;
  B.h = INFINITY;
  for (int c = 0; c < 3; ++c) {
    B.nb[c] = (box->res[c] + kBakeBrick - 1) / kBakeBrick;
    B.scale[c] = (float)box->res[c] / (box->hi[c] - box->lo[c]);
    B.h = std::fmin(B.h, (box->hi[c] - box->lo[c]) / (float)box->res[c]);
  }
  const int64_t blocks = (n_rays + kBakedWarps - 1) / kBakedWarps;
  baked_render_kernel<<<(unsigned)blocks, kBakedWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      B, brick_map, values, use_viewdirs ? 1 : 0, rays, ray_stride, n_rays, white_background ? 1 : 0,
      stop_transmittance, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "baked_render launch");
}

}  // extern "C"
