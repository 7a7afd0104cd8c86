// baked.cu -- baked fields (include/nerfb200.h "baked fields"): the directions and the SH projection of a bake (host,
// fp64), and the renderer that marches a ray through the baked bricks without the MLP.
//   renderer  one warp per ray.  Each round the 32 lanes take 32 consecutive samples: the lane forms its point as the
//             MLP forms one, finds its cube and the cube's brick slot, gathers the cube's 8 corner points (128 B each:
//             sigma_raw and 27 SH coefficients) and interpolates them; sample_terms gives alpha and q as the library's
//             compositing forms them.  T is the warp's exclusive product scan of q; rgb, acc and depth are summed in
//             sample order by broadcasting each lane's terms.  A round whose lanes all miss (ballot) adds nothing and
//             skips its gathers.  No atomics, no shared memory.
//   backward  the renderer's warp re-marches the ray through the same helpers and scatters each sample's 28 channel
//             gradients to its cube's 8 corners with vector fp32 reductions (include/nerfb200.h "baked fields: gradients
//             and fine-tuning"); their order is the hardware's, so raw gradients may differ in the last bits between runs.
//   tie       one thread per float4: the sum over every stored copy of the value's lattice point, gathered in one fixed
//             order, so all copies get the same bits.
//   peak      the renderer's warp re-marches the ray interpolating sigma_raw alone and max-accumulates each sample's
//             weight into its brick slot (include/nerfb200.h "baked fields: pruning"): one integer atomicMax per slot
//             per round, so the result is the same bits for every chunking and order.
//   regularisers  one CTA per slot, one thread per stored point (include/nerfb200.h "baked fields: regularisers"):
//             the TV and sparsity gradient from canonical-copy reads, the same bits at every copy, and the slot's fp64
//             value partial reduced in a fixed order.
#include <cmath>

#include <cuda_fp16.h>

#include "composite.cuh"
#include "mesh_rules.cuh"

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

int check_f16_values(const char* what, const void* values) {
  if (reinterpret_cast<uintptr_t>(values) % 16 != 0) {
    set_error("%s: values must be 16-B aligned", what);
    return NERFB200_ERR_INVALID;
  }
  return NERFB200_OK;
}

namespace {

// the check a field's storage format adds to an entry point's own (what: the entry point's name in the error): none
// for fp32; fp16 values and uint8 codes 16-B aligned, as the vector gathers need; and a dequant table for uint8
template <typename V>
int check_values(const char* what, const V* values, const float* dequant) {
  if (sizeof(V) == 4) return NERFB200_OK;
  if (int rc = check_f16_values(what, values)) return rc;
  if (sizeof(V) == 1 && !dequant) {
    set_error("%s: null dequant (a uint8 field needs its [2][28] scales and offsets)", what);
    return NERFB200_ERR_INVALID;
  }
  return NERFB200_OK;
}

// counts the launch entry point what just made and checks it; a failure reads "<what> launch: <CUDA error>"
int check_launch(const char* what) {
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return NERFB200_OK;
  set_error("%s launch: %s", what, cudaGetErrorString(e));
  return NERFB200_ERR_CUDA;
}

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

// a ray's origin, direction and interval: [near, far] and the box's slabs.  An axis with d_c = +-0 keeps x_c = o_c at
// every sample: it does not restrict the interval when lo_c <= o_c < hi_c and empties the ray otherwise (its slab terms
// would be 0/0 or inf)
__device__ __forceinline__ void baked_ray(const BakedBox& B, const float* rr, float o[3], float d[3], float& ta,
                                          float& tb, float& dnorm, float& dt) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = rr[c];
    d[c] = rr[3 + c];
  }
  ta = rr[6];
  tb = rr[7];
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
  dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
  dt = __fdiv_rn(__fmul_rn(0.5f, B.h), dnorm);
}

// dt > 0 and finite, and sample indices exact in fp32: anything else is an empty ray
__device__ __forceinline__ bool baked_live(float ta, float tb, float dt) {
  return ta < tb && dt > 0.f && dt < INFINITY && __fdiv_rn(__fsub_rn(tb, ta), dt) < 16777216.f;
}

// the sample's point x = o + d t, per axis as the MLP forms its points
__device__ __forceinline__ float baked_x(const float o[3], const float d[3], float t, int c) {
  return __fadd_rn(o[c], __fmul_rn(d[c], t));
}

// the point x (in_ray: whether to look it up at all): its cube's fractions f, its point l inside the brick and the
// brick's slot, or -1 outside the box, in an inactive brick or when !in_ray.  point(c) gives x_c
template <typename Point>
__device__ __forceinline__ int baked_locate(const BakedBox& B, const int* __restrict__ brick_map, Point&& point,
                                            bool in_ray, float f[3], int l[3]) {
  int slot = -1;
  if (in_ray) {
    bool inside = true;
    int bi[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x = point(c);
      const float tc = __fmul_rn(__fsub_rn(x, B.g.lo[c]), B.scale[c]);
      inside = inside && tc >= 0.f && tc < (float)B.g.res[c];
      const int i = inside ? (int)tc : 0;
      f[c] = __fsub_rn(tc, (float)i);
      bi[c] = i >> 3;
      l[c] = i & 7;
    }
    if (inside) slot = brick_map[((int64_t)bi[2] * B.nb[1] + bi[1]) * B.nb[0] + bi[0]];
  }
  return slot;
}

// the sample at depth t (in_ray: t < t_b): baked_locate of its point, -1 past t_b
__device__ __forceinline__ int baked_lookup(const BakedBox& B, const int* __restrict__ brick_map, const float o[3],
                                            const float d[3], float t, bool in_ray, float f[3], int l[3]) {
  return baked_locate(B, brick_map, [&](int c) { return baked_x(o, d, t, c); }, in_ray, f, l);
}

// trilinear weight of corner k = 0 .. 7 of a cube with fractions f
__device__ __forceinline__ float corner_weight(const float f[3], int k) {
  const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
  const float wx = dx ? f[0] : __fsub_rn(1.0f, f[0]), wy = dy ? f[1] : __fsub_rn(1.0f, f[1]);
  const float wz = dz ? f[2] : __fsub_rn(1.0f, f[2]);
  return __fmul_rn(__fmul_rn(wx, wy), wz);
}

// corner k's factor in each axis' derivative of the trilinear interp (include/nerfb200.h "baked fields: normal maps and
// point queries"): +-(the product of the other two axes' weights, in axis order), + where the corner's offset is 1
__device__ __forceinline__ void corner_slopes(const float f[3], int k, float s[3]) {
  const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
  const float wx = dx ? f[0] : __fsub_rn(1.0f, f[0]), wy = dy ? f[1] : __fsub_rn(1.0f, f[1]);
  const float wz = dz ? f[2] : __fsub_rn(1.0f, f[2]);
  const float px = __fmul_rn(wy, wz), py = __fmul_rn(wx, wz), pz = __fmul_rn(wx, wy);
  s[0] = dx ? px : -px;
  s[1] = dy ? py : -py;
  s[2] = dz ? pz : -pz;
}

// 16-B offset of corner k of the cube at brick point l, from the slot's first value: a point is kBakeCh values of type V
// (8 vectors of fp32, 4 of fp16, 2 of uint8 codes)
template <typename V>
__device__ __forceinline__ int corner_offset(const int l[3], int k) {
  const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
  return (((l[2] + dz) * 9 + l[1] + dy) * 9 + l[0] + dx) * (kBakeCh * (int)sizeof(V) / 16);
}

// four fp16 values (the bits of two 32-bit words) widened exactly to fp32
__device__ __forceinline__ void widen4(unsigned a, unsigned b, float out[4]) {
  out[0] = __half2float(__ushort_as_half((unsigned short)(a & 0xffffu)));
  out[1] = __half2float(__ushort_as_half((unsigned short)(a >> 16)));
  out[2] = __half2float(__ushort_as_half((unsigned short)(b & 0xffffu)));
  out[3] = __half2float(__ushort_as_half((unsigned short)(b >> 16)));
}

// code q of channel ch dequantised (include/nerfb200.h "baked fields: 8-bit values"): fl(fl(q s_ch) + o_ch), dq the
// [2][28] scales and offsets
__device__ __forceinline__ float dequant(unsigned q, const float* dq, int ch) {
  return __fadd_rn(__fmul_rn((float)q, dq[ch]), dq[kBakedVals + ch]);
}

// a uint8 field's dequant table copied into the CTA's shared memory dq_s; every thread of the CTA must call it before
// any returns.  Nothing for fp32 and fp16 fields
template <typename V>
__device__ __forceinline__ void stage_dequant(const float* __restrict__ dequant_tab, float* dq_s) {
  if constexpr (sizeof(V) == 1) {
    if (threadIdx.x < 2 * kBakedVals) dq_s[threadIdx.x] = __ldg(dequant_tab + threadIdx.x);
    __syncthreads();
  }
}

// one stored value, widened to fp32 (channel 0 dequantised for uint8; dq is read for uint8 only)
__device__ __forceinline__ float baked_ld(const float* p, const float*) { return __ldg(p); }
__device__ __forceinline__ float baked_ld(const __half* p, const float*) {
  return __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short*>(p))));
}
__device__ __forceinline__ float baked_ld(const uint8_t* p, const float* dq) { return dequant(__ldg(p), dq, 0); }

// channels 0 .. 27 of the stored point off16 16-B vectors past base, widened exactly to fp32 and handed to put(ch, x):
// the one reader of a format's layout.  fp32: seven 16-B loads, each vector put before the next load (loading all seven
// first reschedules the fp32 renderer and its backward); fp16: three 16-B loads and one 8-B load (56 of the point's
// 64 B), each value widened exactly; uint8: two 16-B loads (the point's one 32-B sector), each code dequantised with dq
// (read for uint8 only)
template <typename Put>
__device__ __forceinline__ void baked_point(const float* base, int off16, const float*, Put&& put) {
  const float4* p4 = reinterpret_cast<const float4*>(base) + off16;
#pragma unroll
  for (int c4 = 0; c4 < kBakedVals / 4; ++c4) {
    const float4 u = __ldg(p4 + c4);
    put(4 * c4, u.x);
    put(4 * c4 + 1, u.y);
    put(4 * c4 + 2, u.z);
    put(4 * c4 + 3, u.w);
  }
}
template <typename Put>
__device__ __forceinline__ void baked_point(const __half* base, int off16, const float*, Put&& put) {
  const uint4* p4 = reinterpret_cast<const uint4*>(base) + off16;
  float a[kBakedVals];
#pragma unroll
  for (int c8 = 0; c8 < kBakedVals / 8; ++c8) {  // channels 0 .. 23
    const uint4 u = __ldg(p4 + c8);
    widen4(u.x, u.y, a + 8 * c8);
    widen4(u.z, u.w, a + 8 * c8 + 4);
  }
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p4 + kBakedVals / 8));  // channels 24 .. 27
  widen4(u.x, u.y, a + 24);
#pragma unroll
  for (int ch = 0; ch < kBakedVals; ++ch) put(ch, a[ch]);
}
template <typename Put>
__device__ __forceinline__ void baked_point(const uint8_t* base, int off16, const float* dq, Put&& put) {
  const uint4* p4 = reinterpret_cast<const uint4*>(base) + off16;
  const uint4 u0 = __ldg(p4), u1 = __ldg(p4 + 1);  // channels 28 .. 31 (u1.w) are not read
  const unsigned w[kBakedVals / 4] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z};
  float a[kBakedVals];
#pragma unroll
  for (int ch = 0; ch < kBakedVals; ++ch) a[ch] = dequant((w[ch >> 2] >> (8 * (ch & 3))) & 0xffu, dq, ch);
#pragma unroll
  for (int ch = 0; ch < kBakedVals; ++ch) put(ch, a[ch]);
}

// channels 0 .. 27 interpolated over the cube's corners (0 when slot < 0): each corner's point from baked_point into
// the same fmaf chain for every format.  sigma(k, x) also receives corner k's sigma_raw as it is fed to channel 0
template <typename V, typename Sigma>
__device__ __forceinline__ void baked_interp(const V* __restrict__ values, const float* dq, int slot, const float f[3],
                                             const int l[3], float v[kBakedVals], Sigma&& sigma) {
#pragma unroll
  for (int ch = 0; ch < kBakedVals; ++ch) v[ch] = 0.f;
  if (slot >= 0) {
    const V* sv = values + (int64_t)slot * kBakePts * kBakeCh;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float w = corner_weight(f, k);
      baked_point(sv, corner_offset<V>(l, k), dq, [&](int ch, float x) {
        v[ch] = fmaf(w, x, v[ch]);
        if (ch == 0) sigma(k, x);
      });
    }
  }
}
template <typename V>
__device__ __forceinline__ void baked_interp(const V* __restrict__ values, const float* dq, int slot, const float f[3],
                                             const int l[3], float v[kBakedVals]) {
  baked_interp(values, dq, slot, f, l, v, [](int, float) {});
}

// the gradient of the trilinear sigma_raw inside a cube with fractions f (include/nerfb200.h "baked fields: normal maps
// and point queries"): add(f, k, v_k) takes the corners in the renderer's order, then scale(B) multiplies each axis'
// sum by the cell rule's scale
struct SigmaGrad {
  float g[3] = {0.f, 0.f, 0.f};
  __device__ __forceinline__ void add(const float f[3], int k, float vk) {
    float s[3];
    corner_slopes(f, k, s);
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = fmaf(s[c], vk, g[c]);
  }
  __device__ __forceinline__ void scale(const BakedBox& B) {
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = __fmul_rn(g[c], B.scale[c]);
  }
};

// channel 0 (sigma_raw) of baked_interp: the same corners in the same order through the same fmaf chain, one 4-B (fp32),
// 2-B (fp16) or 1-B (uint8) load per corner
template <typename V>
__device__ __forceinline__ float baked_interp_sigma(const V* __restrict__ values, const float* dq, int slot,
                                                    const float f[3], const int l[3]) {
  float v = 0.f;
  if (slot >= 0) {
    const V* base = values + (int64_t)slot * kBakePts * kBakeCh;
#pragma unroll
    for (int k = 0; k < 8; ++k)
      v = fmaf(corner_weight(f, k), baked_ld(base + (16 / (int)sizeof(V)) * corner_offset<V>(l, k), dq), v);
  }
  return v;
}

// the pre-sigmoid logit s_c of colour channel c from the interpolated coefficients v[1 ..]
__device__ __forceinline__ float baked_logit(int use_viewdirs, const float Y[kBakeSh], const float v[kBakedVals], int c) {
  float s = 0.f;
  if (use_viewdirs) {
#pragma unroll
    for (int j = 0; j < kBakeSh; ++j) s = fmaf(Y[j], v[1 + kBakeSh * c + j], s);
  } else {
    s = __fmul_rn(Y[0], v[1 + kBakeSh * c]);
  }
  return s;
}

// rgb = sigmoid(s_c) of the interpolated coefficients v[1 ..]
__device__ __forceinline__ void baked_colour(int use_viewdirs, const float Y[kBakeSh], const float v[kBakedVals],
                                             float rgb[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) rgb[c] = sigmoidf_(baked_logit(use_viewdirs, Y, v, c));
}

// w n of a sample (include/nerfb200.h "baked fields: normal maps and point queries"): n = -g / |g|, 0 where |g| is 0,
// and 0 for w == 0 (a NaN gradient stays out of rays that never reach it)
__device__ __forceinline__ void weighted_normal(float w, const float g[3], float out[3]) {
  out[0] = out[1] = out[2] = 0.f;
  const float ss = __fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2]));
  if (w != 0.f && ss != 0.f) {
    const float len = __fsqrt_rn(ss);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = __fmul_rn(w, -__fdiv_rn(g[c], len));
  }
}

// kNormals also sums each sample's w n into normals[r][3] (include/nerfb200.h "baked fields: normal maps and point
// queries"), the gradient taken from the sigma_raw corners the interp already reads; kNdc maps each gradient by J^T of
// ndc at the sample's point first.  The instances without normals never read normals or ndc.
template <typename V, bool kNormals = false, bool kNdc = false>
__global__ void __launch_bounds__(kBakedWarps * 32)
baked_render_kernel(const BakedBox B, const int* __restrict__ brick_map, const V* __restrict__ values,
                    int use_viewdirs, const float* __restrict__ rays, int ray_stride, int64_t n_rays, int white_bkgd,
                    float stop_t, float* __restrict__ out, const float* __restrict__ dequant_tab,
                    float* __restrict__ normals, const NdcMap ndc) {
  __shared__ float dq[sizeof(V) == 1 ? 2 * kBakedVals : 1];  // uint8 fields only
  stage_dequant<V>(dequant_tab, dq);
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kBakedWarps + (threadIdx.x >> 5);
  if (r >= n_rays) return;
  const float* rr = rays + r * ray_stride;
  float o[3], d[3], ta, tb, dnorm, dt;
  baked_ray(B, rr, o, d, ta, tb, dnorm, dt);
  float Y[kBakeSh];
  if (use_viewdirs) sh_basis(rr[8], rr[9], rr[10], Y);
  else Y[0] = 0.28209479177387814f;

  float T = 1.0f, ar = 0.f, ag = 0.f, ab = 0.f, aacc = 0.f, adepth = 0.f;
  float N[3] = {0.f, 0.f, 0.f};  // kNormals
  const bool live = baked_live(ta, tb, dt);
  for (int k0 = 0; live; k0 += 32) {
    const float t = __fadd_rn(ta, __fmul_rn(__fadd_rn((float)(k0 + lane), 0.5f), dt));
    if (!(__shfl_sync(0xffffffffu, t, 0) < tb)) break;  // t grows with k: no sample left
    float f[3];
    int l[3];
    const int slot = baked_lookup(B, brick_map, o, d, t, t < tb, f, l);
    if (__ballot_sync(0xffffffffu, slot >= 0) == 0u) continue;  // q = 1 and w = 0 everywhere: T and the sums stay
    float v[kBakedVals];
    SigmaGrad sg;
    if constexpr (kNormals) baked_interp(values, dq, slot, f, l, v, [&](int k, float x) { sg.add(f, k, x); });
    else baked_interp(values, dq, slot, f, l, v);
    float rgb[3] = {0.f, 0.f, 0.f};
    if (slot >= 0) baked_colour(use_viewdirs, Y, v, rgb);
    const SampleTerms st = sample_terms(slot >= 0 ? v[0] : 0.f, 0.f, 0.f, false, t, __fadd_rn(t, dt), false, dnorm);
    const float Tl = __fmul_rn(T, warp_excl_prod(st.q, lane));
    const float w = __fmul_rn(st.alpha, Tl);
    const float cr = __fmul_rn(w, rgb[0]), cg = __fmul_rn(w, rgb[1]), cb = __fmul_rn(w, rgb[2]);
    const float cd = __fmul_rn(w, t);
    float cn[3];  // kNormals: w n
    if constexpr (kNormals) {
      sg.scale(B);
      if constexpr (kNdc) {
        const float x[3] = {baked_x(o, d, t, 0), baked_x(o, d, t, 1), baked_x(o, d, t, 2)};
        const float gn[3] = {sg.g[0], sg.g[1], sg.g[2]};
        ndc_grad_to_world(ndc, x, gn, sg.g);
      }
      weighted_normal(w, sg.g, cn);
    }
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {  // in sample order
      ar = __fadd_rn(ar, __shfl_sync(0xffffffffu, cr, i));
      ag = __fadd_rn(ag, __shfl_sync(0xffffffffu, cg, i));
      ab = __fadd_rn(ab, __shfl_sync(0xffffffffu, cb, i));
      aacc = __fadd_rn(aacc, __shfl_sync(0xffffffffu, w, i));
      adepth = __fadd_rn(adepth, __shfl_sync(0xffffffffu, cd, i));
      if constexpr (kNormals) {
#pragma unroll
        for (int c = 0; c < 3; ++c) N[c] = __fadd_rn(N[c], __shfl_sync(0xffffffffu, cn[c], i));
      }
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
    if constexpr (kNormals) {
#pragma unroll
      for (int c = 0; c < 3; ++c) normals[r * 3 + c] = N[c];
    }
  }
}

constexpr int kQueryThreads = 256;

// One thread per point (include/nerfb200.h "baked fields: normal maps and point queries"): the renderer's lookup, interp
// and logits at pts[i], raw[i] = (s_r, s_g, s_b, sigma_raw) (0 outside the box or in an inactive brick) and grad[i] the
// gradient of sigma_raw; either output may be null.  dirs[i] is read with view directions only, as given.
template <typename V>
__global__ void __launch_bounds__(kQueryThreads)
baked_query_kernel(const BakedBox B, const int* __restrict__ brick_map, const V* __restrict__ values, int use_viewdirs,
                   const float* __restrict__ pts, const float* __restrict__ dirs, int64_t n, float* __restrict__ raw,
                   float* __restrict__ grad, const float* __restrict__ dequant_tab) {
  __shared__ float dq[sizeof(V) == 1 ? 2 * kBakedVals : 1];  // uint8 fields only
  stage_dequant<V>(dequant_tab, dq);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
  float f[3];
  int l[3];
  const int slot = baked_locate(B, brick_map, [&](int c) { return x[c]; }, true, f, l);
  float v[kBakedVals];
  SigmaGrad sg;
  baked_interp(values, dq, slot, f, l, v, [&](int k, float s) { sg.add(f, k, s); });
  sg.scale(B);
  if (raw) {
    float s[3] = {0.f, 0.f, 0.f};
    if (slot >= 0) {
      float Y[kBakeSh];
      if (use_viewdirs) sh_basis(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2], Y);
      else Y[0] = 0.28209479177387814f;
#pragma unroll
      for (int c = 0; c < 3; ++c) s[c] = baked_logit(use_viewdirs, Y, v, c);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) raw[4 * i + c] = s[c];
    raw[4 * i + 3] = v[0];
  }
  if (grad) {
#pragma unroll
    for (int c = 0; c < 3; ++c) grad[3 * i + c] = sg.g[c];
  }
}

// The gradient of baked_render_kernel (stop_transmittance 0) with respect to the values, added into d_values.  The warp
// re-marches the ray as the forward does; per sample v = g_rgb . c + G_acc + G_depth t, dL/dalpha = T v - S / q with
// S = E - (inclusive prefix of w v in sample order) and E = sum w v formed from the forward's totals; the 28 channel
// gradients go to the cube's 8 corners with vector reductions (seven float4 per corner).
__global__ void __launch_bounds__(kBakedWarps * 32)
baked_render_bwd_kernel(const BakedBox B, const int* __restrict__ brick_map, const float* __restrict__ values,
                        int use_viewdirs, const float* __restrict__ rays, int ray_stride, int64_t n_rays, int white_bkgd,
                        const float* __restrict__ out, const float* __restrict__ g_out, float* __restrict__ d_values) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kBakedWarps + (threadIdx.x >> 5);
  if (r >= n_rays) return;
  const float* rr = rays + r * ray_stride;
  float o[3], d[3], ta, tb, dnorm, dt;
  baked_ray(B, rr, o, d, ta, tb, dnorm, dt);
  if (!baked_live(ta, tb, dt)) return;  // no sample: nothing to add
  float Y[kBakeSh];
#pragma unroll
  for (int j = 0; j < kBakeSh; ++j) Y[j] = 0.f;  // without view directions only coefficient 0 is read
  if (use_viewdirs) sh_basis(rr[8], rr[9], rr[10], Y);
  else Y[0] = 0.28209479177387814f;

  const float4 o0 = reinterpret_cast<const float4*>(out + r * 8)[0], o1 = reinterpret_cast<const float4*>(out + r * 8)[1];
  const float4 g0 = reinterpret_cast<const float4*>(g_out + r * 8)[0];
  const float4 g1 = reinterpret_cast<const float4*>(g_out + r * 8)[1];
  const float aacc = o1.x, adepth = o1.y;
  float G_acc = g1.x, G_depth = g1.y;
  composite_upstream(g0, white_bkgd, adepth, aacc, G_acc, G_depth);
  // E = sum_i w_i v_i = g_rgb . rgb + G_acc acc + G_depth depth, rgb without the white background
  float er = o0.x, eg = o0.y, eb = o0.z;
  if (white_bkgd) {
    const float bg = __fsub_rn(1.0f, aacc);
    er = __fsub_rn(er, bg);
    eg = __fsub_rn(eg, bg);
    eb = __fsub_rn(eb, bg);
  }
  const float E = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(g0.x, er), __fmul_rn(g0.y, eg)), __fmul_rn(g0.z, eb)),
                                      __fmul_rn(G_acc, aacc)), __fmul_rn(G_depth, adepth));

  float T = 1.0f, prefix = 0.f;
  for (int k0 = 0;; k0 += 32) {
    const float t = __fadd_rn(ta, __fmul_rn(__fadd_rn((float)(k0 + lane), 0.5f), dt));
    if (!(__shfl_sync(0xffffffffu, t, 0) < tb)) break;
    float f[3];
    int l[3];
    const int slot = baked_lookup(B, brick_map, o, d, t, t < tb, f, l);
    if (__ballot_sync(0xffffffffu, slot >= 0) == 0u) continue;  // as the forward: T and the prefix stay
    float v[kBakedVals];
    baked_interp(values, nullptr, slot, f, l, v);
    float rgb[3] = {0.f, 0.f, 0.f};
    if (slot >= 0) baked_colour(use_viewdirs, Y, v, rgb);
    const SampleTerms st = sample_terms(slot >= 0 ? v[0] : 0.f, 0.f, 0.f, false, t, __fadd_rn(t, dt), false, dnorm);
    const float Tl = __fmul_rn(T, warp_excl_prod(st.q, lane));
    const float w = __fmul_rn(st.alpha, Tl);
    const float vi = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(g0.x, rgb[0]), __fmul_rn(g0.y, rgb[1])),
                                                   __fmul_rn(g0.z, rgb[2])), G_acc), __fmul_rn(G_depth, t));
    const float wv = __fmul_rn(w, vi);
    float incl = 0.f;
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {  // in sample order
      prefix = __fadd_rn(prefix, __shfl_sync(0xffffffffu, wv, i));
      if (i == lane) incl = prefix;
    }
    T = __shfl_sync(0xffffffffu, __fmul_rn(Tl, st.q), 31);
    if (slot < 0 || (!st.gate && w == 0.f)) continue;  // adds nothing
    const float dalpha = __fsub_rn(__fmul_rn(Tl, vi), __fdiv_rn(__fsub_rn(E, incl), st.q));
    const float dsigma = st.gate ? __fmul_rn(__fmul_rn(dalpha, st.delta), st.sigma_delta_exp) : 0.f;
    float ds[3];
    const float gc[3] = {g0.x, g0.y, g0.z};
#pragma unroll
    for (int c = 0; c < 3; ++c)
      ds[c] = __fmul_rn(__fmul_rn(__fmul_rn(w, gc[c]), rgb[c]), __fsub_rn(1.0f, rgb[c]));
    float4* base = reinterpret_cast<float4*>(d_values + (int64_t)slot * kBakePts * kBakeCh);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float wk = corner_weight(f, k);
      float4* pv = base + corner_offset<float>(l, k);
      float gk[kBakedVals];
      gk[0] = __fmul_rn(wk, dsigma);
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < kBakeSh; ++j) gk[1 + kBakeSh * c + j] = __fmul_rn(wk, __fmul_rn(ds[c], Y[j]));
#pragma unroll
      for (int c4 = 0; c4 < kBakedVals / 4; ++c4)
        atomicAdd(pv + c4, make_float4(gk[4 * c4], gk[4 * c4 + 1], gk[4 * c4 + 2], gk[4 * c4 + 3]));
    }
  }
}

// max_w[slot] = max over the ray's samples in the slot of w = alpha T, the renderer's bits (stop_transmittance 0), a NaN
// w as +inf.  The warp re-marches the ray as baked_render_kernel does, interpolating sigma_raw alone; per round the lanes
// with w > 0 are grouped by slot and one lane per group issues an integer atomicMax of the group's largest bits
// (non-negative floats order as unsigned integers).  No stop at T = 0: a NaN later in the ray must still be recorded.
template <typename V>
__global__ void __launch_bounds__(kBakedWarps * 32)
baked_max_weight_kernel(const BakedBox B, const int* __restrict__ brick_map, const V* __restrict__ values,
                        const float* __restrict__ rays, int ray_stride, int64_t n_rays, unsigned* __restrict__ max_w,
                        const float* __restrict__ dequant_tab) {
  __shared__ float dq[sizeof(V) == 1 ? 2 * kBakedVals : 1];  // uint8 fields only
  stage_dequant<V>(dequant_tab, dq);
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kBakedWarps + (threadIdx.x >> 5);
  if (r >= n_rays) return;
  const float* rr = rays + r * ray_stride;
  float o[3], d[3], ta, tb, dnorm, dt;
  baked_ray(B, rr, o, d, ta, tb, dnorm, dt);
  if (!baked_live(ta, tb, dt)) return;  // no sample
  float T = 1.0f;
  for (int k0 = 0;; k0 += 32) {
    const float t = __fadd_rn(ta, __fmul_rn(__fadd_rn((float)(k0 + lane), 0.5f), dt));
    if (!(__shfl_sync(0xffffffffu, t, 0) < tb)) break;
    float f[3];
    int l[3];
    const int slot = baked_lookup(B, brick_map, o, d, t, t < tb, f, l);
    if (__ballot_sync(0xffffffffu, slot >= 0) == 0u) continue;  // as the renderer: T stays
    const float s = baked_interp_sigma(values, dq, slot, f, l);
    const SampleTerms st = sample_terms(slot >= 0 ? s : 0.f, 0.f, 0.f, false, t, __fadd_rn(t, dt), false, dnorm);
    const float Tl = __fmul_rn(T, warp_excl_prod(st.q, lane));
    const float w = __fmul_rn(st.alpha, Tl);
    T = __shfl_sync(0xffffffffu, __fmul_rn(Tl, st.q), 31);
    const bool rec = slot >= 0 && w != 0.f;  // w is >= 0 or NaN; max_w starts at 0
    const unsigned bits = w != w ? __float_as_uint(INFINITY) : __float_as_uint(w);
    const unsigned group = __match_any_sync(0xffffffffu, rec ? slot : -1);
    const unsigned top = __reduce_max_sync(group, rec ? bits : 0u);
    if (rec && lane == __ffs(group) - 1) atomicMax(max_w + slot, top);
  }
}

// the copies of lattice index q along one axis (res cubes, nb bricks): (brick, point) pairs in ascending brick order.
// q < res: (q / 8 - 1, 8) when q is a positive multiple of 8, then (q / 8, q % 8); q = res: (nb - 1, l) for l =
// res - 8 (nb - 1) .. 8 (the upper face's point and its clamped repeats)
struct AxisCopies {
  int n, b0, l0;  // n copies; entry e is (b0, l0 + e) on the upper face, else (b0 + e, l0 - 8 e)
  bool face;
};

__device__ __forceinline__ AxisCopies axis_copies(int q, int res, int nb) {
  if (q == res) return AxisCopies{8 - (res - kBakeBrick * (nb - 1)) + 1, nb - 1, res - kBakeBrick * (nb - 1), true};
  if (q > 0 && (q & 7) == 0) return AxisCopies{2, (q >> 3) - 1, kBakeBrick, false};
  return AxisCopies{1, q >> 3, q & 7, false};
}

__device__ __forceinline__ void axis_entry(const AxisCopies& a, int e, int& b, int& l) {
  b = a.face ? a.b0 : a.b0 + e;
  l = a.face ? a.l0 + e : a.l0 - kBakeBrick * e;
}

// d_tied[copy] = the sum over every stored copy of the copy's lattice point of d_values, in one fixed order (z copies
// outer, then y, then x, each ascending), so every copy of a point gets the same bits.  One thread per float4.
__global__ void baked_tie_kernel(const BakedBox B, const int* __restrict__ brick_map, const int* __restrict__ bricks,
                                 int64_t n_active, const float4* __restrict__ d_values, float4* __restrict__ d_tied) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n_active * kBakePts * (kBakeCh / 4)) return;
  const int c4 = (int)(e & 7);
  if (c4 >= kBakedVals / 4) {  // channels 28 .. 31
    d_tied[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const int64_t sp = e >> 3;
  const int64_t slot = sp / kBakePts;
  const int p = (int)(sp - slot * kBakePts);
  const int brick = bricks[slot];
  const int bc[3] = {brick % B.nb[0], (brick / B.nb[0]) % B.nb[1], brick / (B.nb[0] * B.nb[1])};
  const int lc[3] = {p % 9, (p / 9) % 9, p / 81};
  AxisCopies a[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) a[c] = axis_copies(min(bc[c] * kBakeBrick + lc[c], B.g.res[c]), B.g.res[c], B.nb[c]);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int ez = 0; ez < a[2].n; ++ez) {
    int bz, lz;
    axis_entry(a[2], ez, bz, lz);
    for (int ey = 0; ey < a[1].n; ++ey) {
      int by, ly;
      axis_entry(a[1], ey, by, ly);
      for (int ex = 0; ex < a[0].n; ++ex) {
        int bx, lx;
        axis_entry(a[0], ex, bx, lx);
        const int cs = brick_map[((int64_t)bz * B.nb[1] + by) * B.nb[0] + bx];
        if (cs < 0) continue;
        const float4 g = d_values[((int64_t)cs * kBakePts + (lz * 9 + ly) * 9 + lx) * (kBakeCh / 4) + c4];
        s.x = __fadd_rn(s.x, g.x);
        s.y = __fadd_rn(s.y, g.y);
        s.z = __fadd_rn(s.z, g.z);
        s.w = __fadd_rn(s.w, g.w);
      }
    }
  }
  d_tied[e] = s;
}

// the canonical copy of lattice point q (include/nerfb200.h "baked fields: regularisers"): the float offset of its first
// stored copy in the tie's order whose brick is active, or -1 when no active brick holds q
__device__ __forceinline__ int64_t canonical_copy(const BakedBox& B, const int* __restrict__ brick_map, const int q[3]) {
  AxisCopies a[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) a[c] = axis_copies(q[c], B.g.res[c], B.nb[c]);
  for (int ez = 0; ez < a[2].n; ++ez) {
    int bz, lz;
    axis_entry(a[2], ez, bz, lz);
    for (int ey = 0; ey < a[1].n; ++ey) {
      int by, ly;
      axis_entry(a[1], ey, by, ly);
      for (int ex = 0; ex < a[0].n; ++ex) {
        int bx, lx;
        axis_entry(a[0], ex, bx, lx);
        const int cs = brick_map[((int64_t)bz * B.nb[1] + by) * B.nb[0] + bx];
        if (cs >= 0) return ((int64_t)cs * kBakePts + (lz * 9 + ly) * 9 + lx) * kBakeCh;
      }
    }
  }
  return -1;
}

// whether (q, q + e_c) is an edge: q_c < res_c and an active brick holds both points, brick q_c / 8 along c and any
// brick of q's copy list along the other two axes (at most two distinct bricks each)
__device__ __forceinline__ bool lattice_edge(const BakedBox& B, const int* __restrict__ brick_map, const int q[3], int c) {
  int lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {  // a == c compared, not q[c] indexed: the arrays stay in registers
    if (a == c) {
      if (q[a] >= B.g.res[a]) return false;
      lo[a] = hi[a] = q[a] >> 3;
    } else {
      const AxisCopies ac = axis_copies(q[a], B.g.res[a], B.nb[a]);
      lo[a] = ac.b0;
      hi[a] = ac.face ? ac.b0 : ac.b0 + ac.n - 1;
    }
  }
  for (int bz = lo[2]; bz <= hi[2]; ++bz)
    for (int by = lo[1]; by <= hi[1]; ++by)
      for (int bx = lo[0]; bx <= hi[0]; ++bx)
        if (brick_map[((int64_t)bz * B.nb[1] + by) * B.nb[0] + bx] >= 0) return true;
  return false;
}

// the lattice point a stored point holds: b B + l clamped onto 0 .. res
__device__ __forceinline__ void stored_point(const BakedBox& B, int brick, int p, int q[3]) {
  const int bc[3] = {brick % B.nb[0], (brick / B.nb[0]) % B.nb[1], brick / (B.nb[0] * B.nb[1])};
  const int lc[3] = {p % 9, (p / 9) % 9, p / 81};
#pragma unroll
  for (int c = 0; c < 3; ++c) q[c] = min(bc[c] * kBakeBrick + lc[c], B.g.res[c]);
}

constexpr int kRegThreads = 256;

// *count = P, the lattice points with a copy in an active brick: the stored points that are their point's canonical
// copy, one warp ballot and one integer atomic per warp (*count zeroed first).  One thread per stored point.
__global__ void __launch_bounds__(kRegThreads)
baked_count_kernel(const BakedBox B, const int* __restrict__ brick_map, const int* __restrict__ bricks,
                   int64_t n_active, unsigned long long* __restrict__ count) {
  const int64_t sp = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  bool canon = false;
  if (sp < n_active * kBakePts) {
    const int64_t slot = sp / kBakePts;
    const int p = (int)(sp - slot * kBakePts);
    int q[3];
    stored_point(B, bricks[slot], p, q);
    canon = canonical_copy(B, brick_map, q) == sp * kBakeCh;
  }
  const unsigned votes = __ballot_sync(0xffffffffu, canon);
  if ((threadIdx.x & 31) == 0 && votes) atomicAdd(count, (unsigned long long)__popc(votes));
}

// The regularisers' gradient and value (include/nerfb200.h "baked fields: regularisers").  One CTA per slot, one thread
// per stored point (the CTA strides over the slot's 729): every value is read at its point's canonical copy; S_ch sums
// v_p - v_n over the point's edges in the order -x, +x, -y, +y, -z, +z, g_ch = a_ch S_ch (plus the Cauchy term on
// channel 0) is added into d at the thread's own copy.  A thread whose copy is canonical adds its +x / +y / +z edges'
// squares and its sparsity term to an fp64 sum, reduced over the CTA in a fixed order into partials[slot].
__global__ void __launch_bounds__(kRegThreads)
baked_reg_kernel(const BakedBox B, const int* __restrict__ brick_map, const int* __restrict__ bricks,
                 const float* __restrict__ values, const long long* __restrict__ count, double tv_sigma, double tv_sh,
                 double sparsity, float* __restrict__ d, double* __restrict__ partials) {
  const int64_t slot = blockIdx.x;
  const double P = (double)*count;
  const float a_sigma = (float)(2.0 * tv_sigma / P), a_sh = (float)(2.0 * tv_sh / P);
  const float a_sparse = (float)(4.0 * sparsity / P);
  const int brick = bricks[slot];
  double acc = 0.0;
  for (int p = threadIdx.x; p < kBakePts; p += kRegThreads) {
    const int64_t own = (slot * kBakePts + p) * kBakeCh;
    int q[3];
    stored_point(B, brick, p, q);
    const int64_t cp = canonical_copy(B, brick_map, q);  // >= 0: the thread's own brick is active
    const bool canon = cp == own;
    const float4* vp4 = reinterpret_cast<const float4*>(values + cp);
    float vp[kBakedVals], S[kBakedVals];
#pragma unroll
    for (int c4 = 0; c4 < kBakedVals / 4; ++c4) {
      const float4 a = __ldg(vp4 + c4);
      vp[4 * c4] = a.x;
      vp[4 * c4 + 1] = a.y;
      vp[4 * c4 + 2] = a.z;
      vp[4 * c4 + 3] = a.w;
    }
#pragma unroll
    for (int ch = 0; ch < kBakedVals; ++ch) S[ch] = 0.f;
    double tvs = 0.0, tvh = 0.0;
#pragma unroll 1
    for (int k = 0; k < 6; ++k) {  // -x, +x, -y, +y, -z, +z
      const int c = k >> 1;
      const bool up = k & 1;
      int lo[3], qn[3];  // the edge's lower point and the neighbour
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        lo[a] = a == c && !up ? q[a] - 1 : q[a];
        qn[a] = a == c ? (up ? q[a] + 1 : q[a] - 1) : q[a];
      }
      if ((lo[0] | lo[1] | lo[2]) < 0 || !lattice_edge(B, brick_map, lo, c)) continue;
      const float4* vn4 = reinterpret_cast<const float4*>(values + canonical_copy(B, brick_map, qn));
#pragma unroll
      for (int c4 = 0; c4 < kBakedVals / 4; ++c4) {
        const float4 a = __ldg(vn4 + c4);
        const float n[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ch = 4 * c4 + j;
          S[ch] = __fadd_rn(S[ch], __fsub_rn(vp[ch], n[j]));
          if (up && canon) {
            const double e = (double)vp[ch] - (double)n[j];
            if (ch == 0) tvs += e * e;
            else tvh += e * e;
          }
        }
      }
    }
    const float sp = fmaxf(vp[0], 0.f);
    if (canon) {
      const double s = sp;
      acc += tv_sigma * tvs + tv_sh * tvh + sparsity * log1p(2.0 * s * s);
    }
    if (d) {
      float4* d4 = reinterpret_cast<float4*>(d + own);
#pragma unroll
      for (int c4 = 0; c4 < kBakedVals / 4; ++c4) {
        float g[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ch = 4 * c4 + j;
          g[j] = __fmul_rn(ch == 0 ? a_sigma : a_sh, S[ch]);
        }
        if (c4 == 0)
          g[0] = __fadd_rn(g[0], __fdiv_rn(__fmul_rn(a_sparse, sp), __fadd_rn(1.0f, __fmul_rn(2.0f, __fmul_rn(sp, sp)))));
        float4 o = d4[c4];
        o.x = __fadd_rn(o.x, g[0]);
        o.y = __fadd_rn(o.y, g[1]);
        o.z = __fadd_rn(o.z, g[2]);
        o.w = __fadd_rn(o.w, g[3]);
        d4[c4] = o;
      }
    }
  }
  if (!partials) return;
  // the CTA's sum in a fixed order: each warp by a shuffle tree, then warp 0 over the warps' sums
  __shared__ double warp_sum[kRegThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kRegThreads / 32; ++w) s += warp_sum[w];
    partials[slot] = s / P;
  }
}

BakedBox baked_box(const nerfb200_grid_t* box) {
  BakedBox B;
  B.g = *box;
  B.h = INFINITY;
  for (int c = 0; c < 3; ++c) {
    B.nb[c] = (box->res[c] + kBakeBrick - 1) / kBakeBrick;
    B.scale[c] = (float)box->res[c] / (box->hi[c] - box->lo[c]);
    B.h = std::fmin(B.h, (box->hi[c] - box->lo[c]) / (float)box->res[c]);
  }
  return B;
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

}  // extern "C"

namespace {

// the renderer's checks (what: the entry point's name in the errors), then the format's
template <typename V>
int check_baked_render(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const V* values,
                       int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                       float stop_transmittance, const float* out, const float* dequant) {
  if (int rc = check_grid(box, what)) return rc;
  if (!brick_map || !values || !rays || !out || n_rays <= 0 || ray_stride < (use_viewdirs ? 11 : 8)) {
    set_error("%s: null pointer, n_rays <= 0 or ray_stride %d too short", what, ray_stride);
    return NERFB200_ERR_INVALID;
  }
  if (!(stop_transmittance >= 0.f && stop_transmittance < 1.f)) {
    set_error("%s: stop_transmittance must lie in [0, 1), got %g", what, (double)stop_transmittance);
    return NERFB200_ERR_INVALID;
  }
  return check_values(what, values, dequant);
}

// the renderer's entry points: its checks, then the launch
template <typename V>
int baked_render(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const V* values,
                 int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays, int32_t white_background,
                 float stop_transmittance, float* out, void* stream, const float* dequant) {
  if (int rc = check_baked_render(what, box, brick_map, values, use_viewdirs, rays, ray_stride, n_rays,
                                  stop_transmittance, out, dequant))
    return rc;
  const BakedBox B = baked_box(box);
  const int64_t blocks = (n_rays + kBakedWarps - 1) / kBakedWarps;
  baked_render_kernel<V><<<(unsigned)blocks, kBakedWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      B, brick_map, values, use_viewdirs ? 1 : 0, rays, ray_stride, n_rays, white_background ? 1 : 0,
      stop_transmittance, out, dequant, nullptr, NdcMap{0.f, 0.f});
  return check_launch(what);
}

// the normal-map renderer's entry points: the renderer's checks, a null normals, a camera make_ndc_map refuses (ndc
// NULL: the field's frame), then the launch
template <typename V>
int baked_render_normals(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const V* values,
                         int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                         int32_t white_background, float stop_transmittance, const nerfb200_ndc_t* ndc, float* out,
                         float* normals, void* stream, const float* dequant) {
  if (int rc = check_baked_render(what, box, brick_map, values, use_viewdirs, rays, ray_stride, n_rays,
                                  stop_transmittance, out, dequant))
    return rc;
  if (!normals) {
    set_error("%s: null normals", what);
    return NERFB200_ERR_INVALID;
  }
  NdcMap m{0.f, 0.f};
  if (ndc)
    if (int rc = make_ndc_map(ndc, &m, what)) return rc;
  const BakedBox B = baked_box(box);
  const unsigned blocks = (unsigned)((n_rays + kBakedWarps - 1) / kBakedWarps);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int vd = use_viewdirs ? 1 : 0, white = white_background ? 1 : 0;
  if (ndc)
    baked_render_kernel<V, true, true><<<blocks, kBakedWarps * 32, 0, s>>>(
        B, brick_map, values, vd, rays, ray_stride, n_rays, white, stop_transmittance, out, dequant, normals, m);
  else
    baked_render_kernel<V, true, false><<<blocks, kBakedWarps * 32, 0, s>>>(
        B, brick_map, values, vd, rays, ray_stride, n_rays, white, stop_transmittance, out, dequant, normals, m);
  return check_launch(what);
}

// the point queries' entry points: the box, null pointers, n_points < 0, raw and grad both null, view directions
// without dirs, the format's checks; n_points 0 launches nothing
template <typename V>
int baked_query(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const V* values,
                int32_t use_viewdirs, const float* pts, const float* dirs, int64_t n_points, float* raw, float* grad,
                void* stream, const float* dequant) {
  if (int rc = check_grid(box, what)) return rc;
  if (!brick_map || !values || !pts || n_points < 0 || (!raw && !grad)) {
    set_error("%s: null pointer, raw and grad both null, or n_points %lld < 0", what, (long long)n_points);
    return NERFB200_ERR_INVALID;
  }
  if (use_viewdirs && raw && !dirs) {
    set_error("%s: view directions need dirs", what);
    return NERFB200_ERR_INVALID;
  }
  if (int rc = check_values(what, values, dequant)) return rc;
  if (n_points == 0) return NERFB200_OK;
  baked_query_kernel<V><<<(unsigned)((n_points + kQueryThreads - 1) / kQueryThreads), kQueryThreads, 0,
                          static_cast<cudaStream_t>(stream)>>>(baked_box(box), brick_map, values, use_viewdirs ? 1 : 0,
                                                               pts, dirs, n_points, raw, grad, dequant);
  return check_launch(what);
}

// the peak weights' entry points, as baked_render
template <typename V>
int baked_max_weights(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const V* values,
                      int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays, float* max_w,
                      void* stream, const float* dequant) {
  if (int rc = check_grid(box, what)) return rc;
  if (!brick_map || !values || !rays || !max_w || n_rays <= 0 || ray_stride < (use_viewdirs ? 11 : 8)) {
    set_error("%s: null pointer, n_rays <= 0 or ray_stride %d too short", what, ray_stride);
    return NERFB200_ERR_INVALID;
  }
  if (int rc = check_values(what, values, dequant)) return rc;
  const BakedBox B = baked_box(box);
  const int64_t blocks = (n_rays + kBakedWarps - 1) / kBakedWarps;
  baked_max_weight_kernel<V><<<(unsigned)blocks, kBakedWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      B, brick_map, values, rays, ray_stride, n_rays, reinterpret_cast<unsigned*>(max_w), dequant);
  return check_launch(what);
}

}  // namespace

extern "C" {

int32_t nerfb200_baked_render(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                              int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                              int32_t white_background, float stop_transmittance, float* out, void* stream) {
  return baked_render("baked_render", box, brick_map, values, use_viewdirs, rays, ray_stride, n_rays, white_background,
                      stop_transmittance, out, stream, nullptr);
}

int32_t nerfb200_baked_render_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                  int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                  int32_t white_background, float stop_transmittance, float* out, void* stream) {
  return baked_render("baked_render_f16", box, brick_map, reinterpret_cast<const __half*>(values), use_viewdirs, rays,
                      ray_stride, n_rays, white_background, stop_transmittance, out, stream, nullptr);
}

int32_t nerfb200_baked_render_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                 const float* dequant, int32_t use_viewdirs, const float* rays, int32_t ray_stride,
                                 int64_t n_rays, int32_t white_background, float stop_transmittance, float* out,
                                 void* stream) {
  return baked_render("baked_render_u8", box, brick_map, values, use_viewdirs, rays, ray_stride, n_rays,
                      white_background, stop_transmittance, out, stream, dequant);
}

int32_t nerfb200_baked_render_normals(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                      int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                      int32_t white_background, float stop_transmittance, const nerfb200_ndc_t* ndc,
                                      float* out, float* normals, void* stream) {
  return baked_render_normals("baked_render_normals", box, brick_map, values, use_viewdirs, rays, ray_stride, n_rays,
                              white_background, stop_transmittance, ndc, out, normals, stream, nullptr);
}

int32_t nerfb200_baked_render_normals_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                          int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                          int32_t white_background, float stop_transmittance,
                                          const nerfb200_ndc_t* ndc, float* out, float* normals, void* stream) {
  return baked_render_normals("baked_render_normals_f16", box, brick_map, reinterpret_cast<const __half*>(values),
                              use_viewdirs, rays, ray_stride, n_rays, white_background, stop_transmittance, ndc, out,
                              normals, stream, nullptr);
}

int32_t nerfb200_baked_render_normals_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                         const float* dequant, int32_t use_viewdirs, const float* rays,
                                         int32_t ray_stride, int64_t n_rays, int32_t white_background,
                                         float stop_transmittance, const nerfb200_ndc_t* ndc, float* out,
                                         float* normals, void* stream) {
  return baked_render_normals("baked_render_normals_u8", box, brick_map, values, use_viewdirs, rays, ray_stride,
                              n_rays, white_background, stop_transmittance, ndc, out, normals, stream, dequant);
}

int32_t nerfb200_baked_query(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                             int32_t use_viewdirs, const float* pts, const float* dirs, int64_t n_points, float* raw,
                             float* grad, void* stream) {
  return baked_query("baked_query", box, brick_map, values, use_viewdirs, pts, dirs, n_points, raw, grad, stream,
                     nullptr);
}

int32_t nerfb200_baked_query_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                 int32_t use_viewdirs, const float* pts, const float* dirs, int64_t n_points,
                                 float* raw, float* grad, void* stream) {
  return baked_query("baked_query_f16", box, brick_map, reinterpret_cast<const __half*>(values), use_viewdirs, pts,
                     dirs, n_points, raw, grad, stream, nullptr);
}

int32_t nerfb200_baked_query_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                const float* dequant, int32_t use_viewdirs, const float* pts, const float* dirs,
                                int64_t n_points, float* raw, float* grad, void* stream) {
  return baked_query("baked_query_u8", box, brick_map, values, use_viewdirs, pts, dirs, n_points, raw, grad, stream,
                     dequant);
}

int32_t nerfb200_baked_max_weights(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                   int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                   float* max_w, void* stream) {
  return baked_max_weights("baked_max_weights", box, brick_map, values, use_viewdirs, rays, ray_stride, n_rays, max_w,
                           stream, nullptr);
}

int32_t nerfb200_baked_max_weights_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                       int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                       float* max_w, void* stream) {
  return baked_max_weights("baked_max_weights_f16", box, brick_map, reinterpret_cast<const __half*>(values),
                           use_viewdirs, rays, ray_stride, n_rays, max_w, stream, nullptr);
}

int32_t nerfb200_baked_max_weights_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                      const float* dequant, int32_t use_viewdirs, const float* rays, int32_t ray_stride,
                                      int64_t n_rays, float* max_w, void* stream) {
  return baked_max_weights("baked_max_weights_u8", box, brick_map, values, use_viewdirs, rays, ray_stride, n_rays,
                           max_w, stream, dequant);
}

int32_t nerfb200_baked_render_bwd(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                  int32_t use_viewdirs, const float* rays, int32_t ray_stride, int64_t n_rays,
                                  int32_t white_background, const float* out, const float* g_out, float* d_values,
                                  void* stream) {
  if (int rc = check_grid(box, "baked_render_bwd")) return rc;
  if (!brick_map || !values || !rays || !out || !g_out || !d_values || n_rays <= 0 ||
      ray_stride < (use_viewdirs ? 11 : 8)) {
    set_error("baked_render_bwd: null pointer, n_rays <= 0 or ray_stride %d too short", ray_stride);
    return NERFB200_ERR_INVALID;
  }
  const BakedBox B = baked_box(box);
  const int64_t blocks = (n_rays + kBakedWarps - 1) / kBakedWarps;
  baked_render_bwd_kernel<<<(unsigned)blocks, kBakedWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      B, brick_map, values, use_viewdirs ? 1 : 0, rays, ray_stride, n_rays, white_background ? 1 : 0, out, g_out,
      d_values);
  count_launch();
  return check_cuda(cudaGetLastError(), "baked_render_bwd launch");
}

int32_t nerfb200_baked_tie(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks, int64_t n_active,
                           const float* d_values, float* d_tied, void* stream) {
  if (int rc = check_grid(box, "baked_tie")) return rc;
  const int64_t n_bricks = nerfb200_mesh_sparse_brick_count(box);
  if (!brick_map || !bricks || !d_values || !d_tied || n_active <= 0 || n_active > n_bricks) {
    set_error("baked_tie: null pointer or n_active %lld outside 1 .. %lld", (long long)n_active, (long long)n_bricks);
    return NERFB200_ERR_INVALID;
  }
  const int64_t n4 = n_active * kBakePts * (kBakeCh / 4);
  const float* a_end = d_values + 4 * n4;
  const float* b_end = d_tied + 4 * n4;
  if (d_values < b_end && d_tied < a_end) {
    set_error("baked_tie: d_values and d_tied overlap (the tie is out of place)");
    return NERFB200_ERR_INVALID;
  }
  const BakedBox B = baked_box(box);
  baked_tie_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      B, brick_map, bricks, n_active, reinterpret_cast<const float4*>(d_values), reinterpret_cast<float4*>(d_tied));
  count_launch();
  return check_cuda(cudaGetLastError(), "baked_tie launch");
}

int32_t nerfb200_baked_lattice_count(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                     int64_t n_active, int64_t* count, void* stream) {
  if (int rc = check_grid(box, "baked_lattice_count")) return rc;
  const int64_t n_bricks = nerfb200_mesh_sparse_brick_count(box);
  if (!brick_map || !bricks || !count || n_active <= 0 || n_active > n_bricks) {
    set_error("baked_lattice_count: null pointer or n_active %lld outside 1 .. %lld", (long long)n_active,
              (long long)n_bricks);
    return NERFB200_ERR_INVALID;
  }
  const BakedBox B = baked_box(box);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (int rc = check_cuda(cudaMemsetAsync(count, 0, sizeof(int64_t), s), "baked_lattice_count memset")) return rc;
  const int64_t n = n_active * kBakePts;
  baked_count_kernel<<<(unsigned)((n + kRegThreads - 1) / kRegThreads), kRegThreads, 0, s>>>(
      B, brick_map, bricks, n_active, reinterpret_cast<unsigned long long*>(count));
  count_launch();
  return check_cuda(cudaGetLastError(), "baked_lattice_count launch");
}

int32_t nerfb200_baked_regularizer(const nerfb200_grid_t* box, const int32_t* brick_map, const int32_t* bricks,
                                   int64_t n_active, const float* values, const int64_t* count, double tv_sigma,
                                   double tv_sh, double sparsity, float* d, double* partials, void* stream) {
  if (int rc = check_grid(box, "baked_regularizer")) return rc;
  const int64_t n_bricks = nerfb200_mesh_sparse_brick_count(box);
  if (!brick_map || !bricks || !values || !count || (!d && !partials) || n_active <= 0 || n_active > n_bricks) {
    set_error("baked_regularizer: null pointer, d and partials both null, or n_active %lld outside 1 .. %lld",
              (long long)n_active, (long long)n_bricks);
    return NERFB200_ERR_INVALID;
  }
  const double lam[3] = {tv_sigma, tv_sh, sparsity};
  for (double l : lam)
    if (!(l >= 0.0 && l < INFINITY)) {
      set_error("baked_regularizer: the weights must be finite and >= 0, got %g %g %g", tv_sigma, tv_sh, sparsity);
      return NERFB200_ERR_INVALID;
    }
  const int64_t n = n_active * kBakePts * kBakeCh;
  if (d && d < values + n && values < d + n) {
    set_error("baked_regularizer: d overlaps values");
    return NERFB200_ERR_INVALID;
  }
  const BakedBox B = baked_box(box);
  baked_reg_kernel<<<(unsigned)n_active, kRegThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      B, brick_map, bricks, values, reinterpret_cast<const long long*>(count), tv_sigma, tv_sh, sparsity, d, partials);
  count_launch();
  return check_cuda(cudaGetLastError(), "baked_regularizer launch");
}

}  // extern "C"

// ---- subdivision (include/nerfb200.h "baked fields: subdivision") ----
namespace nerfb200 {
namespace {

constexpr int kSubThreads = 256;
constexpr int kSubStage = 5;  // parent points per axis a child brick reads: 4 delta .. 4 delta + 4 of its parent brick
constexpr int kSubStaged = kSubStage * kSubStage * kSubStage;

// One CTA per child slot.  The 5 x 5 x 5 parent points the child brick reads (channels 0 .. 27, seven float4 each) are
// staged in shared memory from the parent brick's slot; the child slot's 729 x 8 float4 are then written point-major,
// one thread per float4, each channel group summed over the point's 2^m parent points in corner order.
__global__ void __launch_bounds__(kSubThreads)
baked_subdivide_kernel(const BakedBox C, const int* __restrict__ brick_map, int nb0, int nb1, int64_t n_active,
                       const float4* __restrict__ values, const int* __restrict__ child_bricks,
                       float4* __restrict__ child_values) {
  __shared__ float4 stage[kSubStaged][kBakedVals / 4];
  const int64_t slot = blockIdx.x;
  const int cb = child_bricks[slot];
  const int bc[3] = {cb % C.nb[0], (cb / C.nb[0]) % C.nb[1], cb / (C.nb[0] * C.nb[1])};
  const int64_t ps = brick_map[((int64_t)(bc[2] >> 1) * nb1 + (bc[1] >> 1)) * nb0 + (bc[0] >> 1)];
  const bool have = ps >= 0 && ps < n_active;  // a CTA-uniform branch
  float4* out = child_values + slot * (kBakePts * (kBakeCh / 4));
  if (!have) {
    for (int e = threadIdx.x; e < kBakePts * (kBakeCh / 4); e += kSubThreads) out[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float4* src = values + ps * (kBakePts * (kBakeCh / 4));
  for (int e = threadIdx.x; e < kSubStaged * (kBakedVals / 4); e += kSubThreads) {
    const int sp = e / (kBakedVals / 4), c4 = e - sp * (kBakedVals / 4);
    const int sx = sp % kSubStage, sy = (sp / kSubStage) % kSubStage, sz = sp / (kSubStage * kSubStage);
    const int lx = 4 * (bc[0] & 1) + sx, ly = 4 * (bc[1] & 1) + sy, lz = 4 * (bc[2] & 1) + sz;
    stage[sp][c4] = __ldg(src + ((lz * 9 + ly) * 9 + lx) * (kBakeCh / 4) + c4);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kBakePts * (kBakeCh / 4); e += kSubThreads) {
    const int p = e >> 3, c4 = e & 7;
    if (c4 >= kBakedVals / 4) {  // channels 28 .. 31
      out[e] = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const int l[3] = {p % 9, (p / 9) % 9, p / 81};
    int s0[3], odd[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int q = min(kBakeBrick * bc[c] + l[c], C.g.res[c]);  // the child lattice index
      s0[c] = (q >> 1) - 4 * bc[c];
      odd[c] = q & 1;
    }
    const int m = odd[0] + odd[1] + odd[2];
    if (m == 0) {  // a parent point: its bits
      out[e] = stage[(s0[2] * kSubStage + s0[1]) * kSubStage + s0[0]][c4];
      continue;
    }
    const float w = m == 1 ? 0.5f : (m == 2 ? 0.25f : 0.125f);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    bool first = true;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
      if ((dx && !odd[0]) || (dy && !odd[1]) || (dz && !odd[2])) continue;  // absent along an even axis
      const float4 v = stage[((s0[2] + dz) * kSubStage + s0[1] + dy) * kSubStage + s0[0] + dx][c4];
      const float4 t = make_float4(__fmul_rn(w, v.x), __fmul_rn(w, v.y), __fmul_rn(w, v.z), __fmul_rn(w, v.w));
      if (first) {
        acc = t;
        first = false;
      } else {
        acc = make_float4(__fadd_rn(acc.x, t.x), __fadd_rn(acc.y, t.y), __fadd_rn(acc.z, t.z), __fadd_rn(acc.w, t.w));
      }
    }
    out[e] = acc;
  }
}

}  // namespace
}  // namespace nerfb200

extern "C" {

int32_t nerfb200_baked_subdivide(const nerfb200_grid_t* box, const int32_t* brick_map, int64_t n_active,
                                 const float* values, const int32_t* child_bricks, int64_t n_child,
                                 float* child_values, void* stream) {
  if (int rc = check_grid(box, "baked_subdivide")) return rc;
  nerfb200_grid_t child = *box;
  for (int c = 0; c < 3; ++c) {
    if (box->res[c] > NERFB200_GRID_MAX_RES / 2) {
      set_error("baked_subdivide: the child resolution 2 x %d on axis %d is past %d", box->res[c], c,
                NERFB200_GRID_MAX_RES);
      return NERFB200_ERR_INVALID;
    }
    child.res[c] = 2 * box->res[c];
  }
  const int64_t n_bricks = nerfb200_mesh_sparse_brick_count(box);
  const int64_t n_child_bricks = nerfb200_mesh_sparse_brick_count(&child);
  if (!brick_map || !values || !child_bricks || !child_values || n_active < 0 || n_active > n_bricks ||
      n_child < 0 || n_child > n_child_bricks) {
    set_error("baked_subdivide: null pointer, n_active %lld outside 0 .. %lld or n_child %lld outside 0 .. %lld",
              (long long)n_active, (long long)n_bricks, (long long)n_child, (long long)n_child_bricks);
    return NERFB200_ERR_INVALID;
  }
  const int64_t per = (int64_t)kBakePts * kBakeCh;
  if (child_values < values + n_active * per && values < child_values + n_child * per) {
    set_error("baked_subdivide: child_values overlaps values");
    return NERFB200_ERR_INVALID;
  }
  if (n_child == 0) return NERFB200_OK;
  const BakedBox B = baked_box(box), Cb = baked_box(&child);
  baked_subdivide_kernel<<<(unsigned)n_child, kSubThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      Cb, brick_map, B.nb[0], B.nb[1], n_active, reinterpret_cast<const float4*>(values), child_bricks,
      reinterpret_cast<float4*>(child_values));
  count_launch();
  return check_cuda(cudaGetLastError(), "baked_subdivide launch");
}

}  // extern "C"

// ---- meshes (include/nerfb200.h "baked fields: meshes") ----
namespace nerfb200 {
namespace {

constexpr int kMeshAttrThreads = 256;

// the lattice edge (q, a) of an edge key q * 3 + a, or false for a key outside the lattice's edges
__device__ __forceinline__ bool edge_of_key(const Lattice& L, int64_t key, int q[3], int& a) {
  if (key < 0 || key >= 3 * L.total) return false;
  const int64_t p = key / 3;
  a = (int)(key - 3 * p);
  q[0] = (int)(p % L.n[0]);
  q[1] = (int)((p / L.n[0]) % L.n[1]);
  q[2] = (int)(p / L.n01);
  return (a == 0 ? q[0] : (a == 1 ? q[1] : q[2])) < (a == 0 ? L.res[0] : (a == 1 ? L.res[1] : L.res[2]));
}

// sigma_raw at lattice point q, read at its canonical copy; 0 (the renderer's miss) when no active brick holds q
template <typename V>
__device__ __forceinline__ float lattice_sigma(const BakedBox& B, const int* __restrict__ brick_map,
                                               const V* __restrict__ values, const float* dq, const int q[3]) {
  const int64_t cp = canonical_copy(B, brick_map, q);
  return cp < 0 ? 0.f : baked_ld(values + cp, dq);
}

// mesh_emit's gradient at lattice point q over sigma_raw at canonical copies (central differences, one-sided at the
// lattice's faces)
template <typename V>
__device__ __forceinline__ void lattice_grad(const BakedBox& B, const Lattice& L, const int* __restrict__ brick_map,
                                             const V* __restrict__ values, const float* dq, const int q[3],
                                             float g[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int lo = q[c] > 0 ? q[c] - 1 : 0, hi = q[c] < L.res[c] ? q[c] + 1 : L.res[c];
    int ph[3] = {q[0], q[1], q[2]}, pl[3] = {q[0], q[1], q[2]};
    ph[c] = hi;
    pl[c] = lo;
    g[c] = grad_component(L, c, lattice_sigma(B, brick_map, values, dq, ph),
                          lattice_sigma(B, brick_map, values, dq, pl), hi, lo);
  }
}

// One thread per vertex: t on the edge's sigma_raw, the endpoints' gradients, the view direction and (normals may be
// NULL) the outward normal, -dir or 0 where the direction fell back.  NaN for a key off the lattice or an endpoint no
// active brick holds.
template <typename V>
__global__ void __launch_bounds__(kMeshAttrThreads)
baked_mesh_dirs_kernel(const BakedBox B, const Lattice L, const int* __restrict__ brick_map,
                       const V* __restrict__ values, float level, const int64_t* __restrict__ keys, int64_t n,
                       float* __restrict__ dirs, float* __restrict__ normals, const float* __restrict__ dequant_tab) {
  __shared__ float dq[sizeof(V) == 1 ? 2 * kBakedVals : 1];  // uint8 fields only
  stage_dequant<V>(dequant_tab, dq);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float d[3] = {NAN, NAN, NAN}, nrm[3] = {NAN, NAN, NAN};
  int q[3], a;
  if (edge_of_key(L, keys[i], q, a)) {
    const int q1[3] = {q[0] + (a == 0), q[1] + (a == 1), q[2] + (a == 2)};  // a compared, not indexed: registers
    const int64_t c0 = canonical_copy(B, brick_map, q), c1 = canonical_copy(B, brick_map, q1);
    if (c0 >= 0 && c1 >= 0) {
      const float t = edge_t(level, baked_ld(values + c0, dq), baked_ld(values + c1, dq));
      float g0[3], g1[3];
      lattice_grad(B, L, brick_map, values, dq, q, g0);
      lattice_grad(B, L, brick_map, values, dq, q1, g1);
      const bool ok = edge_dir(g0, g1, t, d);
#pragma unroll
      for (int c = 0; c < 3; ++c) nrm[c] = ok ? -d[c] : 0.f;
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) dirs[3 * i + c] = d[c];
  if (normals) {
#pragma unroll
    for (int c = 0; c < 3; ++c) normals[3 * i + c] = nrm[c];
  }
}

// One thread per vertex: channels 0 .. 27 at the vertex by the renderer's fmaf chain over the edge's two endpoints
// (weights 1 - t and t), then the renderer's colour seen along dirs[i] (Y_0 alone without view directions).  NaN where
// baked_mesh_dirs_kernel writes NaN.
template <typename V>
__global__ void __launch_bounds__(kMeshAttrThreads)
baked_mesh_colors_kernel(const BakedBox B, const Lattice L, const int* __restrict__ brick_map,
                         const V* __restrict__ values, int use_viewdirs, float level,
                         const int64_t* __restrict__ keys, const float* __restrict__ dirs, int64_t n,
                         float* __restrict__ colors, const float* __restrict__ dequant_tab) {
  __shared__ float dq[sizeof(V) == 1 ? 2 * kBakedVals : 1];  // uint8 fields only
  stage_dequant<V>(dequant_tab, dq);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float rgb[3] = {NAN, NAN, NAN};
  int q[3], a;
  if (edge_of_key(L, keys[i], q, a)) {
    const int q1[3] = {q[0] + (a == 0), q[1] + (a == 1), q[2] + (a == 2)};  // a compared, not indexed: registers
    const int64_t c0 = canonical_copy(B, brick_map, q), c1 = canonical_copy(B, brick_map, q1);
    if (c0 >= 0 && c1 >= 0) {
      float v0[kBakedVals], v1[kBakedVals], v[kBakedVals];
      baked_point(values + c0, 0, dq, [&](int ch, float x) { v0[ch] = x; });
      baked_point(values + c1, 0, dq, [&](int ch, float x) { v1[ch] = x; });
      const float t = edge_t(level, v0[0], v1[0]), u = __fsub_rn(1.0f, t);
#pragma unroll
      for (int ch = 0; ch < kBakedVals; ++ch) v[ch] = fmaf(t, v1[ch], fmaf(u, v0[ch], 0.f));
      float Y[kBakeSh];
      if (use_viewdirs) sh_basis(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2], Y);
      else Y[0] = 0.28209479177387814f;
      baked_colour(use_viewdirs, Y, v, rgb);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) colors[3 * i + c] = rgb[c];
}

// the checks baked_mesh_dirs and baked_mesh_colors share
int check_baked_mesh(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const void* values,
                     float level, const int64_t* edge_keys, int64_t n_vertices, const void* out) {
  if (int rc = check_grid(box, what)) return rc;
  if (!brick_map || !values || !edge_keys || !out || n_vertices < 0) {
    set_error("%s: null pointer or n_vertices %lld < 0", what, (long long)n_vertices);
    return NERFB200_ERR_INVALID;
  }
  if (!std::isfinite(level)) {
    set_error("%s: level must be finite, got %g", what, (double)level);
    return NERFB200_ERR_INVALID;
  }
  return NERFB200_OK;
}

// the mesh directions' entry points (what: the entry point's name in the errors): the mesh checks, the format's, then
// the launch (none for no vertex)
template <typename V>
int baked_mesh_dirs(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const V* values,
                    float level, const int64_t* edge_keys, int64_t n_vertices, float* dirs, float* normals,
                    void* stream, const float* dequant) {
  if (int rc = check_baked_mesh(what, box, brick_map, values, level, edge_keys, n_vertices, dirs)) return rc;
  if (int rc = check_values(what, values, dequant)) return rc;
  if (n_vertices == 0) return NERFB200_OK;
  baked_mesh_dirs_kernel<V><<<(unsigned)((n_vertices + kMeshAttrThreads - 1) / kMeshAttrThreads), kMeshAttrThreads, 0,
                              static_cast<cudaStream_t>(stream)>>>(baked_box(box), make_lattice(*box), brick_map,
                                                                   values, level, edge_keys, n_vertices, dirs,
                                                                   normals, dequant);
  return check_launch(what);
}

// the mesh colours' entry points, as baked_mesh_dirs
template <typename V>
int baked_mesh_colors(const char* what, const nerfb200_grid_t* box, const int32_t* brick_map, const V* values,
                      int32_t use_viewdirs, float level, const int64_t* edge_keys, const float* dirs,
                      int64_t n_vertices, float* colors, void* stream, const float* dequant) {
  if (int rc = check_baked_mesh(what, box, brick_map, values, level, edge_keys, n_vertices, colors)) return rc;
  if (use_viewdirs && !dirs) {
    set_error("%s: view directions need dirs", what);
    return NERFB200_ERR_INVALID;
  }
  if (int rc = check_values(what, values, dequant)) return rc;
  if (n_vertices == 0) return NERFB200_OK;
  baked_mesh_colors_kernel<V><<<(unsigned)((n_vertices + kMeshAttrThreads - 1) / kMeshAttrThreads), kMeshAttrThreads,
                                0, static_cast<cudaStream_t>(stream)>>>(baked_box(box), make_lattice(*box), brick_map,
                                                                        values, use_viewdirs ? 1 : 0, level, edge_keys,
                                                                        dirs, n_vertices, colors, dequant);
  return check_launch(what);
}

}  // namespace
}  // namespace nerfb200

extern "C" {

int32_t nerfb200_baked_mesh_dirs(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                 float level, const int64_t* edge_keys, int64_t n_vertices, float* dirs,
                                 float* normals, void* stream) {
  return baked_mesh_dirs("baked_mesh_dirs", box, brick_map, values, level, edge_keys, n_vertices, dirs, normals, stream,
                         nullptr);
}

int32_t nerfb200_baked_mesh_dirs_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                     float level, const int64_t* edge_keys, int64_t n_vertices, float* dirs,
                                     float* normals, void* stream) {
  return baked_mesh_dirs("baked_mesh_dirs_f16", box, brick_map, reinterpret_cast<const __half*>(values), level,
                         edge_keys, n_vertices, dirs, normals, stream, nullptr);
}

int32_t nerfb200_baked_mesh_colors(const nerfb200_grid_t* box, const int32_t* brick_map, const float* values,
                                   int32_t use_viewdirs, float level, const int64_t* edge_keys, const float* dirs,
                                   int64_t n_vertices, float* colors, void* stream) {
  return baked_mesh_colors("baked_mesh_colors", box, brick_map, values, use_viewdirs, level, edge_keys, dirs,
                           n_vertices, colors, stream, nullptr);
}

int32_t nerfb200_baked_mesh_colors_f16(const nerfb200_grid_t* box, const int32_t* brick_map, const uint16_t* values,
                                       int32_t use_viewdirs, float level, const int64_t* edge_keys, const float* dirs,
                                       int64_t n_vertices, float* colors, void* stream) {
  return baked_mesh_colors("baked_mesh_colors_f16", box, brick_map, reinterpret_cast<const __half*>(values),
                           use_viewdirs, level, edge_keys, dirs, n_vertices, colors, stream, nullptr);
}

int32_t nerfb200_baked_mesh_dirs_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                    const float* dequant, float level, const int64_t* edge_keys, int64_t n_vertices,
                                    float* dirs, float* normals, void* stream) {
  return baked_mesh_dirs("baked_mesh_dirs_u8", box, brick_map, values, level, edge_keys, n_vertices, dirs, normals,
                         stream, dequant);
}

int32_t nerfb200_baked_mesh_colors_u8(const nerfb200_grid_t* box, const int32_t* brick_map, const uint8_t* values,
                                      const float* dequant, int32_t use_viewdirs, float level, const int64_t* edge_keys,
                                      const float* dirs, int64_t n_vertices, float* colors, void* stream) {
  return baked_mesh_colors("baked_mesh_colors_u8", box, brick_map, values, use_viewdirs, level, edge_keys, dirs,
                           n_vertices, colors, stream, dequant);
}

}  // extern "C"
