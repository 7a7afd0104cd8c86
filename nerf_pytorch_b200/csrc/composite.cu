// composite.cu -- volume_render_radiance_field (nerf/volume_rendering_utils.py:6-53) with the
// exclusive cumprod of nerf/nerf_helpers.py:43-64, forward and backward.  One warp per ray; lane L
// owns the contiguous chunk of samples [L*C, (L+1)*C), C = ceil(S/32); the exclusive product /
// suffix sum across chunks is a warp shuffle scan.
//
// Algorithmic HBM bytes per ray (fp32): forward reads raw (16 S) + z (4 S) + noise (4 S; none when the noise is
// generated in-kernel from the seeded stream) + ray (12), writes weights (4 S, coarse only) + 32 B of outputs;
// SURVEY.md section 8(d).
#include "composite.cuh"

namespace nerfb200 {

constexpr int kCompWarps = 4;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// exclusive additive SUFFIX scan across lanes: sum of v over lanes > lane
__device__ __forceinline__ float warp_excl_suffix_sum(float v, int lane) {
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_down_sync(0xffffffffu, inc, o);
    if (lane + o < 32) inc += n;
  }
  const float ex = __shfl_down_sync(0xffffffffu, inc, 1);
  return lane == 31 ? 0.0f : ex;
}

__global__ void __launch_bounds__(kCompWarps * 32)
composite_fwd_kernel(const float* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ dirs,
                     int dir_stride, const RandSrc noise, int64_t n_rays, int S, float noise_std,
                     int white_bkgd, float* __restrict__ out, float* __restrict__ weights) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = blockIdx.x * (int64_t)kCompWarps + warp;
  if (r >= n_rays) return;
  float* s_alpha = smem + (size_t)warp * S;
  const int C = (S + 31) >> 5;
  const int j0 = lane * C, j1 = min(S, j0 + C);
  const float* rd = dirs + r * dir_stride;
  const float dx = rd[0], dy = rd[1], dz = rd[2];
  const float dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
  const float4* raw4 = reinterpret_cast<const float4*>(raw) + r * S;
  const float* zr = z + r * S;
  const bool has_noise = noise.present() && noise_std > 0.f;

  float prod = 1.0f;
  for (int j = j0; j < j1; ++j) {
    const float zi = zr[j];
    const bool last = (j == S - 1);
    const float zn = last ? 0.f : zr[j + 1];
    const SampleTerms t = sample_terms(raw4[j].w, has_noise ? noise.normal(r, j) : 0.f, noise_std, has_noise, zi, zn, last, dnorm);
    s_alpha[j] = t.alpha;
    prod *= t.q;
  }
  float T = warp_excl_prod(prod, lane);
  float ar = 0.f, ag = 0.f, ab = 0.f, adepth = 0.f, aacc = 0.f;
  for (int j = j0; j < j1; ++j) {
    const float a = s_alpha[j];
    const float w = a * T;
    T *= __fadd_rn(__fsub_rn(1.0f, a), 1e-10f);
    const float4 rv = raw4[j];
    ar += w * sigmoidf_(rv.x);
    ag += w * sigmoidf_(rv.y);
    ab += w * sigmoidf_(rv.z);
    adepth += w * zr[j];
    aacc += w;
    if (weights) weights[r * S + j] = w;
  }
  ar = warp_sum(ar); ag = warp_sum(ag); ab = warp_sum(ab); adepth = warp_sum(adepth); aacc = warp_sum(aacc);
  if (lane == 0) {
    const float disp = 1.0f / fmaxf(1e-10f, adepth / aacc);  // :48 (NaN when acc == 0, like the reference)
    if (white_bkgd) {                                        // :50-51
      const float bg = 1.0f - aacc;
      ar += bg; ag += bg; ab += bg;
    }
    float4* o = reinterpret_cast<float4*>(out + r * 8);
    // fmaxf drops NaNs; keep the reference's NaN for empty rays
    const float ratio = adepth / aacc;
    const float disp_out = (ratio != ratio) ? ratio : disp;
    o[0] = make_float4(ar, ag, ab, disp_out);
    o[1] = make_float4(aacc, adepth, 0.f, 0.f);
  }
}

// kSampleGrads: the upstream gradient also has a depth slot g_out[r][5] and, when g_w is not null, per-sample
// weight terms g_w[r][S]; the render path's instance reads neither
template <bool kSampleGrads>
__global__ void __launch_bounds__(kCompWarps * 32)
composite_bwd_kernel(const float* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ dirs,
                     int dir_stride, const RandSrc noise, const float* __restrict__ g_out,
                     const float* __restrict__ g_w, int64_t n_rays, int S, float noise_std, int white_bkgd,
                     float* __restrict__ d_raw) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = blockIdx.x * (int64_t)kCompWarps + warp;
  if (r >= n_rays) return;
  float* s_alpha = smem + (size_t)warp * 3 * S;
  float* s_v = s_alpha + S;
  float* s_T = s_v + S;
  const int C = (S + 31) >> 5;
  const int j0 = lane * C, j1 = min(S, j0 + C);
  const float* rd = dirs + r * dir_stride;
  const float dx = rd[0], dy = rd[1], dz = rd[2];
  const float dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
  const float4* raw4 = reinterpret_cast<const float4*>(raw) + r * S;
  const float* zr = z + r * S;
  const bool has_noise = noise.present() && noise_std > 0.f;
  const float4 g0 = reinterpret_cast<const float4*>(g_out + r * 8)[0];  // d r g b disp
  const float g_acc_in = g_out[r * 8 + 4];

  // pass 1: alpha, per-lane product of q, first moments (needed for the disp gradient)
  float prod = 1.0f;
  for (int j = j0; j < j1; ++j) {
    const bool last = (j == S - 1);
    const SampleTerms t =
        sample_terms(raw4[j].w, has_noise ? noise.normal(r, j) : 0.f, noise_std, has_noise, zr[j], last ? 0.f : zr[j + 1], last, dnorm);
    s_alpha[j] = t.alpha;
    prod *= t.q;
  }
  float T = warp_excl_prod(prod, lane);
  float adepth = 0.f, aacc = 0.f;
  for (int j = j0; j < j1; ++j) {
    const float a = s_alpha[j];
    s_T[j] = T;
    const float w = a * T;
    T *= __fadd_rn(__fsub_rn(1.0f, a), 1e-10f);
    adepth += w * zr[j];
    aacc += w;
  }
  adepth = warp_sum(adepth);
  aacc = warp_sum(aacc);

  // upstream coefficients: L = sum_i w_i * v_i,  v_i = g_rgb . c_i + G_acc + G_depth * z_i (+ g_w_i)
  float G_acc = g_acc_in, G_depth = kSampleGrads ? g_out[r * 8 + 5] : 0.f;
  composite_upstream(g0, white_bkgd, adepth, aacc, G_acc, G_depth);

  // pass 2: v_i and the suffix sums S_i = sum_{j>i} v_j w_j
  float local = 0.f;
  for (int j = j0; j < j1; ++j) {
    const float4 rv = raw4[j];
    float v = g0.x * sigmoidf_(rv.x) + g0.y * sigmoidf_(rv.y) + g0.z * sigmoidf_(rv.z) + G_acc + G_depth * zr[j];
    if (kSampleGrads && g_w) v += g_w[r * S + j];
    s_v[j] = v;
    local += v * s_alpha[j] * s_T[j];
  }
  float suffix = warp_excl_suffix_sum(local, lane);  // contributions of lanes above this one

  // pass 3 (descending within the chunk): dL/dalpha_i = T_i v_i - S_i / q_i
  float4* d4 = reinterpret_cast<float4*>(d_raw) + r * S;
  for (int j = j1 - 1; j >= j0; --j) {
    const float a = s_alpha[j], Tj = s_T[j], v = s_v[j];
    const float q = __fadd_rn(__fsub_rn(1.0f, a), 1e-10f);
    const float dalpha = Tj * v - suffix / q;
    suffix += v * a * Tj;
    const bool last = (j == S - 1);
    const SampleTerms t =
        sample_terms(raw4[j].w, has_noise ? noise.normal(r, j) : 0.f, noise_std, has_noise, zr[j], last ? 0.f : zr[j + 1], last, dnorm);
    const float dsigma = t.gate ? dalpha * t.delta * t.sigma_delta_exp : 0.f;
    const float w = a * Tj;
    const float4 rv = raw4[j];
    const float cr = sigmoidf_(rv.x), cg = sigmoidf_(rv.y), cb = sigmoidf_(rv.z);
    d4[j] = make_float4(w * g0.x * cr * (1.f - cr), w * g0.y * cg * (1.f - cg), w * g0.z * cb * (1.f - cb), dsigma);
  }
}

// Early ray termination (nerfb200.h): after round `round` of a pass's MLP, one warp per ray multiplies the q of the
// ray's rows of that round into its T, in sample order, with the terms composite_fwd_kernel uses.  A ray with samples
// left stops when T < threshold: the rest of its evaluated samples get raw = [0 0 0 -inf] and its count is cut to what
// it ran.  One CTA per compaction group writes the group's rows of the next round.
constexpr int kStopGroupRays = kGridGroupRays;

__global__ void __launch_bounds__(kStopGroupRays * 32)
stop_update_kernel(float* __restrict__ raw, const float* __restrict__ z, const float* __restrict__ dirs, int dir_stride,
                   const RandSrc noise, float noise_std, int64_t n_rays, int S, int round, float threshold, StopState st,
                   const int64_t* __restrict__ round_rows, int64_t* __restrict__ n_evaluated) {
  __shared__ int rows[kStopGroupRays];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * kStopGroupRays + w;
  const int k0 = round * kStopRound;
  int next = 0;
  if (r < n_rays) {
    int n = st.n_eval[r];
    const int end = min(n, k0 + kStopRound);
    if (end > k0) {
      const float* rd = dirs + r * dir_stride;
      const float dx = rd[0], dy = rd[1], dz = rd[2];
      const float dnorm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
      const bool has_noise = noise.present() && noise_std > 0.f;
      const int* ord = st.order + r * S;
      const float4* raw4 = reinterpret_cast<const float4*>(raw) + r * S;
      const float* zr = z + r * S;
      float T = st.T[r];
      for (int b = k0; b < end; b += 32) {
        float q = 1.f;
        if (b + lane < end) {
          const int j = ord[b + lane];
          const bool last = j == S - 1;
          q = sample_terms(raw4[j].w, has_noise ? noise.normal(r, j) : 0.f, noise_std, has_noise, zr[j],
                           last ? 0.f : zr[j + 1], last, dnorm).q;
        }
        const int m = min(32, end - b);
        for (int i = 0; i < m; ++i) T = __fmul_rn(T, __shfl_sync(0xffffffffu, q, i));
      }
      if (T < threshold && end < n) {
        float4* out4 = reinterpret_cast<float4*>(raw) + r * S;
        for (int i = end + lane; i < n; i += 32) out4[ord[i]] = make_float4(0.f, 0.f, 0.f, -INFINITY);
        n = end;
        if (lane == 0) {
          st.n_eval[r] = n;
          if (st.stop) st.stop[r] = ord[end - 1] + 1;
        }
      }
      if (lane == 0) st.T[r] = T;
    }
    next = min(max(n - (k0 + kStopRound), 0), kStopRound);
  }
  if (lane == 0) rows[w] = next;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int i = 0; i < kStopGroupRays; ++i) total += rows[i];
    st.counts[blockIdx.x] = total;
    if (n_evaluated && blockIdx.x == 0) *n_evaluated = (round ? *n_evaluated : 0) + *round_rows;
  }
}

int launch_stop_update(float* raw, const float* z, const float* dirs, int dir_stride, const RandSrc& noise,
                       float noise_std, int64_t n_rays, int n_samples, int round, float threshold, const StopState& st,
                       const int64_t* round_rows, int64_t* n_evaluated, cudaStream_t s) {
  const int64_t groups = (n_rays + kStopGroupRays - 1) / kStopGroupRays;
  stop_update_kernel<<<(unsigned)groups, kStopGroupRays * 32, 0, s>>>(raw, z, dirs, dir_stride, noise, noise_std, n_rays,
                                                                      n_samples, round, threshold, st, round_rows,
                                                                      n_evaluated);
  count_launch();
  return check_cuda(cudaGetLastError(), "stop_update launch");
}

int launch_composite_fwd(const float* raw, const float* z, const float* dirs, int dir_stride, const RandSrc& noise,
                         int64_t n_rays, int n_samples, float noise_std, int white_bkgd, float* out,
                         float* weights, cudaStream_t s) {
  const size_t smem = (size_t)kCompWarps * n_samples * sizeof(float);
  const int64_t blocks = (n_rays + kCompWarps - 1) / kCompWarps;
  composite_fwd_kernel<<<(unsigned)blocks, kCompWarps * 32, smem, s>>>(raw, z, dirs, dir_stride, noise, n_rays,
                                                                       n_samples, noise_std, white_bkgd, out, weights);
  count_launch();
  return check_cuda(cudaGetLastError(), "composite_fwd launch");
}

int launch_composite_bwd(const float* raw, const float* z, const float* dirs, int dir_stride, const RandSrc& noise,
                         const float* g_out, const float* g_w, bool sample_grads, int64_t n_rays, int n_samples,
                         float noise_std, int white_bkgd, float* d_raw, cudaStream_t s) {
  const size_t smem = (size_t)kCompWarps * 3 * n_samples * sizeof(float);
  const int64_t blocks = (n_rays + kCompWarps - 1) / kCompWarps;
  auto kern = sample_grads ? composite_bwd_kernel<true> : composite_bwd_kernel<false>;
  kern<<<(unsigned)blocks, kCompWarps * 32, smem, s>>>(raw, z, dirs, dir_stride, noise, g_out, g_w, n_rays, n_samples,
                                                       noise_std, white_bkgd, d_raw);
  count_launch();
  return check_cuda(cudaGetLastError(), "composite_bwd launch");
}

}  // namespace nerfb200
