// mlp_simt.cu -- fp32 CUDA-core implementation of the fused per-point pipeline
//     points = o + d * z                     nerf/train_utils.py:67,107
//     positional encoding of xyz and viewdir nerf/nerf_helpers.py:113-157, train_utils.py:10-17
//     FlexibleNeRFModel.forward              nerf/models.py:233-256
// and of its backward w.r.t. the parameters.  This is the "parity" implementation: every product
// is an fp32 FMA, exactly the arithmetic class of the reference's fp32 SGEMM path.
//
// Forward: one CTA = one tile of 128 consecutive points.  The encoded inputs and the running
// activation live in shared memory (the (N*S, 90) tensor of train_utils.py:17 never exists in HBM);
// each layer's transposed weights stream from L2 through a double-buffered cp.async ring; each
// thread owns an 8 x (4*NJ) register tile of the 128 x (64*NJ) layer output.
//
// Backward: kernel A walks the layers in reverse for one tile (dgrad chain, ReLU masks from the
// forward stash) and writes the gradient w.r.t. every layer's pre-activation output; kernel B
// reduces dW = dY^T X over all points, one (layer, weight-block) item per blockIdx.y, split over
// blockIdx.x point ranges, accumulated in registers and flushed with one atomicAdd per element.
#include <type_traits>

#include "common.cuh"
#include "wgrad_items.cuh"

namespace nerfb200 {

// ---------------------------------------------------------------------------------------------
// shared-memory GEMM: acc[8][4*NJ] (+)= A[128 x K] * Wt[K x 64*NJ]
//   A = [act (k_h columns, row stride act_ld) | enc (k_enc columns, row stride enc_ld)]  (smem)
//   Wt row-major in global memory with row stride w_ld, staged through wst (2 x kc x N floats).
// thread (ty = tid / 16, tx = tid % 16) owns rows r*16 + ty (r < 8), cols tx*4 + 64*j + i.
// ---------------------------------------------------------------------------------------------
template <int NJ>
__device__ __forceinline__ void gemm_tile(const float* __restrict__ Wt, int w_ld, int k_h, const float* act,
                                          int act_ld, int k_enc, const float* enc, int enc_ld, float* wst, int kc,
                                          float (&acc)[8][4 * NJ], int tid) {
  constexpr int N = 64 * NJ;
  const int ty = tid >> 4, tx = tid & 15;
  const int K = k_h + k_enc;
  const int nchunks = (K + kc - 1) / kc;
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int c = 0; c < 4 * NJ; ++c) acc[r][c] = 0.f;

  auto load_chunk = [&](int c, int buf) {
    const int k0 = c * kc;
    const int rows = min(kc, K - k0);
    float* dst = wst + buf * kc * N;
    const int vec_per_row = N / 4;
    for (int i = tid; i < rows * vec_per_row; i += kThreads) {
      const int rr = i / vec_per_row, cc = i - rr * vec_per_row;
      cp_async16(dst + rr * N + cc * 4, Wt + (size_t)(k0 + rr) * w_ld + cc * 4);
    }
    cp_async_commit();
  };

  load_chunk(0, 0);
  for (int c = 0; c < nchunks; ++c) {
    if (c + 1 < nchunks) {
      load_chunk(c + 1, (c + 1) & 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int k0 = c * kc;
    const int rows = min(kc, K - k0);
    const float* a;
    int lda;
    if (k0 < k_h) {
      a = act + k0;
      lda = act_ld;
    } else {
      a = enc + (k0 - k_h);
      lda = enc_ld;
    }
    a += ty * lda;
    const float* wb = wst + (c & 1) * kc * N + tx * 4;
    for (int k = 0; k < rows; k += 4) {
      float4 x[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) x[r] = *reinterpret_cast<const float4*>(a + r * 16 * lda + k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        float4 w[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) w[j] = *reinterpret_cast<const float4*>(wb + (k + kk) * N + 64 * j);
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const float xv = kk == 0 ? x[r].x : kk == 1 ? x[r].y : kk == 2 ? x[r].z : x[r].w;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            acc[r][4 * j + 0] = fmaf(xv, w[j].x, acc[r][4 * j + 0]);
            acc[r][4 * j + 1] = fmaf(xv, w[j].y, acc[r][4 * j + 1]);
            acc[r][4 * j + 2] = fmaf(xv, w[j].z, acc[r][4 * j + 2]);
            acc[r][4 * j + 3] = fmaf(xv, w[j].w, acc[r][4 * j + 3]);
          }
        }
      }
    }
    __syncthreads();
  }
}

// encodings of the tile's points into shared memory (rows beyond the last point replicate it)
__device__ __forceinline__ void encode_tile(const Plan& p, const PointSrc& src, int64_t p0, int64_t P, int S, int rows,
                                            float* encx, int encx_ld, float* encd, int encd_ld, int tid,
                                            int nthreads) {
  for (int it = tid; it < rows * 6; it += nthreads) {
    const int row = it / 6, rem = it - row * 6;
    const int c = rem % 3, half = rem / 3;
    int64_t pt = p0 + row;
    if (pt >= P) pt = P - 1;
    float x;
    if (src.pts) {
      x = src.pts[pt * 3 + c];
    } else {
      const int64_t ray = pt / S;
      const float o = src.rays[ray * src.ray_stride + c], d = src.rays[ray * src.ray_stride + 3 + c];
      x = __fadd_rn(o, __fmul_rn(d, src.z[pt]));  // pts = ro + rd * z  (train_utils.py:67)
    }
    const int nf = p.n_freq_xyz, mid = nf >> 1;
    encode_coord(x, c, p.inc_xyz, half ? mid : 0, half ? nf : mid, p.freq_xyz, encx + row * encx_ld);
  }
  const int padx = p.dim_xyz_pad - p.dim_xyz;
  for (int it = tid; it < rows * padx; it += nthreads) {
    const int row = it / padx, c = it - row * padx;
    encx[row * encx_ld + p.dim_xyz + c] = 0.f;
  }
  if (encd != nullptr) {
    for (int it = tid; it < rows * 3; it += nthreads) {
      const int row = it / 3, c = it - row * 3;
      int64_t pt = p0 + row;
      if (pt >= P) pt = P - 1;
      const int64_t ray = pt / S;
      const float v = src.dirs[ray * src.dir_stride + c];  // viewdirs = ray_batch[..., -3:]  (train_utils.py:13)
      encode_coord(v, c, p.inc_dir, 0, p.n_freq_dir, p.freq_dir, encd + row * encd_ld);
    }
    const int padd = p.dim_dir_pad - p.dim_dir;
    for (int it = tid; it < rows * padd; it += nthreads) {
      const int row = it / padd, c = it - row * padd;
      encd[row * encd_ld + p.dim_dir + c] = 0.f;
    }
  }
}

struct FwdSmem {
  int act_ld, encx_ld, encd_ld, kc;
  int act_off, encx_off, encd_off, wst_off, hw_off, total_floats;
};

static FwdSmem fwd_smem_layout(const Plan& p) {
  FwdSmem s;
  s.act_ld = p.hidden + 4;
  s.encx_ld = p.dim_xyz_pad + 4;
  s.encd_ld = p.use_viewdirs ? p.dim_dir_pad + 4 : 0;
  s.kc = p.hidden >= 256 ? 16 : 32;
  int off = 0;
  s.act_off = off; off += kTileRows * s.act_ld;
  s.encx_off = off; off += kTileRows * s.encx_ld;
  s.encd_off = off; off += kTileRows * s.encd_ld;
  s.wst_off = off; off += 2 * s.kc * p.hidden;
  s.hw_off = off; off += 5 * p.hidden + 16;  // head weights: <= 4*H (fc_out) or H + 3*H/2, + 2 x 4 biases
  s.total_floats = off;
  return s;
}

// narrow head (fc_alpha / fc_rgb / fc_out): out[row][c] = act[row] . W[c] + b[c], threads 0..127
__device__ __forceinline__ void head_eval(const HeadLayer& h, const float* act, int act_ld, const float* hw,
                                          const float* hb, float* __restrict__ raw, int64_t p0, int64_t P, int tid) {
  if (tid >= kTileRows) return;
  const float* a = act + tid * act_ld;
  float o[4] = {hb[0], hb[1], hb[2], hb[3]};
  for (int k = 0; k < h.k; k += 4) {
    const float4 x = *reinterpret_cast<const float4*>(a + k);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (c < h.n_out) {
        const float4 w = *reinterpret_cast<const float4*>(hw + c * h.k + k);
        o[c] = fmaf(x.x, w.x, o[c]);
        o[c] = fmaf(x.y, w.y, o[c]);
        o[c] = fmaf(x.z, w.z, o[c]);
        o[c] = fmaf(x.w, w.w, o[c]);
      }
    }
  }
  const int64_t pt = p0 + tid;
  if (pt < P) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (c < h.n_out) raw[pt * 4 + h.out_col + c] = o[c];
  }
}

template <int NJH>  // hidden = 64 * NJH
__global__ void __launch_bounds__(kThreads, 1)
mlp_fwd_simt_kernel(const __grid_constant__ Plan p, const FwdSmem sm, const float* __restrict__ blob,
                    const PointSrc src, int64_t P, int S, float* __restrict__ raw, float* __restrict__ stash) {
  extern __shared__ __align__(16) float smem[];
  float* act = smem + sm.act_off;
  float* encx = smem + sm.encx_off;
  float* encd = p.use_viewdirs ? smem + sm.encd_off : nullptr;
  float* wst = smem + sm.wst_off;
  float* hw = smem + sm.hw_off;
  const int tid = threadIdx.x;
  const int64_t p0 = (int64_t)blockIdx.x * kTileRows;

  // head weights + biases -> smem: [h0.W | h1.W | h0.b(4) | h1.b(4)]
  const int hw1 = p.h[0].n_out * p.h[0].k;
  const int hw2 = p.n_head > 1 ? p.h[1].n_out * p.h[1].k : 0;
  float* hb = hw + ((hw1 + hw2 + 3) & ~3);
  for (int i = tid; i < hw1; i += kThreads) hw[i] = blob[p.h[0].w_off + i];
  for (int i = tid; i < hw2; i += kThreads) hw[hw1 + i] = blob[p.h[1].w_off + i];
  if (tid < 4) hb[tid] = blob[p.h[0].b_off + tid];
  if (tid >= 4 && tid < 8 && p.n_head > 1) hb[tid] = blob[p.h[1].b_off + tid - 4];

  encode_tile(p, src, p0, P, S, kTileRows, encx, sm.encx_ld, encd, sm.encd_ld, tid, kThreads);
  if (stash) {  // the backward reads the encodings back instead of recomputing 60 sin/cos per point
    __syncthreads();
    float* sx = stash + (size_t)P * p.enc_cum[0];
    const int vx = p.dim_xyz_pad / 4;
    for (int i = tid; i < kTileRows * vx; i += kThreads) {
      const int row = i / vx, cc = i - row * vx;
      if (p0 + row < P)
        *reinterpret_cast<float4*>(sx + (size_t)(p0 + row) * p.dim_xyz_pad + 4 * cc) =
            *reinterpret_cast<const float4*>(encx + row * sm.encx_ld + 4 * cc);
    }
    if (encd) {
      float* sd = stash + (size_t)P * p.enc_cum[1];
      const int vd = p.dim_dir_pad / 4;
      for (int i = tid; i < kTileRows * vd; i += kThreads) {
        const int row = i / vd, cc = i - row * vd;
        if (p0 + row < P)
          *reinterpret_cast<float4*>(sd + (size_t)(p0 + row) * p.dim_dir_pad + 4 * cc) =
              *reinterpret_cast<const float4*>(encd + row * sm.encd_ld + 4 * cc);
      }
    }
  }
  // (the first __syncthreads inside gemm_tile orders the encoding writes before any read)

  const int ty = tid >> 4, tx = tid & 15;
  for (int gi = 0; gi < p.n_gemm; ++gi) {
    const GemmLayer& g = p.g[gi];
    const float* enc = g.enc_sel ? encd : encx;
    const int enc_ld = g.enc_sel ? sm.encd_ld : sm.encx_ld;
    float* st = stash ? stash + (size_t)P * g.cum_n : nullptr;

    auto epilogue = [&](auto& acc, auto nj_tag) {
      constexpr int NJ = decltype(nj_tag)::value;
      // all reads of `act` finished at the trailing __syncthreads of gemm_tile: update in place
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const float4 b = *reinterpret_cast<const float4*>(blob + g.b_off + tx * 4 + 64 * j);
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          float4 v = make_float4(acc[r][4 * j + 0] + b.x, acc[r][4 * j + 1] + b.y, acc[r][4 * j + 2] + b.z,
                                 acc[r][4 * j + 3] + b.w);
          if (g.relu) {
            v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
          }
          const int row = r * 16 + ty, col = tx * 4 + 64 * j;
          *reinterpret_cast<float4*>(act + row * sm.act_ld + col) = v;
          if (st && p0 + row < P) *reinterpret_cast<float4*>(st + (size_t)(p0 + row) * g.n + swz_col(col, p0 + row)) = v;
        }
      }
      __syncthreads();
      if (stash && tid < kTileRows && p0 + tid < P) {
        // ReLU bit mask of this row, bit c = output c > 0: it fills the stash's mask section, which only the wgmma
        // backward reads (from its own forward's stash); the fp32 backward does not
        uint32_t* mk = reinterpret_cast<uint32_t*>(stash) + (size_t)P * (p.mask_base + g.mask_cum) +
                       (size_t)(p0 + tid) * (g.n / 32);
        for (int w = 0; w < g.n / 32; ++w) {
          uint32_t bits = 0;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 a = *reinterpret_cast<const float4*>(act + tid * sm.act_ld + 32 * w + 4 * q);
            bits |= (a.x > 0.f ? 1u : 0u) << (4 * q) | (a.y > 0.f ? 1u : 0u) << (4 * q + 1) |
                    (a.z > 0.f ? 1u : 0u) << (4 * q + 2) | (a.w > 0.f ? 1u : 0u) << (4 * q + 3);
          }
          mk[w] = bits;
        }
      }
    };

    if (g.n == 64 * NJH) {
      float acc[8][4 * NJH];
      gemm_tile<NJH>(blob + g.wt_off, g.n, g.k_h, act, sm.act_ld, g.k_enc, enc, enc_ld, wst, sm.kc, acc, tid);
      epilogue(acc, std::integral_constant<int, NJH>{});
    } else {
      float acc[8][2 * NJH];
      gemm_tile<NJH / 2>(blob + g.wt_off, g.n, g.k_h, act, sm.act_ld, g.k_enc, enc, enc_ld, wst, sm.kc, acc, tid);
      epilogue(acc, std::integral_constant<int, NJH / 2>{});
    }
    if (p.h[0].src == gi) head_eval(p.h[0], act, sm.act_ld, hw, hb, raw, p0, P, tid);
    if (p.n_head > 1 && p.h[1].src == gi) head_eval(p.h[1], act, sm.act_ld, hw + hw1, hb + 4, raw, p0, P, tid);
  }
}

// the forward's tiles must fit one CTA's shared memory (the backward kernels need less)
int simt_supported(const Plan& p, const char* what) {
  const size_t bytes = (size_t)fwd_smem_layout(p).total_floats * sizeof(float);
  if (bytes > 227 * 1024) {
    set_error("%s: configuration needs %zu bytes of shared memory (> 227 KB)", what, bytes);
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

int launch_mlp_fwd_simt(const Plan& p, const float* blob, const PointSrc& src, int64_t n_rays, int n_samples, float* raw,
                        float* stash, cudaStream_t s) {
  const FwdSmem sm = fwd_smem_layout(p);
  const size_t bytes = (size_t)sm.total_floats * sizeof(float);
  const int64_t P = n_rays * n_samples;
  const int64_t tiles = (P + kTileRows - 1) / kTileRows;
  auto kern = p.hidden == 256 ? mlp_fwd_simt_kernel<4> : mlp_fwd_simt_kernel<2>;
  int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes),
                      "mlp_fwd smem attribute");
  if (rc) return rc;
  kern<<<(unsigned)tiles, kThreads, bytes, s>>>(p, sm, blob, src, P, n_samples, raw, stash);
  count_launch();
  return check_cuda(cudaGetLastError(), "mlp_fwd_simt launch");
}

// =============================================================================================
// backward, kernel A: dgrad chain for one tile
// =============================================================================================
struct BwdSmem {
  int g_ld, kc;
  int g_off, wst_off, dr_off, hw_off, total_floats;
};

static BwdSmem bwd_smem_layout(const Plan& p) {
  BwdSmem s;
  s.g_ld = p.hidden + 4;
  s.kc = p.hidden >= 256 ? 16 : 32;
  int off = 0;
  s.g_off = off; off += kTileRows * s.g_ld;
  s.wst_off = off; off += 2 * s.kc * p.hidden;
  s.dr_off = off; off += kTileRows * 4;
  s.hw_off = off; off += 5 * p.hidden + 16;
  s.total_floats = off;
  return s;
}

template <int NJH>
__global__ void __launch_bounds__(kThreads, 1)
mlp_bwd_dgrad_kernel(const __grid_constant__ Plan p, const BwdSmem sm, const float* __restrict__ blob,
                     const float* __restrict__ d_raw, const float* __restrict__ stash, float* __restrict__ gstash,
                     int64_t P) {
  extern __shared__ __align__(16) float smem[];
  float* G = smem + sm.g_off;
  float* wst = smem + sm.wst_off;
  float* dr = smem + sm.dr_off;
  float* hw = smem + sm.hw_off;
  const int tid = threadIdx.x;
  const int ty = tid >> 4, tx = tid & 15;
  const int64_t p0 = (int64_t)blockIdx.x * kTileRows;

  const int hw1 = p.h[0].n_out * p.h[0].k;
  const int hw2 = p.n_head > 1 ? p.h[1].n_out * p.h[1].k : 0;
  for (int i = tid; i < hw1; i += kThreads) hw[i] = blob[p.h[0].w_off + i];
  for (int i = tid; i < hw2; i += kThreads) hw[hw1 + i] = blob[p.h[1].w_off + i];
  for (int i = tid; i < kTileRows; i += kThreads) {
    const int64_t pt = p0 + i;
    reinterpret_cast<float4*>(dr)[i] =
        pt < P ? reinterpret_cast<const float4*>(d_raw)[pt] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();

  for (int t = p.n_gemm - 1; t >= 0; --t) {
    const GemmLayer& gt = p.g[t];
    // gemm layer consuming gt's output (at most one), and head consuming it (at most one)
    int s = -1;
    for (int c = t + 1; c < p.n_gemm; ++c)
      if (p.g[c].src == t) s = c;
    int hsel = -1;
    for (int c = 0; c < p.n_head; ++c)
      if (p.h[c].src == t) hsel = c;
    const float* hwp = hsel == 1 ? hw + hw1 : hw;
    const float* st = stash + (size_t)P * gt.cum_n;
    float* gs = gstash + (size_t)P * gt.cum_n;

    auto finish = [&](auto& acc, auto nj_tag) {
      constexpr int NJ = decltype(nj_tag)::value;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int row = r * 16 + ty, col = tx * 4 + 64 * j;
          float4 v = make_float4(acc[r][4 * j + 0], acc[r][4 * j + 1], acc[r][4 * j + 2], acc[r][4 * j + 3]);
          if (hsel >= 0) {
            const HeadLayer& h = p.h[hsel];
            for (int c = 0; c < h.n_out; ++c) {
              const float dv = dr[row * 4 + h.out_col + c];
              const float4 w = *reinterpret_cast<const float4*>(hwp + c * h.k + col);
              v.x = fmaf(dv, w.x, v.x); v.y = fmaf(dv, w.y, v.y); v.z = fmaf(dv, w.z, v.z); v.w = fmaf(dv, w.w, v.w);
            }
          }
          const bool inb = p0 + row < P;
          if (gt.relu) {
            float4 a = inb ? *reinterpret_cast<const float4*>(st + (size_t)(p0 + row) * gt.n + swz_col(col, p0 + row))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
            v.x = a.x > 0.f ? v.x : 0.f; v.y = a.y > 0.f ? v.y : 0.f;
            v.z = a.z > 0.f ? v.z : 0.f; v.w = a.w > 0.f ? v.w : 0.f;
          }
          *reinterpret_cast<float4*>(G + row * sm.g_ld + col) = v;
          if (inb) *reinterpret_cast<float4*>(gs + (size_t)(p0 + row) * gt.n + swz_col(col, p0 + row)) = v;
        }
      }
      __syncthreads();
    };

    if (gt.n == 64 * NJH) {
      float acc[8][4 * NJH];
      if (s >= 0) {
        gemm_tile<NJH>(blob + p.g[s].wh_off, p.g[s].k_h, p.g[s].n, G, sm.g_ld, 0, nullptr, 0, wst, sm.kc, acc, tid);
      } else {
#pragma unroll
        for (int r = 0; r < 8; ++r)
#pragma unroll
          for (int c = 0; c < 4 * NJH; ++c) acc[r][c] = 0.f;
        __syncthreads();
      }
      finish(acc, std::integral_constant<int, NJH>{});
    } else {
      float acc[8][2 * NJH];
      if (s >= 0) {
        gemm_tile<NJH / 2>(blob + p.g[s].wh_off, p.g[s].k_h, p.g[s].n, G, sm.g_ld, 0, nullptr, 0, wst, sm.kc, acc,
                           tid);
      } else {
#pragma unroll
        for (int r = 0; r < 8; ++r)
#pragma unroll
          for (int c = 0; c < 2 * NJH; ++c) acc[r][c] = 0.f;
        __syncthreads();
      }
      finish(acc, std::integral_constant<int, NJH / 2>{});
    }
  }
}

// =============================================================================================
// backward, kernel B: weight gradients  dW[n][k] = sum_p dY[p][n] X[p][k],  db[n] = sum_p dY[p][n]
// =============================================================================================
constexpr int kWgPts = 32;  // points per pipeline stage

// register-tile accumulation for one item: RN rows (n = ty*RN + r) x RK cols (k = tx + 16*i)
template <int RN, int RK>
__device__ __forceinline__ void wgrad_block(const Plan& p, const WgItem& it, const float* __restrict__ rays,
                                            int ray_stride, const float* __restrict__ z, int S,
                                            const float* __restrict__ stash, const float* __restrict__ gstash,
                                            int64_t P, int64_t pt_begin, int64_t pt_end, float* smem,
                                            float* __restrict__ flat_grad) {
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const GemmLayer& g = p.g[it.t];
  const int ldy = it.nblk + 4, ldx = it.kblk + 4;  // +4 keeps rows 16-byte aligned and skews banks
  float* ys[2] = {smem, smem + kWgPts * ldy};
  float* xs[2] = {smem + 2 * kWgPts * ldy, smem + 2 * kWgPts * ldy + kWgPts * ldx};
  const float* dY = gstash + (size_t)P * g.cum_n + it.n0;  // [P][g.n]
  const float* X = it.kind == 0 ? stash + (size_t)P * p.g[g.src].cum_n + it.k0 : nullptr;  // [P][k_h]
  const int xw = it.kind == 0 ? p.g[g.src].n : 0;

  float acc[RN][RK];
  float bacc[RN];
#pragma unroll
  for (int r = 0; r < RN; ++r) {
    bacc[r] = 0.f;
#pragma unroll
    for (int i = 0; i < RK; ++i) acc[r][i] = 0.f;
  }

  auto load_stage = [&](int64_t q0, int buf) {
    // dY tile [32][nblk]
    const int vy = it.nblk / 4;
    for (int i = tid; i < kWgPts * vy; i += kThreads) {
      const int pp = i / vy, cc = i - pp * vy;
      float* dst = ys[buf] + pp * ldy + cc * 4;
      if (q0 + pp < pt_end) cp_async16(dst, dY + (size_t)(q0 + pp) * g.n + swz_col(cc * 4, q0 + pp));
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (it.kind == 0) {
      const int vx = it.kblk / 4;
      for (int i = tid; i < kWgPts * vx; i += kThreads) {
        const int pp = i / vx, cc = i - pp * vx;
        float* dst = xs[buf] + pp * ldx + cc * 4;
        if (q0 + pp < pt_end) cp_async16(dst, X + (size_t)(q0 + pp) * xw + swz_col(cc * 4, q0 + pp));
        else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else {
      // encoded-input columns: read the stashed encoding (zero in its padding columns)
      const int ew = g.enc_sel ? p.dim_dir_pad : p.dim_xyz_pad;
      const float* E = stash + (size_t)P * p.enc_cum[g.enc_sel];
      const int vx = it.kblk / 4;
      for (int i = tid; i < kWgPts * vx; i += kThreads) {
        const int pp = i / vx, cc = i - pp * vx;
        float* dst = xs[buf] + pp * ldx + cc * 4;
        if (q0 + pp < pt_end && 4 * cc < ew) cp_async16(dst, E + (size_t)(q0 + pp) * ew + cc * 4);
        else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    cp_async_commit();
  };

  const bool row_active = ty * RN < it.nblk;
  int buf = 0;
  if (pt_begin < pt_end) load_stage(pt_begin, 0);
  for (int64_t q0 = pt_begin; q0 < pt_end; q0 += kWgPts) {
    const bool more = q0 + kWgPts < pt_end;
    if (more) {
      load_stage(q0 + kWgPts, buf ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (row_active) {
      const float* yb = ys[buf] + ty * RN;
      const float* xb = xs[buf] + tx;
#pragma unroll 4
      for (int pp = 0; pp < kWgPts; ++pp) {
        float dy[RN];
#pragma unroll
        for (int r4 = 0; r4 < RN / 4; ++r4) {
          const float4 v = *reinterpret_cast<const float4*>(yb + pp * ldy + 4 * r4);
          dy[4 * r4 + 0] = v.x; dy[4 * r4 + 1] = v.y; dy[4 * r4 + 2] = v.z; dy[4 * r4 + 3] = v.w;
        }
        float xv[RK];
#pragma unroll
        for (int i = 0; i < RK; ++i) xv[i] = xb[pp * ldx + 16 * i];
#pragma unroll
        for (int r = 0; r < RN; ++r) {
#pragma unroll
          for (int i = 0; i < RK; ++i) acc[r][i] = fmaf(dy[r], xv[i], acc[r][i]);
          bacc[r] += dy[r];
        }
      }
    }
    __syncthreads();
    buf ^= 1;
  }

  if (!row_active) return;
  const int in_real = g.k_h + g.enc_real;
  const int coff = it.kind == 0 ? it.k0 : g.k_h;
  const int kreal = it.kind == 0 ? it.kblk : g.enc_real;
#pragma unroll
  for (int r = 0; r < RN; ++r) {
    const int n = it.n0 + ty * RN + r;
#pragma unroll
    for (int i = 0; i < RK; ++i) {
      const int k = tx + 16 * i;
      if (k < kreal) atomicAdd(flat_grad + g.flat_w + (size_t)n * in_real + coff + k, acc[r][i]);
    }
    if (it.bias && tx == 0) atomicAdd(flat_grad + g.flat_b + n, bacc[r]);
  }
}

// narrow heads: dW[c][k] = sum_p d_raw[p][out_col + c] * X[p][k]
__device__ __forceinline__ void wgrad_head(const Plan& p, const WgItem& it, const float* __restrict__ d_raw,
                                           const float* __restrict__ stash, int64_t P, int64_t pt_begin,
                                           int64_t pt_end, float* __restrict__ flat_grad) {
  const HeadLayer& h = p.h[it.t];
  const int tid = threadIdx.x;
  const int groups = kThreads / h.k > 0 ? kThreads / h.k : 1;
  const int k = tid % h.k, grp = tid / h.k;
  if (grp >= groups) return;
  const float* X = stash + (size_t)P * p.g[h.src].cum_n;
  const int xw = p.g[h.src].n;
  float acc[4] = {0.f, 0.f, 0.f, 0.f}, bacc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int64_t pt = pt_begin + grp; pt < pt_end; pt += groups) {
    const float4 d = reinterpret_cast<const float4*>(d_raw)[pt];
    const float dv[4] = {d.x, d.y, d.z, d.w};
    const float x = X[(size_t)pt * xw + swz_col(k, pt)];
    for (int c = 0; c < h.n_out; ++c) {
      acc[c] = fmaf(dv[h.out_col + c], x, acc[c]);
      bacc[c] += dv[h.out_col + c];
    }
  }
  for (int c = 0; c < h.n_out; ++c) {
    atomicAdd(flat_grad + h.flat_w + c * h.k + k, acc[c]);
    if (k == 0) atomicAdd(flat_grad + h.flat_b + c, bacc[c]);
  }
}

__global__ void __launch_bounds__(kThreads, 2)
mlp_bwd_wgrad_kernel(const __grid_constant__ Plan p, const float* __restrict__ rays, int ray_stride,
                     const float* __restrict__ z, int S, const float* __restrict__ d_raw,
                     const float* __restrict__ stash, const float* __restrict__ gstash, int64_t P,
                     float* __restrict__ flat_grad) {
  extern __shared__ __align__(16) float smem[];
  const WgItem it = wg_decode(p, blockIdx.y);
  // contiguous point range of this CTA, in units of kWgPts
  const int64_t stages = (P + kWgPts - 1) / kWgPts;
  const int64_t per = (stages + gridDim.x - 1) / gridDim.x;
  const int64_t pt_begin = min(P, (int64_t)blockIdx.x * per * kWgPts);
  const int64_t pt_end = min(P, pt_begin + per * kWgPts);
  if (pt_begin >= pt_end) return;
  if (it.kind == 2) {
    wgrad_head(p, it, d_raw, stash, P, pt_begin, pt_end, flat_grad);
    return;
  }
  const int rk = it.kblk / 16;
#define NB_WG(RN, RK)                                                                                        \
  wgrad_block<RN, RK>(p, it, rays, ray_stride, z, S, stash, gstash, P, pt_begin, pt_end, smem, flat_grad)
  if (it.nblk > 64) {
    switch (rk) {
      case 2: NB_WG(8, 2); break;
      case 3: NB_WG(8, 3); break;
      case 4: NB_WG(8, 4); break;
      case 5: NB_WG(8, 5); break;
      case 6: NB_WG(8, 6); break;
      case 7: NB_WG(8, 7); break;
      default: NB_WG(8, 8); break;
    }
  } else {
    switch (rk) {
      case 2: NB_WG(4, 2); break;
      case 3: NB_WG(4, 3); break;
      case 4: NB_WG(4, 4); break;
      case 5: NB_WG(4, 5); break;
      case 6: NB_WG(4, 6); break;
      case 7: NB_WG(4, 7); break;
      default: NB_WG(4, 8); break;
    }
  }
#undef NB_WG
}

int launch_dgrad_simt(const Plan& p, const float* blob, const float* d_raw, const float* stash, float* gstash,
                      int64_t P, cudaStream_t s) {
  const BwdSmem sm = bwd_smem_layout(p);
  const size_t bytes = (size_t)sm.total_floats * sizeof(float);
  const int64_t tiles = (P + kTileRows - 1) / kTileRows;
  auto kern = p.hidden == 256 ? mlp_bwd_dgrad_kernel<4> : mlp_bwd_dgrad_kernel<2>;
  int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes),
                      "mlp_bwd_dgrad smem attribute");
  if (rc) return rc;
  kern<<<(unsigned)tiles, kThreads, bytes, s>>>(p, sm, blob, d_raw, stash, gstash, P);
  count_launch();
  return check_cuda(cudaGetLastError(), "mlp_bwd_dgrad launch");
}

// every weight-gradient item of wgrad_items.cuh on the CUDA cores
int launch_wgrad_simt(const Plan& p, const float* rays, int ray_stride, const float* z, int n_samples,
                      const float* d_raw, const float* stash, const float* gstash, int64_t P, float* flat_grad,
                      cudaStream_t s) {
  const int n_items = wg_item_count(p);
  const size_t bytes = (size_t)2 * kWgPts * (132 + 132) * sizeof(float);
  int rc = check_cuda(
      cudaFuncSetAttribute(mlp_bwd_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes),
      "mlp_bwd_wgrad smem attribute");
  if (rc) return rc;
  const int64_t stages = (P + kWgPts - 1) / kWgPts;
  const int sms = device_sms();
  int split = (int)((sms * 8 + n_items - 1) / n_items);
  if (split > sms * 8) split = sms * 8;
  if (split > stages) split = (int)stages;
  if (split < 1) split = 1;
  dim3 grid(split, n_items);
  mlp_bwd_wgrad_kernel<<<grid, kThreads, bytes, s>>>(p, rays, ray_stride, z, n_samples, d_raw, stash, gstash, P,
                                                     flat_grad);
  count_launch();
  return check_cuda(cudaGetLastError(), "mlp_bwd_wgrad launch");
}

}  // namespace nerfb200
