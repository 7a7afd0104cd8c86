// mlp_tc.cu -- Hopper tensor-core (wgmma) implementation of the layer-chained forward kernel
//   points -> positional encoding -> FlexibleNeRFModel   (nerf/train_utils.py:67, :8-25; nerf/models.py:233-256)
// (the backward lives in mlp_tc_bwd.cu) for hidden_size 128 (and 256 in inference), fp32-faithful through a 3-term split of every product
//     a * w  ~=  a_hi*w_hi + a_lo*w_hi + a_hi*w_lo          (SURVEY.md section 7.3 item 1)
// on wgmma.mma_async (fp16 operands, K = 16 per instruction, fp32 accumulator): both operands are fp16 pairs
// (hi = fp16(x), lo = fp16((x - hi) 2^11), 22 significant bits, tc_common.cuh split_f16x2); the weights come in three
// pre-scaled copies (hs | h | l, split_w3) so that the three products of a k-step land at the SAME scale 2^11 in ONE
// fp32 accumulator.  The A operand holds activation / 16 (fp16 range 65504 -> 1.05e6: the shipped lego checkpoints
// reach 6e4); conversions do not saturate, an out-of-range value turns the output into inf / NaN instead of clamping.
//
// Persistent kernel, one CTA per SM.  A tile is 64 points per consumer warpgroup: three warpgroups (192 points) for
// hidden 128, one (64 points) for hidden 256, whose 64 x 256 fp32 accumulator takes half of a thread's registers.
// Three warpgroups and the producer warp put four warps on one of the SM's schedulers, whose quarter of the register
// file then allows 128 registers per thread.  The stash keeps 128-point tiles (the fused backward's operand tiles): the
// 64-row block b of a batch is half b & 1 of stash tile b >> 1, whichever CTA tile b / 3 computes it.
//   consumer warpgroups  per tile: positional encodings of its 64 rows -> fp16 operand tile (shared memory); per layer:
//              wgmma over the ring's weight stages (A = the warpgroup's rows of the activation or encoding tile, B =
//              the weight copies), then the epilogue on the accumulator registers: bias at the accumulator's 2^11
//              scale, NaN-propagating max (ReLU), narrow heads as register dot products reduced over the quad, split
//              into fp16 hi + lo (mixed-precision FMA, tc_common.cuh split_f16x2_y) -> the activation tile in shared
//              memory, the next layer's A operand.  Training: the same hi / lo registers also go to the activation
//              stash as an operand tile (tc_common.cuh "Operand tiles"), plus one ReLU bit per activation.
//              The warpgroups run independently on the same weight stages; each one's epilogue overlaps the others'
//              MMAs.
//   last warp  weight producer: fills the weight ring (tc_common.cuh WeightRing) with one cp.async.bulk per stage
//              (12 KB, one N = 128 k-step, at hidden 128: the 192-row tiles leave the ring 48 KB, four stages; 24 KB
//              at hidden 256) from the L2-resident blob, mbarrier complete_tx; a stage is free again once every
//              consumer warp has seen its MMAs complete.
// The direction encoding enters layers_dir[0] through a per-ray fp32 bias computed on the CUDA cores (it is constant
// along a ray: SURVEY.md section 7.3 item 5), so that layer contracts over K = H only.
//
// Single-pass variant (kFast, inference only, impl 3): one wgmma per k-step, a_hi * hs, against the hs = fp16(w) 2^11
// copy the blob already holds, so the accumulator sits at the same 2^11 scale and bias, ReLU, heads and the per-ray
// view bias are unchanged.  Products are fp16(activation / 16) * fp16(w) with fp32 accumulation (~11 significant bits
// per operand instead of 22); the heads and the direction term stay fp32.  The producer streams only the hs part of
// each k-step (32 n bytes, contiguous in the blob) and packs stage bytes / (32 n) k-steps into a ring stage; the
// prologue and the epilogue write only the hi half of the operand tiles.
#include "common.cuh"
#include "tc_common.cuh"

namespace nerfb200 {

namespace tc {
// consumer warpgroups at hidden 128 (-DNERFB200_FWD_WG=2 builds the two-warpgroup shape, for timing one against the other)
#ifndef NERFB200_FWD_WG
#define NERFB200_FWD_WG 3
#endif
constexpr int kFwdWG128 = NERFB200_FWD_WG;
static_assert(kFwdWG128 == 2 || kFwdWG128 == 3, "hidden 128 runs two or three consumer warpgroups");

constexpr int kStepsPerStage = 2;                       // k-steps per ring stage at most (split products)
constexpr int kStageBytes = kStepsPerStage * 96 * 128;  // 24 KB: 3 copies x 2 slabs x 128 rows x 16 B per k-step

__host__ __device__ constexpr int n_wg(int hidden) { return hidden == 128 ? kFwdWG128 : 1; }  // consumer warpgroups = tile / 64
// bytes of a ring stage: 24 KB, or 12 KB (one N = 128 k-step) beside the 192-row tiles of three warpgroups, which leave
// the ring 48 KB: four shallow stages keep more copies in flight than two deep ones
__host__ __device__ constexpr int stage_bytes(int hidden) { return n_wg(hidden) == 3 ? kStageBytes / 2 : kStageBytes; }

// Shared memory map (bytes from the 1 KB-aligned base), computed identically on host and device.
struct SmemMap {
  int act, enc, ring, bias, headw, viewb, encd, wv, bars, total, n_stages;
};
__host__ __device__ inline SmemMap smem_map(const Plan& p) {
  SmemMap m;
  const int rows = 64 * n_wg(p.hidden);
  m.act = 0;                                        // activation operand tile, hi | lo, up to hidden wide
  int off = rows * p.hidden * 4;
  m.enc = off;       off += rows * 64 * 4;          // encoding operand tile, hi | lo (<= 64 wide)
  m.bias = off;      off += p.enc_cum[0] * 4;       // sum of n over the gemm layers (bias * 2048 / 16)
  m.headw = off;     off += (4 * p.hidden + 3 * (p.hidden / 2) + 16) * 4;
  m.viewb = off;     off += n_wg(p.hidden) * kMaxRaysPerTile * (p.hidden / 2) * 4;
  m.encd = off;      off += n_wg(p.hidden) * kMaxRaysPerTile * 32 * 4;
  m.wv = off;        off += 32 * (p.hidden / 2) * 4;  // direction-encoding rows of layers_dir[0]'s weight: Wt[k_h + k][n]
  m.bars = off;      off += 256;
  m.ring = (off + 1023) & ~1023;
  m.n_stages = ring_depth(m.ring, stage_bytes(p.hidden));
  m.total = m.ring + (m.n_stages > 0 ? m.n_stages : 0) * stage_bytes(p.hidden);
  return m;
}

// what the MMAs of layer e contract: weights, shapes
struct MmaInfo {
  const uint8_t* src;   // blob copy of the layer's weights (three fp16 copies, k-step major)
  uint32_t kbytes;      // bytes of one k-step
  int ksteps, ksteps_h; // k-steps, of which the first ksteps_h read the activation tile (the rest: encodings)
  int sps;              // k-steps per ring stage (split_sps, single pass: fast_sps)
};
// split products: k-steps of 96 n bytes per ring stage, two if they fit and one otherwise (24 KB: two at N <= 128, one
// at N = 256; 12 KB: two at N = 64, one at N = 128)
__host__ __device__ constexpr int split_sps(int stage, int n) { return n > stage / (96 * kStepsPerStage) ? 1 : kStepsPerStage; }
// single pass: k-steps per ring stage, each the 32 n bytes of its hs copy (24 KB: 12 at N = 64, 6 at 128, 3 at 256)
__host__ __device__ constexpr int fast_sps(int stage, int n) { return stage / (32 * n); }
__device__ __forceinline__ MmaInfo mma_info(const Plan& p, const float* blob, int e, bool fast, int stage) {
  MmaInfo mi;
  const GemmLayer& g = p.g[e];
  mi.src = reinterpret_cast<const uint8_t*>(blob + g.tc_off);
  mi.ksteps = (g.k_tc + 15) >> 4;
  mi.ksteps_h = g.k_h >> 4;
  mi.kbytes = 96u * (uint32_t)g.n;
  mi.sps = fast ? fast_sps(stage, g.n) : split_sps(stage, g.n);
  return mi;
}

}  // namespace tc

using namespace tc;

// One layer of one warpgroup: MMAs over the ring, then the epilogue on the accumulator fragment.
// Fragment of wgmma m64nN (per warp 16 rows): thread (warp wi, lane) holds rows r = 16 wi + lane / 4 (+ 8) and columns
// 8 j + 2 (lane % 4) + {0, 1}: acc[4 j + 2 i + c] = (row r + 8 i, column 8 j + 2 (lane % 4) + c).
// kStage: bytes of a ring stage.  blk (kTrain): the warpgroup's 64-row block of the batch, whose rows are half blk & 1 of
// stash tile blk >> 1.
// kGrad (the density-gradient kernel's trunk, below): the ReLU bits go to the warpgroup's shared-memory masks s_mask
// ([64 rows][mask_words], layer e at word g.mask_cum) instead of a stash, and the head writes raw sigma alone, to
// column 0 of raw.  Every other instance compiles without these paths.
template <bool kTrain, bool kFast, int N, int kStage, bool kGrad = false>
__device__ __forceinline__ void fwd_layer(const Plan& p, const float* blob, float* __restrict__ raw, float* __restrict__ stash,
                                          uint8_t* sm, const SmemMap& mp, int e, int wg, int rows, int64_t blk,
                                          int64_t P_pad, const RowState& rs, WeightRing<kStage>& ring, const float* s_bias,
                                          const float* s_headw, const float* s_headb, const float* viewb, int hw1,
                                          uint32_t* s_mask = nullptr, int mask_words = 0) {
  static_assert(!(kTrain && kFast), "the single-pass forward is inference only");
  static_assert(!(kGrad && (kTrain || kFast)), "the density gradient runs the split-precision inference trunk");
  // k-steps a ring stage can hold (the unrolled bound; 24 KB stages keep two for every width, mi.sps decides at run time)
  constexpr int kSps = kFast ? fast_sps(kStage, N) : kStage == kStageBytes ? kStepsPerStage : split_sps(kStage, N);
  const int wt = threadIdx.x & 127, wi = wt >> 5, lane = wt & 31, q = lane & 3;
  const GemmLayer& g = p.g[e];
  const MmaInfo mi = mma_info(p, blob, e, kFast, kStage);
  const int enc_w = p.enc_tile_w;
  const uint32_t act_a = smem_u32(sm + mp.act), enc_a = smem_u32(sm + mp.enc);
  const int fin = g.k_h > 0 ? g.k_h : 16;
  // this warpgroup's 64 rows of the K-major operand tiles (SBO = next 8 points, LBO = next 8 features)
  const uint64_t a_hi0 = make_desc(act_a + (uint32_t)(wg * 64 * fin * 2), 128, (uint32_t)fin * 16);
  const uint32_t a_lo_off = (uint32_t)(rows * fin * 2);
  const uint64_t e_hi0 = make_desc(enc_a + (uint32_t)(wg * 64 * enc_w * 2), 128, (uint32_t)enc_w * 16);
  const uint32_t e_lo_off = (uint32_t)(rows * enc_w * 2);
  const uint32_t slab_b = 16u * (uint32_t)N;
  const uint64_t b_ring = make_desc(ring.base, slab_b, 128);

  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  wgmma_fence();
  for (int ks0 = 0; ks0 < mi.ksteps; ks0 += mi.sps) {
    const uint32_t st = ring.acquire();
    const uint64_t b_st = desc_adv(b_ring, st * (uint32_t)kStage);
#pragma unroll
    for (int hh = 0; hh < kSps; ++hh) {
      const int ks = ks0 + hh;
      if (hh < mi.sps && ks < mi.ksteps) {
        // a stage holds per k-step [hs | h | l][2 slabs], or [hs][2 slabs] alone in the single pass
        const uint64_t b_hs = desc_adv(b_st, hh * (kFast ? 2 : 6) * slab_b);
        uint64_t ah, al;
        if (ks < mi.ksteps_h) {
          ah = desc_adv(a_hi0, (uint32_t)ks * 256u);
          al = desc_adv(ah, a_lo_off);
        } else {
          ah = desc_adv(e_hi0, (uint32_t)(ks - mi.ksteps_h) * 256u);
          al = desc_adv(ah, e_lo_off);
        }
        wgmma_f16<N>(acc, ah, b_hs, ks > 0 ? 1 : 0);
        if (!kFast) {
          const uint64_t b_h = desc_adv(b_hs, 2 * slab_b), b_l = desc_adv(b_hs, 4 * slab_b);
          wgmma_f16<N>(acc, al, b_h, 1);
          wgmma_f16<N>(acc, ah, b_l, 1);
        }
      }
    }
    wgmma_commit();
    ring.release_behind(acc);
  }
  ring.release_last(acc);

  // ---------------- epilogue ----------------
  const int wg_bar_id = 1 + wg;
  asm volatile("bar.sync %0, 128;" ::"r"(wg_bar_id) : "memory");  // every warp's MMAs have read the activation tile
  const bool has_next = e + 1 < p.n_gemm;
  const int hsel = head_of(p, e);
  const float* hw = hsel == 1 ? s_headw + hw1 : s_headw;
  const int hk = hsel >= 0 ? p.h[hsel].k : 0, hn = hsel >= 0 ? p.h[hsel].n_out : 0;
  const bool is_dir = p.use_viewdirs && e == p.n_gemm - 1;
  const float lb = g.relu ? 0.f : -3.4e38f;
  const int vbs = p.hidden / 2;
  const float* brow[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) brow[i] = is_dir ? viewb + rs.ray_slot[i] * vbs : s_bias + g.cum_n;
  float hacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  uint32_t mbits[2][N / 32];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int m = 0; m < N / 32; ++m) mbits[i][m] = 0u;
  uint8_t* act = sm + mp.act;
  const int act_lo = rows * N * 2;
  // the stash tile's hi block, moved so that the shared-memory tile's offsets (rows 64 wg ...) land on rows 64 (blk & 1) ...:
  // 64 rows of a hi block are 128 N bytes
  uint8_t* st_hi = nullptr;
  if (kTrain)
    st_hi = reinterpret_cast<uint8_t*>(stash + (size_t)P_pad * g.cum_n) + (size_t)(blk >> 1) * tile_bytes(N) +
            ((int)(blk & 1) - wg) * (128 * N);
  const int r0 = 64 * wg + 16 * wi + (lane >> 2);  // tile row of acc row 0 (row 1: + 8)

#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int col = 8 * j + 2 * q;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float2 b = *reinterpret_cast<const float2*>(brow[i] + col);
      const float Y0 = fmax_nan(acc[4 * j + 2 * i] + b.x, lb), Y1 = fmax_nan(acc[4 * j + 2 * i + 1] + b.y, lb);
      const float x0 = Y0 * kLoInv, x1 = Y1 * kLoInv;
      if (hn > 0) {
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < hn) {
            const float2 w = *reinterpret_cast<const float2*>(hw + c * hk + col);
            hacc[i][c] = fmaf(x0, w.x, fmaf(x1, w.y, hacc[i][c]));
          }
      }
      if (kTrain || kGrad)  // ReLU bits (Y >= 0 here: Y > 0 <=> a nonzero bit pattern)
        mbits[i][j >> 2] |= (min(__float_as_uint(Y0), 1u) | (min(__float_as_uint(Y1), 1u) << 1)) << (8 * (j & 3) + 2 * q);
      if (kFast) {
        if (has_next)
          *reinterpret_cast<uint32_t*>(act + tile_piece(r0 + 8 * i, j, N) + q * 4) = f16x2_hi(x0, x1);
      } else if (has_next || kTrain) {
        uint32_t hi, lo;
        split_f16x2_y(Y0, Y1, x0, x1, hi, lo);
        const int off = tile_piece(r0 + 8 * i, j, N) + q * 4;
        if (has_next) {
          *reinterpret_cast<uint32_t*>(act + off) = hi;
          *reinterpret_cast<uint32_t*>(act + act_lo + off) = lo;
        }
        if (kTrain) {
          __stcs(reinterpret_cast<unsigned int*>(st_hi + off), hi);
          __stcs(reinterpret_cast<unsigned int*>(st_hi + tile_half_bytes(N) + off), lo);
        }
      }
    }
  }
  if (has_next) {
    fence_proxy_async();  // generic-proxy stores -> the next layer's wgmma reads them through the async proxy
    asm volatile("bar.sync %0, 128;" ::"r"(wg_bar_id) : "memory");
  }
  if (kTrain) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int m = 0; m < N / 32; ++m) {
        uint32_t w = mbits[i][m];
        w |= __shfl_xor_sync(0xffffffffu, w, 1);
        w |= __shfl_xor_sync(0xffffffffu, w, 2);
        if ((m & 3) == q && rs.valid[i])
          reinterpret_cast<uint32_t*>(stash)[(size_t)P_pad * (p.mask_base + g.mask_cum) + (size_t)rs.pt[i] * (N >> 5) + m] = w;
      }
    }
  }
  if (kGrad) {  // the same bits into this warpgroup's shared-memory masks (row-local; read back by the reverse chain)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int m = 0; m < N / 32; ++m) {
        uint32_t w = mbits[i][m];
        w |= __shfl_xor_sync(0xffffffffu, w, 1);
        w |= __shfl_xor_sync(0xffffffffu, w, 2);
        if ((m & 3) == q) s_mask[(16 * wi + (lane >> 2) + 8 * i) * mask_words + g.mask_cum + m] = w;
      }
    }
  }
  if (hsel >= 0) {
    const int hcol = p.h[hsel].out_col;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        hacc[i][c] += __shfl_xor_sync(0xffffffffu, hacc[i][c], 1);
        hacc[i][c] += __shfl_xor_sync(0xffffffffu, hacc[i][c], 2);
      }
      if (kGrad) {  // raw sigma: output column 3 of the trunk's head (fc_alpha, or fc_out without view directions)
        if (q == 0 && rs.valid[i])
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (c < hn && hcol + c == 3) raw[(int64_t)rs.pt[i] * 4] = hacc[i][c] + s_headb[hsel * 4 + c];
      } else if (q == 0 && rs.valid[i])
        for (int c = 0; c < hn; ++c) raw[(int64_t)rs.pt[i] * 4 + hcol + c] = hacc[i][c] + s_headb[hsel * 4 + c];
    }
  }
}

// kTrain: the forward also writes the activation stash (operand tiles + ReLU bit masks + the encoding tile).
// kH = hidden size (compile-time: the accumulator width and the warpgroup count fold into constants)
// kFast: the single-pass fp16 products (inference only, see the file header)
// kPts: the points come from pts[P][3] and the view directions from (dirs, dir_stride) instead of o + d z and the ray
// rows' columns 8..10 (a template parameter, so that the render path's instances compile as they did without it)
// kMap: inference over an occupancy grid's row map (occupancy.cu): tile rows are map rows, row -> point through map[],
// each 64-row block's rays from blocks[], and the tile count from *n_blocks in device memory.  Every row is computed as
// the default instance computes its point, so an evaluated point's raw has the same bits.
template <bool kTrain, int kH, bool kFast, bool kPts, bool kMap>
__global__ void __launch_bounds__(128 * n_wg(kH) + 32, 1)
mlp_fwd_tc_kernel(const __grid_constant__ Plan p, const float* __restrict__ blob, const float* __restrict__ rays,
                  int ray_stride, const float* __restrict__ z, int64_t P, int S, int64_t n_tiles,
                  float* __restrict__ raw,          // out [P][4]
                  float* __restrict__ stash,        // out (kTrain)
                  const float* __restrict__ pts, const float* __restrict__ dirs, int dir_stride,  // kPts
                  const int* __restrict__ map, const int2* __restrict__ blocks, const int* __restrict__ n_blocks,  // kMap
                  int64_t stash_tiles) {  // kTrain: 128-point tiles of the stash, ceil(P / 128)
  static_assert(!(kMap && (kTrain || kPts)), "the row map is an inference path of the render points");
  constexpr int kWG = n_wg(kH), kRows = 64 * kWG, kThreads = 128 * kWG + 32, kStage = stage_bytes(kH);
  using Ring = WeightRing<kStage>;
  uint8_t* sm = smem_base();
  const SmemMap mp = smem_map(p);
  float* s_bias = reinterpret_cast<float*>(sm + mp.bias);
  float* s_headw = reinterpret_cast<float*>(sm + mp.headw);
  float* s_viewb = reinterpret_cast<float*>(sm + mp.viewb);
  float* s_encd = reinterpret_cast<float*>(sm + mp.encd);
  float* s_wv = reinterpret_cast<float*>(sm + mp.wv);
  Ring ring{smem_u32(sm + mp.ring), smem_u32(sm + mp.bars), (uint32_t)mp.n_stages};

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // warp-uniform for ptxas: the role branches hold the wgmma
  const int64_t P_pad = stash_tiles * kTileRows;   // the stash sections are sized in 128-point tiles
  const int enc_w = p.enc_tile_w;                  // encoding operand tile width (dim_xyz padded to 16)

  if (tid == 0) {
    ring.init(4 * kWG);
    fence_barrier_init();
  }
  // biases (/16) + head weights (x16, they multiply activation / 16): once per CTA
  for (int gi = 0; gi < p.n_gemm; ++gi)
    for (int i = tid; i < p.g[gi].n; i += kThreads) s_bias[p.g[gi].cum_n + i] = blob[p.g[gi].b_off + i] * (kActScale * kLoScale);
  const int hw1 = p.h[0].n_out * p.h[0].k;
  const int hw2 = p.n_head > 1 ? p.h[1].n_out * p.h[1].k : 0;
  for (int i = tid; i < hw1; i += kThreads) s_headw[i] = blob[p.h[0].w_off + i] * kActInv;
  for (int i = tid; i < hw2; i += kThreads) s_headw[hw1 + i] = blob[p.h[1].w_off + i] * kActInv;
  float* s_headb = s_headw + ((hw1 + hw2 + 3) & ~3);
  if (tid < 4) s_headb[tid] = blob[p.h[0].b_off + tid];
  if (tid >= 4 && tid < 8) s_headb[tid] = p.n_head > 1 ? blob[p.h[1].b_off + tid - 4] : 0.f;
  for (int i = tid; i < kWG * kMaxRaysPerTile * 32; i += kThreads) s_encd[i] = 0.f;  // padding channels stay zero
  if (p.use_viewdirs) {
    const GemmLayer& gd = p.g[p.n_gemm - 1];
    const float* wv_g = blob + gd.wt_off + (size_t)gd.k_h * gd.n;  // rows k_h.. of Wt[k][n]
    for (int i = tid; i < p.dim_dir * gd.n; i += kThreads) s_wv[i] = wv_g[i];
  }
  __syncthreads();

  if constexpr (kMap) n_tiles = ((int64_t)*n_blocks + kWG - 1) / kWG;
  const int my_tiles = (n_tiles > blockIdx.x) ? (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;

  if (warp == 4 * kWG) {
    // ===================== weight producer =====================
    if ((tid & 31) == 0) {
      const uint64_t pol = l2_policy_evict_last();
      for (int j = 0; j < my_tiles; ++j)
        for (int e = 0; e < p.n_gemm; ++e) {
          const MmaInfo mi = mma_info(p, blob, e, kFast, kStage);
          for (int ks = 0; ks < mi.ksteps; ks += mi.sps) {
            const uint32_t nk = (uint32_t)min(mi.sps, mi.ksteps - ks);
            const uint8_t* src = mi.src + (size_t)ks * mi.kbytes;
            if (kFast)  // the hs part of each k-step: one bulk copy each
              ring.fill(src, nk, mi.kbytes / 3, mi.kbytes, pol);
            else        // the k-steps' three copies are contiguous in the blob: one bulk copy
              ring.fill(src, 1, nk * mi.kbytes, 0, pol);
          }
        }
    }
  } else {
    // ===================== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of every tile =====================
    const int wg = warp >> 2, wt = tid & 127;
    const int row = wt & 63, half = wt >> 6;       // prologue: two threads per row split the frequencies
    const int vbs = kH / 2;
    float* viewb = s_viewb + wg * kMaxRaysPerTile * vbs;
    float* encd = s_encd + wg * kMaxRaysPerTile * 32;
    uint8_t* enc = sm + mp.enc;
    const int enc_hb = kRows * enc_w * 2;          // bytes of the hi (or lo) block of the encoding tile
    auto wg_bar = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); };
#pragma unroll 1
    for (int j = 0; j < my_tiles; ++j) {
      const int64_t tile = blockIdx.x + (int64_t)j * gridDim.x;
      const int64_t p0 = tile * kRows + 64 * wg;   // first point (kMap: first map row) of this warpgroup's 64-row block
      // kTrain: the block is one half of a 128-point stash tile.  A block past P inside the last stash tile fills its
      // half from the last point, so the backward reads whole tiles.  A block past the last stash tile (the end of the
      // last CTA tile) has nowhere to write: its warpgroup runs the layers as the inference forward does, which keeps it
      // walking the weight ring with the others, and every row of it is invalid.
      const int64_t blk = p0 >> 6;
      const bool stashes = kTrain && (blk >> 1) < stash_tiles;
      TileRays tr;
      RowState rs;
      bool block_live = true;                      // kMap: this warpgroup's 64-row block exists
      if constexpr (kMap) {
        block_live = (p0 >> 6) < *n_blocks;        // an odd block count leaves the last tile's second half empty
        const int2 b = block_live ? blocks[p0 >> 6] : make_int2(0, 0);
        tr.first = b.x;
        tr.n = b.y - b.x + 1;
        rs = map_row_state(map, p0, 16 * (wt >> 5) + ((tid & 31) >> 2), block_live, S, tr.first);
      } else {
        tr = tile_rays(p0, 64, P, S);
        rs = row_state(p0, 16 * (wt >> 5) + ((tid & 31) >> 2), P, S, tr.first);
      }
      const int64_t first_ray = tr.first;
      const int n_rays_wg = tr.n;
      // ================= encodings of this row -> operand tile (value / 16), the two halves split the frequencies
      if (kTrain) {  // the previous tile's encoding store must have finished reading the tile
        if (wt == 0) bulk_wait_read();
        wg_bar();
      }
      {
        int64_t pt;
        if constexpr (kMap) {  // a padding row encodes the block's first ray's first point; its raw is never written
          const int m = block_live ? map[p0 + row] : -1;
          pt = m >= 0 ? m : first_ray * S;
        } else {
          pt = (p0 + row < P) ? p0 + row : P - 1;
        }
        const int64_t ray = (int64_t)((uint32_t)pt / (uint32_t)S);
        const float* rr = rays + ray * ray_stride;
        const float zz = kPts ? 0.f : z[pt];
        const int nf = p.n_freq_xyz, mid = nf >> 1;
        const int f0 = half ? mid : 0, f1 = half ? nf : mid;
        const int base = p.inc_xyz ? 3 : 0;
        const int trow = 64 * wg + row;
        auto put = [&](int k, float v) {
          uint32_t hi, lo = 0;
          if (kFast)
            hi = f16x2_hi(v * kActScale, 0.f);
          else
            split_f16x2(v * kActScale, 0.f, hi, lo);  // this element in the low halves
          const int off = tile_piece(trow, k >> 3, enc_w) + (k & 7) * 2;
          *reinterpret_cast<uint16_t*>(enc + off) = (uint16_t)hi;
          if (!kFast) *reinterpret_cast<uint16_t*>(enc + enc_hb + off) = (uint16_t)lo;
        };
        for (int c = 0; c < 3; ++c) {
          // pts = ro + rd * z (train_utils.py:67), or the caller's point
          const float x = kPts ? pts[pt * 3 + c] : __fadd_rn(rr[c], __fmul_rn(rr[3 + c], zz));
          if (p.inc_xyz && half == 0) put(c, x);
          for (int f = f0; f < f1; ++f) {
            float sn, cs;
            sincosf(__fmul_rn(x, p.freq_xyz[f]), &sn, &cs);
            put(base + 6 * f + c, sn);
            put(base + 6 * f + 3 + c, cs);
          }
        }
        if (half == 1)  // zero padding up to the operand width (one fp16 k-step = 16 granular)
          for (int k = p.dim_xyz; k < enc_w; ++k) put(k, 0.f);
      }
      // ---- per-ray direction term of layers_dir[0]: vb[ray][n] = (sum_k enc_dir(ray)[k] * W[n][H + k] + b[n]) / 16
      if (p.use_viewdirs) {
        if (wt < n_rays_wg * 3) {
          const int jr = wt / 3, c = wt - 3 * jr;
          const float v = kPts ? dirs[(first_ray + jr) * dir_stride + c] : rays[(first_ray + jr) * ray_stride + 8 + c];
          encode_coord(v, c, p.inc_dir, 0, p.n_freq_dir, p.freq_dir, encd + jr * 32);
        }
        wg_bar();
        const GemmLayer& gd = p.g[p.n_gemm - 1];
        for (int i = wt; i < n_rays_wg * gd.n; i += 128) {
          const int jr = i / gd.n, n = i - jr * gd.n;
          float a = 0.f;
          for (int k = 0; k < p.dim_dir; ++k) a = fmaf(encd[jr * 32 + k], s_wv[k * gd.n + n], a);
          viewb[jr * vbs + n] = fmaf(a, kActScale * kLoScale, s_bias[gd.cum_n + n]);  // per-ray bias of layers_dir[0] (x 2048 / 16)
        }
      }
      fence_proxy_async();  // the tile was written through the generic proxy; wgmma / the bulk store read it via the async proxy
      wg_bar();             // also publishes viewb
      if (stashes && wt == 0) {  // this warpgroup's rows of the encoding tile go to the stash as they are:
        // two bulk stores into half blk & 1 of stash tile blk >> 1 (64 rows of a hi or lo block are contiguous)
        uint8_t* dst = reinterpret_cast<uint8_t*>(stash + (size_t)P_pad * p.enc_cum[0]) + (size_t)(blk >> 1) * tile_bytes(enc_w);
        const int part = enc_hb / kWG, dpart = (int)(blk & 1) * part;
        bulk_s2g(dst + dpart, enc + wg * part, (uint32_t)part);
        bulk_s2g(dst + tile_half_bytes(enc_w) + dpart, enc + enc_hb + wg * part, (uint32_t)part);
      }
#pragma unroll 1
      for (int e = 0; e < p.n_gemm; ++e) {
        auto layer = [&](auto train, auto width) {
          fwd_layer<decltype(train)::value, kFast, decltype(width)::value, kStage>(
              p, blob, raw, stash, sm, mp, e, wg, kRows, blk, P_pad, rs, ring, s_bias, s_headw, s_headb, viewb, hw1);
        };
        using std::bool_constant;
        using std::integral_constant;
        if (p.g[e].n == kH) {
          if (stashes || !kTrain) layer(bool_constant<kTrain>{}, integral_constant<int, kH>{});
          else layer(bool_constant<false>{}, integral_constant<int, kH>{});
        } else {
          if (stashes || !kTrain) layer(bool_constant<kTrain>{}, integral_constant<int, kH / 2>{});
          else layer(bool_constant<false>{}, integral_constant<int, kH / 2>{});
        }
      }
    }
    if (kTrain && wt == 0) bulk_wait_all();  // this warpgroup's encoding-tile stores
  }
}

// training = the forward must also write the activation stash for the fused backward (hidden 128 only); the
// inference forwards also run hidden 256 (one warpgroup, 64-point tiles, N = 256 MMAs).  The single-pass forward
// (impl 3) is accepted exactly where the inference forward is.  `what` names the call and the impl.
int tc_supported(const Plan& p, int n_samples, bool training, const char* what) {
  if (p.hidden != 128 && (training || p.hidden != 256)) {
    set_error("%s: hidden_size %d not supported (training: 128 only; inference: 128 or 256); use impl=0", what,
              p.hidden);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (p.dim_xyz_pad > 64 || p.dim_dir > 32) {
    set_error("%s: encodings wider than 64 (xyz) / 32 (dir) not supported; use impl=0", what);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (n_samples > 0 && (kTileRows + n_samples - 1) / n_samples + 1 > kMaxRaysPerTile) {
    set_error("%s: fewer than 15 samples per ray not supported; use impl=0", what);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (smem_map(p).n_stages < 2) {
    set_error("%s: network too deep for the shared-memory budget (%d layers); use impl=0", what, p.n_gemm);
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

template <bool kTrain, int kH, bool kFast>
static int launch_fwd(const Plan& p, const float* blob, const PointSrc& src, int64_t P, int n_samples, float* raw,
                      float* stash, cudaStream_t s, const char* what) {
  constexpr int kRows = 64 * n_wg(kH), kThreads = 2 * kRows + 32;
  const int64_t stash_tiles = (P + kTileRows - 1) / kTileRows;  // the stash keeps 128-point tiles whatever the CTA tile
  // training covers both halves of every stash tile, the last one's second half too when it lies past P
  const int64_t tiles = ((kTrain ? stash_tiles * kTileRows : P) + kRows - 1) / kRows;
  auto kern = src.pts ? mlp_fwd_tc_kernel<kTrain, kH, kFast, true, false>
                      : mlp_fwd_tc_kernel<kTrain, kH, kFast, false, false>;
  return launch_persistent(kern, tiles, kThreads, smem_map(p).total, s, what, p, blob, src.rays, src.ray_stride, src.z, P,
                           n_samples, tiles, raw, stash, src.pts, src.dirs, src.dir_stride, (const int*)nullptr,
                           (const int2*)nullptr, (const int*)nullptr, stash_tiles);
}

// over a row map: the grid covers max_blocks blocks; the kernel reads the live count from m.n_blocks
template <int kH, bool kFast>
static int launch_fwd_map(const Plan& p, const float* blob, const float* rays, int ray_stride, const float* z,
                          int64_t P, int n_samples, const RowMap& m, int64_t max_blocks, float* raw, cudaStream_t s,
                          const char* what) {
  constexpr int kWG = n_wg(kH), kThreads = 128 * kWG + 32;
  const int64_t tiles = (max_blocks + kWG - 1) / kWG;
  return launch_persistent(mlp_fwd_tc_kernel<false, kH, kFast, false, true>, tiles, kThreads, smem_map(p).total, s, what,
                           p, blob, rays, ray_stride, z, P, n_samples, tiles, raw, (float*)nullptr,
                           (const float*)nullptr, rays + 8, ray_stride, m.map, m.blocks, m.n_blocks, (int64_t)0);
}

int launch_mlp_fwd_tc_map(const Plan& p, const float* blob, const float* rays, int ray_stride, const float* z,
                          int64_t n_rays, int n_samples, const RowMap& m, int64_t max_blocks, float* raw, bool fast,
                          cudaStream_t s) {
  const int64_t P = n_rays * n_samples;
  auto go = [&](auto launch, const char* what) {
    return launch(p, blob, rays, ray_stride, z, P, n_samples, m, max_blocks, raw, s, what);
  };
  if (fast)
    return go(p.hidden == 256 ? launch_fwd_map<256, true> : launch_fwd_map<128, true>, "mlp_fwd_tc_fast grid launch");
  return go(p.hidden == 256 ? launch_fwd_map<256, false> : launch_fwd_map<128, false>, "mlp_fwd_tc grid launch");
}

// stash non-null: the training forward; fast: the single-pass forward (never with a stash)
int launch_mlp_fwd_tc(const Plan& p, const float* blob, const PointSrc& src, int64_t n_rays, int n_samples, float* raw,
                      float* stash, bool fast, cudaStream_t s) {
  auto go = [&](auto launch, const char* what) {
    return launch(p, blob, src, n_rays * n_samples, n_samples, raw, stash, s, what);
  };
  if (stash) return go(launch_fwd<true, 128, false>, "mlp_fwd_tc launch");
  if (fast)
    return go(p.hidden == 256 ? launch_fwd<false, 256, true> : launch_fwd<false, 128, true>, "mlp_fwd_tc_fast launch");
  return go(p.hidden == 256 ? launch_fwd<false, 256, false> : launch_fwd<false, 128, false>, "mlp_fwd_tc launch");
}


// ---------------------------------------------------------------------------------------------------------------
// Density gradient (nerfb200.h "density gradient"): sigma_raw and d sigma_raw / d x at a flat list of points, x in the
// coordinates the MLP encodes.  A kernel of its own beside mlp_fwd_tc_kernel, so that the forward's instances stay as
// they are: its trunk is fwd_layer<..., kGrad> (the forward's encoding, operand split, MMAs and epilogue, so sigma has
// the forward's bits), which keeps each layer's ReLU bits in shared memory.  Then, per 64-row block, the reverse chain
//     G_{L-1} = w_sigma (.) mask_{L-1},    G_{t-1} = (G_t W_t[:, :H]) (.) mask_{t-1}     (layer1 has no ReLU: no mask)
// on wgmma with the three-term split -- A = G_t / 16, split hi / lo into the activation tile's place; B = the blob's
// transposed dgrad copies (tcd_off), as the fused backward's chain_mma reads them -- and the encoding gradient
//     d_enc = sum over the layers that read the xyz encoding (layer1, the skip layers) of G_t W_t[:, enc]
// against the forward's own weight copies read MN-major: one 16-column k-step of the encoding per ring stage, N = 16
// MMAs into register accumulators that live through the chain.  The epilogue takes d_enc through the positional
// encoding to x.  No view direction, fc_feat, layers_dir or fc_rgb runs; HBM traffic is the points in and 16 B out.
// ---------------------------------------------------------------------------------------------------------------
namespace tc {
// consumer warpgroups: two at hidden 128 (the chain accumulator and the encoding-gradient accumulators are live
// together, which the 128 registers per thread of three warpgroups do not hold), one at 256
__host__ __device__ constexpr int grad_wg(int hidden) { return hidden == 128 ? 2 : 1; }
constexpr int kMaxEncSteps = 4;  // 16-column k-steps of the xyz encoding (tc_supported: at most 64 wide)

struct GradSmemMap {
  SmemMap m;       // act (the G tile once the trunk has run), enc, bias, headw, bars and ring, as fwd_layer reads them
  int mask;        // the trunk's ReLU bits: [warpgroup][64 rows][mask_words]
  int mask_words;  // per row: the sum over the trunk of n / 32
};
__host__ __device__ inline GradSmemMap grad_smem_map(const Plan& p) {
  GradSmemMap gm;
  SmemMap& m = gm.m;
  const int rows = 64 * grad_wg(p.hidden);
  gm.mask_words = 0;
  for (int t = 0; t < p.n_trunk; ++t) gm.mask_words += p.g[t].n / 32;
  m.act = 0;
  int off = rows * p.hidden * 4;
  m.enc = off;    off += rows * 64 * 4;
  m.bias = off;   off += p.enc_cum[0] * 4;
  m.headw = off;  off += (4 * p.hidden + 3 * (p.hidden / 2) + 16) * 4;
  gm.mask = off;  off += rows * gm.mask_words * 4;
  m.viewb = m.encd = m.wv = 0;  // no view directions
  m.bars = off;   off += 256;
  m.ring = (off + 1023) & ~1023;
  m.n_stages = ring_depth(m.ring, kStageBytes);
  m.total = m.ring + (m.n_stages > 0 ? m.n_stages : 0) * kStageBytes;
  return gm;
}
}  // namespace tc

// G_t of this thread's fragment (y at the accumulator's 2^11 scale, G / 16) (.) the ReLU bits of layer t (none without
// a ReLU) -> hi / lo -> the warpgroup's rows of the activation tile, the K-major A operand of the next MMAs.
// mrow[i]: the mask row of accumulator row i; r0: tile row of accumulator row 0.
template <int N>
__device__ __forceinline__ void grad_g_store(const Plan& p, const float (&y)[N / 2], int t, uint8_t* act, int rows,
                                             const uint32_t* const (&mrow)[2], int r0) {
  const int q = threadIdx.x & 3;
  const GemmLayer& g = p.g[t];
  const int act_lo = rows * N * 2;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t word = g.relu ? mrow[i][g.mask_cum + (j >> 2)] : 0xFFFFFFFFu;
      const int bit = 8 * (j & 3) + 2 * q;
      const float Y0 = (word & (1u << bit)) ? y[4 * j + 2 * i] : 0.f;
      const float Y1 = (word & (2u << bit)) ? y[4 * j + 2 * i + 1] : 0.f;
      uint32_t hi, lo;
      split_f16x2_y(Y0, Y1, Y0 * kLoInv, Y1 * kLoInv, hi, lo);
      const int off = tile_piece(r0 + 8 * i, j, N) + q * 4;
      *reinterpret_cast<uint32_t*>(act + off) = hi;
      *reinterpret_cast<uint32_t*>(act + act_lo + off) = lo;
    }
  }
}

// acc = 2^11 G_t W_t[:, :N] of this warpgroup's rows: A = the G tile (a_hi, lo block a_lo_off on), B = layer t's tcd
// copy, one k-step (16 n x all N columns: [hs | h | l][slab 0 | 1][k][8 n]) per ring stage
template <int N, int kStage>
__device__ __forceinline__ void grad_chain_mma(float (&acc)[N / 2], WeightRing<kStage>& ring, uint64_t a_hi,
                                               uint32_t a_lo_off) {
  const uint32_t slab = 16u * N;
  const uint64_t b_ring = make_desc(ring.base, slab, 128);
  wgmma_fence();
#pragma unroll 1
  for (int ks = 0; ks < N / 16; ++ks) {
    const uint32_t st = ring.acquire();
    const uint64_t b = desc_adv(b_ring, st * (uint32_t)kStage);
    const uint64_t ah = desc_adv(a_hi, (uint32_t)ks * 256u);
    wgmma_f16<N>(acc, ah, b, ks > 0 ? 1 : 0);
    wgmma_f16<N>(acc, desc_adv(ah, a_lo_off), desc_adv(b, 2 * slab), 1);
    wgmma_f16<N>(acc, ah, desc_adv(b, 4 * slab), 1);
    wgmma_commit();
    ring.release_behind(acc);
  }
  ring.release_last(acc);
}

// acc_e[c] += 2^11 G_t W_t[:, k_h + 16 c .. + 16] for the nch encoding k-steps of layer t: B = the forward copy's k-step
// k_h / 16 + c ([hs | h | l][slab 0 | 1][n][8 k]) read MN-major -- the n rows are K (8-deep groups 128 B apart), the
// two slabs the two 8-wide column groups (16 N bytes apart)
template <int N, int kStage>
__device__ __forceinline__ void grad_enc_mma(float (&acc_e)[kMaxEncSteps][8], WeightRing<kStage>& ring, uint64_t a_hi,
                                             uint32_t a_lo_off, int nch) {
  const uint32_t slab = 16u * N;
  const uint64_t b_ring = make_desc(ring.base, 128, slab);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < kMaxEncSteps; ++c) {
    if (c < nch) {
      const uint32_t st = ring.acquire();
      const uint64_t b_st = desc_adv(b_ring, st * (uint32_t)kStage);
#pragma unroll 4
      for (int ks = 0; ks < N / 16; ++ks) {
        const uint64_t ah = desc_adv(a_hi, (uint32_t)ks * 256u), b = desc_adv(b_st, (uint32_t)ks * 256u);
        wgmma_f16<16, 0, 1>(acc_e[c], ah, b, 1);
        wgmma_f16<16, 0, 1>(acc_e[c], desc_adv(ah, a_lo_off), desc_adv(b, 2 * slab), 1);
        wgmma_f16<16, 0, 1>(acc_e[c], ah, desc_adv(b, 4 * slab), 1);
      }
      wgmma_commit();
      ring.release_behind(acc_e[c]);
    }
  }
  ring.release_last(acc_e[0]);  // waits for every group; the other chunks are fenced before they are read
}

// d_enc (acc_e: 2^11 / 16 times its value) -> d sigma / d x of this thread's two rows through the positional encoding
// (x itself, then f cos(f x) and -f sin(f x) per band, the bands' arguments rounded as the forward rounds them),
// summed over the quad and written beside sigma
__device__ __forceinline__ void grad_x_store(const Plan& p, const float (&acc_e)[kMaxEncSteps][8], int nch,
                                             const float* __restrict__ pts, float* __restrict__ out, const RowState& rs) {
  const int q = threadIdx.x & 3;
  const int base = p.inc_xyz ? 3 : 0;
  float x[2][3], gx[2][3];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      x[i][c] = pts[(int64_t)rs.pt[i] * 3 + c];
      gx[i][c] = 0.f;
    }
#pragma unroll
  for (int ch = 0; ch < kMaxEncSteps; ++ch) {
    if (ch < nch) {
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const int k = 16 * ch + 8 * j + 2 * q + cc;
          if (k < p.dim_xyz) {
            const int kk = k - base, f = kk >= 0 ? kk / 6 : 0, r = kk - 6 * f;
            const int co = k < base ? k : (r >= 3 ? r - 3 : r);
            const float fr = p.freq_xyz[f];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float d = acc_e[ch][4 * j + 2 * i + cc] * (kActInv * kLoInv);
              const float xc = co == 0 ? x[i][0] : co == 1 ? x[i][1] : x[i][2];
              float v = d;
              if (k >= base) {
                float sn, cs;
                sincosf(__fmul_rn(xc, fr), &sn, &cs);
                v = r < 3 ? d * fr * cs : -(d * fr * sn);
              }
              gx[i][0] += co == 0 ? v : 0.f;
              gx[i][1] += co == 1 ? v : 0.f;
              gx[i][2] += co == 2 ? v : 0.f;
            }
          }
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gx[i][c] += __shfl_xor_sync(0xffffffffu, gx[i][c], 1);
      gx[i][c] += __shfl_xor_sync(0xffffffffu, gx[i][c], 2);
    }
    if (q == 0 && rs.valid[i])
#pragma unroll
      for (int c = 0; c < 3; ++c) out[(int64_t)rs.pt[i] * 4 + 1 + c] = gx[i][c];
  }
}

template <int kH>
__global__ void __launch_bounds__(128 * grad_wg(kH) + 32, 1)
density_grad_tc_kernel(const __grid_constant__ Plan p, const float* __restrict__ blob, const float* __restrict__ pts,
                       int64_t P, int64_t n_tiles, float* __restrict__ out,  // out [P][4] = sigma_raw, d/dx, d/dy, d/dz
                       const int* __restrict__ n_dev) {  // non-null: the point count in device memory (at most P)
  constexpr int kWG = grad_wg(kH), kRows = 64 * kWG, kThreads = 128 * kWG + 32, kStage = kStageBytes;
  using Ring = WeightRing<kStage>;
  uint8_t* sm = smem_base();
  const GradSmemMap gm = grad_smem_map(p);
  const SmemMap& mp = gm.m;
  float* s_bias = reinterpret_cast<float*>(sm + mp.bias);
  float* s_headw = reinterpret_cast<float*>(sm + mp.headw);
  Ring ring{smem_u32(sm + mp.ring), smem_u32(sm + mp.bars), (uint32_t)mp.n_stages};

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // warp-uniform for ptxas: the role branches hold the wgmma
  const int enc_w = p.enc_tile_w;
  const int L = p.n_trunk;

  if (tid == 0) {
    ring.init(4 * kWG);
    fence_barrier_init();
  }
  // the trunk's biases and the sigma head, scaled as mlp_fwd_tc_kernel scales them
  for (int gi = 0; gi < L; ++gi)
    for (int i = tid; i < p.g[gi].n; i += kThreads) s_bias[p.g[gi].cum_n + i] = blob[p.g[gi].b_off + i] * (kActScale * kLoScale);
  const int hw1 = p.h[0].n_out * p.h[0].k;
  for (int i = tid; i < hw1; i += kThreads) s_headw[i] = blob[p.h[0].w_off + i] * kActInv;
  float* s_headb = s_headw + ((hw1 + 3) & ~3);
  if (tid < 4) s_headb[tid] = blob[p.h[0].b_off + tid];
  __syncthreads();

  if (n_dev) {
    P = *n_dev;
    n_tiles = (P + kRows - 1) / kRows;
  }
  const int my_tiles = (n_tiles > blockIdx.x) ? (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;

  if (warp == 4 * kWG) {
    // ===================== weight producer: the trunk forward's copies, then per layer from the last: the encoding
    // k-steps of its forward copy (layers that read the encoding), its tcd copy (layers after layer1) =============
    if ((tid & 31) == 0) {
      const uint64_t pol = l2_policy_evict_last();
      for (int j = 0; j < my_tiles; ++j) {
        for (int e = 0; e < L; ++e) {
          const MmaInfo mi = mma_info(p, blob, e, false, kStage);
          for (int ks = 0; ks < mi.ksteps; ks += mi.sps) {
            const uint32_t nk = (uint32_t)min(mi.sps, mi.ksteps - ks);
            ring.fill(mi.src + (size_t)ks * mi.kbytes, 1, nk * mi.kbytes, 0, pol);
          }
        }
        for (int t = L - 1; t >= 0; --t) {
          const GemmLayer& g = p.g[t];
          if (g.k_enc > 0 && g.enc_sel == 0) {
            const MmaInfo mi = mma_info(p, blob, t, false, kStage);
            for (int ks = mi.ksteps_h; ks < mi.ksteps; ++ks) ring.fill(mi.src + (size_t)ks * mi.kbytes, 1, mi.kbytes, 0, pol);
          }
          if (t > 0) {
            const uint8_t* src = reinterpret_cast<const uint8_t*>(blob + g.tcd_off);
            const uint32_t kbytes = 96u * (uint32_t)g.k_h;
            for (int ks = 0; ks < (g.n >> 4); ++ks) ring.fill(src + (size_t)ks * kbytes, 1, kbytes, 0, pol);
          }
        }
      }
    }
  } else {
    // ===================== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of every tile =====================
    const int wg = warp >> 2, wt = tid & 127, lane = tid & 31;
    const int row = wt & 63, half = wt >> 6;  // prologue: two threads per row split the frequencies
    uint8_t* act = sm + mp.act;
    uint8_t* enc = sm + mp.enc;
    const int enc_hb = kRows * enc_w * 2;
    uint32_t* s_mask = reinterpret_cast<uint32_t*>(sm + gm.mask) + wg * 64 * gm.mask_words;
    const int lr0 = 16 * (wt >> 5) + (lane >> 2);  // warpgroup row of accumulator row 0 (row 1: + 8)
    const uint32_t* const mrow[2] = {s_mask + lr0 * gm.mask_words, s_mask + (lr0 + 8) * gm.mask_words};
    const uint64_t g_hi = make_desc(smem_u32(act) + (uint32_t)(wg * 64 * kH * 2), 128, kH * 16);
    const uint32_t g_lo_off = (uint32_t)(kRows * kH * 2);
    auto wg_bar = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); };
#pragma unroll 1
    for (int j = 0; j < my_tiles; ++j) {
      const int64_t tile = blockIdx.x + (int64_t)j * gridDim.x;
      const int64_t p0 = tile * kRows + 64 * wg;
      const RowState rs = row_state(p0, lr0, P, 1, 0);
      // ---- encodings of this row -> operand tile (value / 16), as mlp_fwd_tc_kernel's prologue writes them for pts
      {
        const int64_t pt = (p0 + row < P) ? p0 + row : P - 1;
        const int nf = p.n_freq_xyz, mid = nf >> 1;
        const int f0 = half ? mid : 0, f1 = half ? nf : mid;
        const int base = p.inc_xyz ? 3 : 0;
        const int trow = 64 * wg + row;
        auto put = [&](int k, float v) {
          uint32_t hi, lo;
          split_f16x2(v * kActScale, 0.f, hi, lo);
          const int off = tile_piece(trow, k >> 3, enc_w) + (k & 7) * 2;
          *reinterpret_cast<uint16_t*>(enc + off) = (uint16_t)hi;
          *reinterpret_cast<uint16_t*>(enc + enc_hb + off) = (uint16_t)lo;
        };
        for (int c = 0; c < 3; ++c) {
          const float x = pts[pt * 3 + c];
          if (p.inc_xyz && half == 0) put(c, x);
          for (int f = f0; f < f1; ++f) {
            float sn, cs;
            sincosf(__fmul_rn(x, p.freq_xyz[f]), &sn, &cs);
            put(base + 6 * f + c, sn);
            put(base + 6 * f + 3 + c, cs);
          }
        }
        if (half == 1)
          for (int k = p.dim_xyz; k < enc_w; ++k) put(k, 0.f);
      }
      fence_proxy_async();
      wg_bar();
      // ---- the trunk: sigma_raw -> out[pt][0], the ReLU bits -> s_mask
#pragma unroll 1
      for (int e = 0; e < L; ++e)
        fwd_layer<false, false, kH, kStage, true>(p, blob, out, nullptr, sm, mp, e, wg, kRows, 0, 0, rs, ring, s_bias,
                                                  s_headw, s_headb, nullptr, hw1, s_mask, gm.mask_words);
      wg_bar();  // the last layer's bits are in place
      // ---- the reverse chain from G_{L-1} = w_sigma (.) mask_{L-1}, stored / 16 (s_headw holds 16 w: Y = 8 s_headw)
      float chain[kH / 2];
      {
        const float* wsig = s_headw + (3 - p.h[0].out_col) * p.h[0].k;
        const int q = tid & 3;
#pragma unroll
        for (int jj = 0; jj < kH / 8; ++jj)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            chain[4 * jj + 2 * i] = wsig[8 * jj + 2 * q] * 8.f;
            chain[4 * jj + 2 * i + 1] = wsig[8 * jj + 2 * q + 1] * 8.f;
          }
      }
      grad_g_store<kH>(p, chain, L - 1, act, kRows, mrow, 64 * wg + lr0);
      float acc_e[kMaxEncSteps][8];
#pragma unroll
      for (int c = 0; c < kMaxEncSteps; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc_e[c][i] = 0.f;
      int nch = 0;
#pragma unroll 1
      for (int t = L - 1; t >= 0; --t) {
        fence_proxy_async();  // generic-proxy stores of G_t -> the MMAs read them through the async proxy
        wg_bar();
        const GemmLayer& g = p.g[t];
        if (g.k_enc > 0 && g.enc_sel == 0) {
          nch = ((g.k_tc + 15) >> 4) - (g.k_h >> 4);
          grad_enc_mma<kH, kStage>(acc_e, ring, g_hi, g_lo_off, nch);
        }
        if (t > 0) {
          grad_chain_mma<kH, kStage>(chain, ring, g_hi, g_lo_off);
          wg_bar();  // every warp's MMAs have read G_t
          grad_g_store<kH>(p, chain, t - 1, act, kRows, mrow, 64 * wg + lr0);
        }
      }
#pragma unroll
      for (int c = 0; c < kMaxEncSteps; ++c) reg_fence(acc_e[c]);
      grad_x_store(p, acc_e, nch, pts, out, rs);
    }
  }
}

// what the density gradient needs beyond the wgmma inference forward (tc_supported); `what` names the call and the impl
int grad_tc_supported(const Plan& p, const char* what) {
  if (grad_smem_map(p).m.n_stages < 2) {
    set_error("%s: network too deep for the density gradient's shared-memory budget (%d trunk layers)", what, p.n_trunk);
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

template <int kH>
static int launch_grad(const Plan& p, const float* blob, const float* pts, int64_t P, float* out, const int* n_dev,
                       cudaStream_t s) {
  constexpr int kRows = 64 * grad_wg(kH), kThreads = 2 * kRows + 32;
  const int64_t tiles = (P + kRows - 1) / kRows;
  return launch_persistent(density_grad_tc_kernel<kH>, tiles, kThreads, grad_smem_map(p).m.total, s, "density_grad launch",
                           p, blob, pts, P, tiles, out, n_dev);
}

// n_dev non-null: the kernel reads the point count there (at most n_points, which sizes the grid)
int launch_density_grad_tc(const Plan& p, const float* blob, const float* pts, int64_t n_points, float* out,
                           const int* n_dev, cudaStream_t s) {
  return p.hidden == 256 ? launch_grad<256>(p, blob, pts, n_points, out, n_dev, s)
                         : launch_grad<128>(p, blob, pts, n_points, out, n_dev, s);
}

}  // namespace nerfb200
