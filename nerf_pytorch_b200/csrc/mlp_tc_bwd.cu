// mlp_tc_bwd.cu -- Hopper tensor-core (wgmma) backward of FlexibleNeRFModel (nerf/models.py:233-256, autograd of
// train_nerf.py:259) for hidden_size 128: the data-gradient chain AND every weight gradient of a 128-point tile in ONE
// kernel, so that the per-layer pre-activation gradients G_t never leave the SM (no gradient stash in HBM).
//
//   chain  : G_t = (G_{t+1} W_{t+1}[:, :hidden] + d_raw W_head) (.) relu'(layer t)          (M = points, K = features)
//   wgrad  : dW_t[n][k] += sum_p G_t[p][n] X_{t-1}[p][k]                                    (M = features n, K = points)
// Both are 3-term split-precision products on wgmma with fp16 operands (tc_common.cuh split_f16x2).  G_t is split into
// fp16 hi / lo ONCE in the epilogue registers and stored ONCE to a shared-memory operand tile (tc_common.cuh "Operand
// tiles"): its K-major view is the A operand of the chain, its MN-major view the A operand of the weight-gradient MMAs;
// the forward stashed every layer's activation X_t as the same kind of tile, so the B operand of the weight-gradient
// MMAs is a plain bulk copy from HBM.  Nothing is transposed on the CUDA cores.
//
// Precision: the whole tile runs in ONE power-of-two scale (max |d_raw| of the tile -> [4, 8)): the reduction of a
// weight gradient runs over points, so rows must share a scale, and rows that are tiny next to the tile's largest
// contribute below fp32 resolution to dW anyway.  The residual products carry a factor 2^11 (lo = (x - hi) 2^11 on
// both sides); they are accumulated first, the accumulator registers are multiplied by 2^-11, then the hi*hi products
// are added: ONE accumulator per weight gradient and no pre-scaled operand copies.
//
// Persistent kernel, one CTA per SM, two consumer warpgroups (warpgroup w owns points [64 w, 64 w + 64) of the chain
// and features [64 w, 64 w + 64) of every weight gradient) and one producer warpgroup, of which one thread streams the
// chain's weight copies through the weight ring (tc_common.cuh WeightRing); the producer gives its registers to the
// consumers (setmaxnreg), which hold the chain accumulator and a job accumulator at once.  Every wgmma is issued in
// warpgroup-uniform control flow (the warp index is broadcast from lane 0), so ptxas keeps the MMAs of a k-loop
// asynchronous.  The consumers' phases, per tile: tile_scale; per event e (layer t = n_gemm - 1 - e): g_epilogue (chain +
// head term, ReLU mask, hi / lo split -> G tile), chain_mma, then one job loop whose wgrad_job waits for the job's
// activation tile (bulk-copied from the stash one job ahead), runs its MMAs, hands the tile back (thread 0 requests the
// next job's once both warpgroups have) and drains the accumulator into the L2-resident gradient blob as 64-bit fixed
// point with red.global.add.u64 -- integer sums do not depend on the order of the adds, so the gradients are
// reproducible bit for bit; indicator_sums and dir_accumulate; at the end flush_cta.
#include "common.cuh"
#include "tc_common.cuh"

namespace nerfb200 {

using namespace tc;

namespace tcb {
constexpr int kWG = 2;                            // consumer warpgroups
constexpr int kThreadsB = 128 * (kWG + 1);       // + the producer warpgroup (one thread of it streams the weights)
constexpr int kProdRegs = 24, kConsRegs = 240;   // setmaxnreg split: (24 + 2 x 240) x 128 = 168 x 384 registers
constexpr int kWStage = 96 * 128;                 // one k-step of a 128-wide layer: 3 copies x 2 slabs x 128 x 16 B
                                                  // (all kMaxStages fit for A0 and A1: 73 KB for A1)
constexpr int kGBytes = 65536;                    // G tile: hi block 32 KB, lo block 32 KB (128 features)
constexpr int kXBytes = 65536;                    // activation tile of the running job
constexpr int kIndBytes = 4096;                   // ray-indicator tile: 128 points x 16 "features" (hi only)

struct SmemMapB {
  int g, x, ind, headw, bgrad, encd, sums, dacc, misc, bars, ring, total, n_stages;
};
__host__ __device__ inline SmemMapB smem_map_b(const Plan& p) {
  SmemMapB m;
  int off = 0;
  m.g = off;      off += kGBytes;
  m.x = off;      off += kXBytes;
  m.ind = off;    off += kIndBytes;
  m.headw = off;  off += (4 * 128 + 3 * 64 + 16) * 4;
  m.bgrad = off;  off += (p.enc_cum[0] + 8) * 4;   // bias gradients of every gemm layer + the heads' (8)
  m.encd = off;   off += kMaxRaysPerTile * 32 * 4;
  m.sums = off;   off += 64 * 16 * 4;             // per-ray sums of layers_dir[0]'s G (one tile)
  m.dacc = off;   off += 64 * 28 * 4;             // direction-encoding part of dW(layers_dir[0]), whole kernel
  m.misc = off;   off += 256;                     // tile maxima
  m.bars = off;   off += 256;
  m.ring = (off + 1023) & ~1023;
  m.n_stages = ring_depth(m.ring, kWStage);
  m.total = m.ring + (m.n_stages > 0 ? m.n_stages : 0) * kWStage;
  return m;
}

// One weight-gradient job: accumulator[n][k] = sum_p A[p][n] * B[p][k] over the tile's 128 points.
struct BwdJob {
  int src_enc;   // B tile: 1 = the xyz-encoding tile, 0 = the stashed output of gemm layer `src`
  int src;
  int n_b;       // columns = width of the B tile (multiple of 16)
  int nrows;     // accumulator rows 0.. that carry gradients
  int gb_off;    // kind 0: offset (int64 words) of this job's block in the gradient blob: 128 rows x n_b words, layout below blob_map
  int dst;       // kind 0: the gemm layer whose weight gradient this is; kind 1: the head, rows 0.. are its outputs
  int dst_col0;  // kind 0: first input column of the destination weight this block covers
  int ncols;     // kind 0: real columns
  int kind;      // 0: A = G tile, B = activation tile;  1: head job, A = activation tile (rows = its features), B = d_raw tile
};
constexpr int kMaxJobs = 3;

// the job table of a network, built on the host once per launch and passed by value (no per-thread enumeration)
struct BwdPlan {
  int n_jobs[kMaxGemm];
  BwdJob jobs[kMaxGemm][kMaxJobs];  // [event e (layer t = n_gemm - 1 - e)][job]
  int gb_total;                      // words of the jobs' blocks, laid out in event and job order
};
// The gradient blob: ONE L2-resident buffer of 64-bit fixed-point sums (value * 2^32, two's complement) that every CTA
// adds into.  Integer addition is associative, so the sums -- and the gradients -- are the same bits whatever order the
// CTAs' reduce-adds and atomics arrive in.  Resolution 2^-32 (2.3e-10) per added term; every partial sum must stay
// below 2^31 in magnitude.
//   [0, gb_total)  weight-gradient blocks of the jobs (red.global.add.u64 from the accumulator registers)
//   xb: bias gradients of the gemm layers (cum_n order) + the heads' 4 biases (+ 4 spare)
//   xd: direction-encoding part of dW(layers_dir[0]) [64][28]
//   xh: the heads' weight gradients [head][4 outputs][128 inputs]
constexpr float kFix = 4294967296.f;   // 2^32
struct BlobMap {
  int xb, xd, xh, words;
};
__host__ __device__ inline BlobMap blob_map(const Plan& p, int gb_total) {
  BlobMap m;
  m.xb = gb_total;
  m.xd = m.xb + p.enc_cum[0] + 8;
  m.xh = m.xd + 64 * 28;
  m.words = (m.xh + 2 * 4 * 128 + 15) & ~15;
  return m;
}
__device__ __forceinline__ unsigned long long to_fix(float v) { return (unsigned long long)__float2ll_rn(v * kFix); }
// A job's block (128 rows x ncol columns, ncol = n_b rounded up to 16) follows the accumulator fragment: element
// (row, col) is word  ((row >> 3) (ncol >> 3) + (col >> 3)) 64 + (col & 1) 32 + (row & 7) 4 + ((col & 7) >> 1),
// i.e. 8 x 8 (row-octet, column-octet) sub-blocks of 64 words, row-octets outer, each ordered [col & 1][row & 7]
// [(col & 7) / 2].  A wgmma m64nNk16 fragment holds rows 16 warp + lane / 4 (+ 8) and columns 8 j + 2 (lane & 3) (+ 1),
// so one warp-wide red of one accumulator register covers 256 contiguous bytes (8 whole 32-byte sectors).  With a
// row-major block the same reds touch 8 rows x 4 strided words each and reach less than half the aggregate rate
// (tools/mb_l2.cu).

inline BwdPlan make_bwd_plan(const Plan& p) {
  BwdPlan bp;
  bp.gb_total = 0;
  for (int e = 0; e < p.n_gemm; ++e) {
    const int t = p.n_gemm - 1 - e;
    const GemmLayer& g = p.g[t];
    int& n = bp.n_jobs[e];
    n = 0;
    auto add = [&](int src_enc, int src, int n_b, int nrows, int dst, int dst_col0, int ncols, int kind) {
      BwdJob& j = bp.jobs[e][n++];
      j.src_enc = src_enc; j.src = src; j.n_b = n_b; j.nrows = nrows;
      j.gb_off = bp.gb_total; j.dst = dst; j.dst_col0 = dst_col0; j.ncols = ncols; j.kind = kind;
      if (kind == 0) bp.gb_total += ((n_b + 15) / 16) * 128 * 16;
    };
    if (g.k_h > 0) add(0, g.src, g.k_h, g.n, t, 0, g.k_h, 0);
    if (g.k_enc > 0 && g.enc_sel == 0) add(1, 0, p.enc_tile_w, g.n, t, g.k_h, g.enc_real, 0);
    if (p.use_viewdirs && t == p.n_gemm - 1) {
      // the narrow heads: dW_head[c][k] = sum_p d_raw[p][c] X[p][k] with the activation tile on the M side
      add(0, t, g.n, p.h[1].k, 1, 0, 16, 1);                               // fc_rgb reads this layer's output
      add(0, p.h[0].src, p.g[p.h[0].src].n, p.h[0].k, 0, 0, 16, 1);        // fc_alpha reads the trunk output
    }
  }
  return bp;
}

}  // namespace tcb

using namespace tcb;
using RingB = WeightRing<kWStage>;

__device__ __forceinline__ void cta_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // both warpgroups

// shared-memory regions of the consumers
struct BwdSmem {
  uint8_t *g, *x, *ind;  // G tile, activation tile of the running job, ray-indicator tile
  float *headw, *bgrad, *encd, *sums, *dacc;
  uint32_t* max;         // [2]: tile max of |d_raw| (alternating tiles)
};

// per-tile state of a consumer thread
struct BwdTile {
  RowState rs;   // its two accumulator rows
  TileRays tr;   // the tile's rays
  float sc, us;  // d_raw scale of the tile, and the factor that takes the gradients back (and undoes the stash's / 16)
};

// Tile scale: max |d_raw| of the tile's points (warpgroup 0, one point per thread) -> a power of two that puts it in
// [4, 8).  The maxima alternate between two slots, so the one barrier both publishes this tile's and orders the reset
// of the next tile's slot after every read of the previous one.
__device__ __forceinline__ void tile_scale(const float* __restrict__ d_raw, int64_t p0, int64_t P, uint32_t* s_max, int it,
                                           BwdTile& tl) {
  const int tid = threadIdx.x, rowm = tid & 127;
  const float4 d4 = (p0 + rowm < P && tid < 128) ? reinterpret_cast<const float4*>(d_raw)[p0 + rowm]
                                                 : make_float4(0.f, 0.f, 0.f, 0.f);
  const float m = fmaxf(fmaxf(fabsf(d4.x), fabsf(d4.y)), fmaxf(fabsf(d4.z), fabsf(d4.w)));
  uint32_t mb = __float_as_uint(m);
  mb = __reduce_max_sync(0xffffffffu, mb);
  if ((tid & 31) == 0) atomicMax(&s_max[it & 1], mb);
  cta_bar();
  if (tid == 0) s_max[(it + 1) & 1] = 0u;  // reset the other slot for the next tile
  const uint32_t ex = (s_max[it & 1] >> 23) & 0xFFu;
  const bool scaled = ex >= 3u && ex <= 254u;
  tl.sc = scaled ? __uint_as_float((256u - ex) << 23) : 1.f;
  tl.us = (scaled ? __uint_as_float((ex - 2u) << 23) : 1.f) * kActInv;  // activations are stored / 16
}

// G-tile epilogue of event e (layer t): G_t of this thread's elements = (chain + d_raw W_head) (.) relu'(layer t) -> hi /
// lo -> the G tile (r0: warpgroup-local row of accumulator row 0).  The 64-wide layers_dir[0] also puts d_raw into feature
// rows 64..67 (zeros up to 79) for the heads' jobs; event 0 writes the ray-indicator tile and the direction encodings.
__device__ __forceinline__ void g_epilogue(const Plan& p, int e, const float (&chain)[64], const BwdTile& tl,
                                           const float* __restrict__ d_raw, const float* __restrict__ stash, int64_t P_pad,
                                           const float* __restrict__ dirs, int dir_stride, const BwdSmem& s, int hw1, int wg,
                                           int r0) {
  const int tid = threadIdx.x, q = tid & 3;
  const int t = p.n_gemm - 1 - e;
  const GemmLayer& g = p.g[t];
  const int hsel = head_of(p, t);
  const float* hw = hsel == 1 ? s.headw + hw1 : s.headw;
  const int hk = hsel >= 0 ? p.h[hsel].k : 0, hn = hsel >= 0 ? p.h[hsel].n_out : 0;
  const int hcol = hsel >= 0 ? p.h[hsel].out_col : 0;
  // this thread's ReLU mask words (two rows, up to four 32-column words each)
  uint32_t mw[2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      mw[i][m] = 0xFFFFFFFFu;
      if (g.relu && m < (g.n >> 5)) {
        const uint32_t* mask_row = reinterpret_cast<const uint32_t*>(stash) + (size_t)P_pad * (p.mask_base + g.mask_cum) +
                                   (size_t)tl.rs.pt[i] * (g.n >> 5);
        mw[i][m] = tl.rs.valid[i] ? __ldg(mask_row + m) : 0u;
      }
    }
  // d_raw of this thread's rows at the tile scale (re-read per event rather than kept live through the MMAs), and
  // the head outputs' entries of it selected once (a runtime index into dr would put it in local memory)
  float dr[2][4], hd[2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float4 d4 = tl.rs.valid[i] ? reinterpret_cast<const float4*>(d_raw)[tl.rs.pt[i]] : make_float4(0.f, 0.f, 0.f, 0.f);
    dr[i][0] = d4.x * tl.sc; dr[i][1] = d4.y * tl.sc; dr[i][2] = d4.z * tl.sc; dr[i][3] = d4.w * tl.sc;
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int k = (hcol + c) & 3;
      hd[i][c] = k == 0 ? dr[i][0] : k == 1 ? dr[i][1] : k == 2 ? dr[i][2] : dr[i][3];
    }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    if (j < (g.n >> 3)) {
      const int col = 8 * j + 2 * q;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float y0 = chain[4 * j + 2 * i], y1 = chain[4 * j + 2 * i + 1];  // Y = 2048 x, the accumulator's own scale
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if (c < hn) {
            const float2 w = *reinterpret_cast<const float2*>(hw + c * hk + col);
            y0 = fmaf(hd[i][c], w.x, y0);
            y1 = fmaf(hd[i][c], w.y, y1);
          }
        }
        const uint32_t word = mw[i][j >> 2];
        const int bit = 8 * (j & 3) + 2 * q;
        y0 = (word & (1u << bit)) ? y0 : 0.f;
        y1 = (word & (2u << bit)) ? y1 : 0.f;
        uint32_t hi, lo;
        split_f16x2_y(y0, y1, y0 * kLoInv, y1 * kLoInv, hi, lo);
        const int off = tile_piece(64 * wg + r0 + 8 * i, j, 128) + 4 * q;
        *reinterpret_cast<uint32_t*>(s.g + off) = hi;
        *reinterpret_cast<uint32_t*>(s.g + 32768 + off) = lo;
      }
    }
  }
  if (g.n == 64 && q == 0) {
    // 64-wide layer (layers_dir[0], first event of a tile): feature rows 64..67 carry d_raw for the heads' weight
    // gradients, the rest of the upper half is zero
    const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 64 * wg + r0 + 8 * i;
      uint32_t h01, l01, h23, l23;
      split_f16x2(dr[i][0], dr[i][1], h01, l01);
      split_f16x2(dr[i][2], dr[i][3], h23, l23);
      *reinterpret_cast<uint4*>(s.g + tile_piece(r, 8, 128)) = make_uint4(h01, h23, 0u, 0u);
      *reinterpret_cast<uint4*>(s.g + 32768 + tile_piece(r, 8, 128)) = make_uint4(l01, l23, 0u, 0u);
#pragma unroll
      for (int fb = 9; fb < 16; ++fb) {
        *reinterpret_cast<uint4*>(s.g + tile_piece(r, fb, 128)) = z4;
        *reinterpret_cast<uint4*>(s.g + 32768 + tile_piece(r, fb, 128)) = z4;
      }
    }
  }
  if (e == 0) {
    // ray-indicator tile of this tile: I[p][j] = 1 iff point p belongs to the tile's j-th ray; direction encodings
    if (q == 0) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        uint32_t w[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t lo16 = (tl.rs.ray_slot[i] == 2 * k && tl.rs.valid[i]) ? 0x3C00u : 0u;
          const uint32_t hi16 = (tl.rs.ray_slot[i] == 2 * k + 1 && tl.rs.valid[i]) ? 0x3C00u : 0u;
          w[k] = lo16 | (hi16 << 16);
        }
        const int r = 64 * wg + r0 + 8 * i;
        *reinterpret_cast<uint4*>(s.ind + tile_piece(r, 0, 16)) = make_uint4(w[0], w[1], w[2], w[3]);
        *reinterpret_cast<uint4*>(s.ind + tile_piece(r, 1, 16)) = make_uint4(w[4], w[5], w[6], w[7]);
      }
    }
    if (p.use_viewdirs && tid < tl.tr.n * 3) {
      const int jr = tid / 3, c = tid - 3 * jr;
      const float vv = dirs[(tl.tr.first + jr) * dir_stride + c];
      encode_coord(vv, c, p.inc_dir, 0, p.n_freq_dir, p.freq_dir, s.encd + jr * 32);
    }
  }
}

// chain[p][k] = 2^11 sum_n G_t[p][n] W_t[n][k] of this warpgroup's rows, N = k_h = 128, K = n: A = the warpgroup's rows
// of the G tile (K-major), B = the three weight copies from the ring (one k-step per stage)
__device__ __forceinline__ void chain_mma(float (&chain)[64], RingB& ring, const uint8_t* sG, int n, int wg) {
  const uint64_t a_hi = make_desc(smem_u32(sG) + (uint32_t)wg * 16384u, 128, 2048);
  const uint64_t b_ring = make_desc(ring.base, 2048, 128);
  wgmma_fence();
#pragma unroll 1
  for (int ks = 0; ks < (n >> 4); ++ks) {
    const uint32_t st = ring.acquire();
    const uint64_t b_hs = desc_adv(b_ring, st * (uint32_t)kWStage);
    const uint64_t ah = desc_adv(a_hi, ks * 256u);
    wgmma_f16<128>(chain, ah, b_hs, ks > 0 ? 1 : 0);
    wgmma_f16<128>(chain, desc_adv(ah, 32768u), desc_adv(b_hs, 2 * 2048u), 1);
    wgmma_f16<128>(chain, ah, desc_adv(b_hs, 4 * 2048u), 1);
    wgmma_commit();
    ring.release_behind(chain);
  }
  ring.release_last(chain);
}

// weight-gradient MMAs of width N (columns of the B tile) for this warpgroup's 64 accumulator rows:
//   acc = 2^-11 sum_ks (A_lo^T B_hi + A_hi^T B_lo) + sum_ks A_hi^T B_hi     (A, B MN-major; K = the tile's 128 points)
// plus, when kInd, the 16-column indicator product into acc_i (B = the exact 0 / 1 indicator tile, no lo part)
template <int N, bool kInd>
__device__ __forceinline__ void job_mma(float (&acc)[N / 2], float (&acc_i)[8], uint64_t a_hi, uint32_t a_lo_off,
                                        uint32_t a_ks, uint64_t b_hi, uint32_t b_lo_off, uint32_t b_ks, uint64_t i_d) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const uint64_t ah = desc_adv(a_hi, ks * a_ks), bh = desc_adv(b_hi, ks * b_ks);
    wgmma_f16<N, 1, 1>(acc, desc_adv(ah, a_lo_off), bh, ks > 0 ? 1 : 0);
    wgmma_f16<N, 1, 1>(acc, ah, desc_adv(bh, b_lo_off), 1);
    if (kInd) wgmma_f16<16, 1, 1>(acc_i, desc_adv(ah, a_lo_off), desc_adv(i_d, ks * 512u), ks > 0 ? 1 : 0);
  }
  wgmma_commit();
  wgmma_wait<0>();
  reg_fence(acc);
  if (kInd) reg_fence(acc_i);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] *= kLoInv;
  if (kInd) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc_i[i] *= kLoInv;
  }
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const uint64_t ah = desc_adv(a_hi, ks * a_ks);
    wgmma_f16<N, 1, 1>(acc, ah, desc_adv(b_hi, ks * b_ks), 1);
    if (kInd) wgmma_f16<16, 1, 1>(acc_i, ah, desc_adv(i_d, ks * 512u), 1);
  }
  wgmma_commit();
  wgmma_wait<0>();
  reg_fence(acc);
  if (kInd) reg_fence(acc_i);
}

// the finished accumulator (64 rows of this warpgroup x N columns) -> unscale -> fixed point -> red.global.add.u64 into
// the job's block of the gradient blob (the fragment layout above: one 256-byte span per warp and register)
template <int N>
__device__ __forceinline__ void job_drain(const float (&acc)[N / 2], float us, unsigned long long* gdst, int wg) {
  const int wt = threadIdx.x & 127, lane = wt & 31;
  // row-octets 8 wg + 2 warp (+ 1) of the block; lane = 4 (row & 7) + (col & 7) / 2
  unsigned long long* d = gdst + (8 * wg + 2 * (wt >> 5)) * (N / 8) * 64 + lane;
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) red_add_u64(d + (i * (N / 8) + j) * 64 + 32 * c, to_fix(acc[4 * j + 2 * i + c] * us));
}

// a head job's accumulator (rows = the head's inputs k, columns = d_raw channels) -> its outputs' weight gradients
__device__ __forceinline__ void head_drain(const float (&acc)[8], const HeadLayer& h, int head, float us,
                                           unsigned long long* gh, int wg, int r0) {
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int jj = 0; jj < 2; ++jj)
#pragma unroll
    for (int ii = 0; ii < 2; ++ii)
#pragma unroll
      for (int cc = 0; cc < 2; ++cc) {
        const int k = 64 * wg + r0 + 8 * ii, c = 8 * jj + 2 * q + cc - h.out_col;
        if (k < h.k && c >= 0 && c < h.n_out) atomicAdd(gh + head * 512 + c * 128 + k, to_fix(acc[4 * jj + 2 * ii + cc] * us));
      }
}

// indicator sums of layer t (event e): its bias gradient (all rays) and, for layers_dir[0], the per-ray sums that
// dir_accumulate turns into the direction-encoding part of its weight gradient
__device__ __forceinline__ void indicator_sums(const Plan& p, int e, const float (&acc_i)[8], float us, const BwdSmem& s,
                                               int wg, int r0) {
  const int q = threadIdx.x & 3;
  const GemmLayer& g = p.g[p.n_gemm - 1 - e];
  const float su = us * kActScale;  // the indicator is an exact 1, not an activation / 16
#pragma unroll
  for (int ii = 0; ii < 2; ++ii) {
    const int n = 64 * wg + r0 + 8 * ii;
    float tot = acc_i[2 * ii] + acc_i[2 * ii + 1] + acc_i[4 + 2 * ii] + acc_i[4 + 2 * ii + 1];
    tot += __shfl_xor_sync(0xffffffffu, tot, 1);
    tot += __shfl_xor_sync(0xffffffffu, tot, 2);
    if (q == 0) {
      if (n < g.n) s.bgrad[g.cum_n + n] += tot * su;
      if (e == 0 && p.use_viewdirs && n >= 64 && n < 68) s.bgrad[p.enc_cum[0] + n - 64] += tot * su;  // d_rgb, d_sigma sums
    }
    if (e == 0 && p.use_viewdirs && n < 64) {
      s.sums[n * 16 + 2 * q] = acc_i[2 * ii] * su;
      s.sums[n * 16 + 2 * q + 1] = acc_i[2 * ii + 1] * su;
      s.sums[n * 16 + 8 + 2 * q] = acc_i[4 + 2 * ii] * su;
      s.sums[n * 16 + 9 + 2 * q] = acc_i[4 + 2 * ii + 1] * su;
    }
  }
}

// direction-encoding part of dW(layers_dir[0]) of this tile: the per-ray sums of G x the rays' direction encodings
__device__ __forceinline__ void dir_accumulate(const Plan& p, const BwdSmem& s, int n_rays) {
  for (int idx = threadIdx.x; idx < 64 * p.dim_dir; idx += 128 * kWG) {
    const int n = idx / p.dim_dir, k = idx - n * p.dim_dir;
    float a = 0.f;
    for (int jr = 0; jr < n_rays; ++jr) a = fmaf(s.sums[n * 16 + jr], s.encd[jr * 32 + k], a);
    s.dacc[n * 28 + k] += a;
  }
}

// whether this warpgroup runs a job's MMAs (warpgroup-uniform): it has accumulator rows in the job -- or, for warpgroup 1
// of layers_dir[0]'s first job, only the d_raw rows 64..67 of the indicator product
__device__ __forceinline__ bool takes_part(const Plan& p, const BwdJob& jq, int e, bool first, int wg) {
  return 64 * wg < jq.nrows || (jq.kind == 0 && first && e == 0 && p.use_viewdirs);
}

// One weight-gradient job of width N (kHead: a narrow head's job; N = 0: this warpgroup takes no part) on the landed
// activation tile: the MMAs, hand_back() once they are complete, then the drain.
template <int N, bool kHead, class HandBack>
__device__ __forceinline__ void wgrad_job(const Plan& p, const BwdJob& jq, int e, bool first, const BwdSmem& s,
                                          const BwdTile& tl, unsigned long long* gb, const BlobMap& bm, int wg, int r0,
                                          HandBack&& hand_back) {
  const uint32_t fstr = (uint32_t)(jq.n_b >> 3) * 128u;  // bytes between 8-point blocks of the activation tile
  const bool ind = !kHead && first;                       // the event's first job also runs the indicator product
  float acc[N > 0 ? N / 2 : 1], acc_i[8];
  if constexpr (N > 0) {
    if constexpr (kHead) {
      // A = activation tile (rows = its features, MN-major), B = d_raw (feature rows 64..79 of the G tile); the residual
      // products first as in every job, with B's lo block 32 KB on
      const uint64_t xa = make_desc(smem_u32(s.x) + (uint32_t)wg * 1024u, fstr, 128);
      const uint64_t db = make_desc(smem_u32(s.g) + 1024u, 2048, 128);
      job_mma<16, false>(acc, acc_i, xa, 32768u, 2 * fstr, db, 32768u, 4096u, 0);
    } else {
      const uint64_t ga = make_desc(smem_u32(s.g) + (uint32_t)wg * 1024u, 2048, 128);  // G^T: rows = features
      const uint64_t xb = make_desc(smem_u32(s.x), fstr, 128);
      const uint64_t id = make_desc(smem_u32(s.ind), 256, 128);
      if (ind) job_mma<N, true>(acc, acc_i, ga, 32768u, 4096u, xb, 32768u, 2 * fstr, id);
      else job_mma<N, false>(acc, acc_i, ga, 32768u, 4096u, xb, 32768u, 2 * fstr, id);
    }
  }
  hand_back();
  if constexpr (N == 0) {
    return;
  } else if constexpr (kHead) {
    head_drain(acc, p.h[jq.dst], jq.dst, tl.us, gb + bm.xh, wg, r0);
  } else {
    if (64 * wg < jq.nrows) job_drain<N>(acc, tl.us, gb + jq.gb_off, wg);
    if (ind) indicator_sums(p, e, acc_i, tl.us, s, wg, r0);
  }
}

// the CTA's bias and direction-encoding sums -> the gradient blob
__device__ __forceinline__ void flush_cta(const Plan& p, const BwdSmem& s, unsigned long long* gb, const BlobMap& bm) {
  for (int i = threadIdx.x; i < p.enc_cum[0] + 8; i += kThreadsB) atomicAdd(gb + bm.xb + i, to_fix(s.bgrad[i]));
  for (int i = threadIdx.x; i < 64 * 28; i += kThreadsB) atomicAdd(gb + bm.xd + i, to_fix(s.dacc[i]));
}

__global__ void __launch_bounds__(kThreadsB, 1)
mlp_bwd_tc_kernel(const __grid_constant__ Plan p, const float* __restrict__ blob, const float* __restrict__ dirs,
                  int dir_stride, const float* __restrict__ d_raw, const float* __restrict__ stash, int64_t P, int S,
                  int64_t n_tiles, float* __restrict__ gblob,
                  const __grid_constant__ BwdPlan bp) {
  uint8_t* sm = smem_base();
  const SmemMapB mp = smem_map_b(p);
  BwdSmem s;
  s.g = sm + mp.g;
  s.x = sm + mp.x;
  s.ind = sm + mp.ind;
  s.headw = reinterpret_cast<float*>(sm + mp.headw);
  s.bgrad = reinterpret_cast<float*>(sm + mp.bgrad);
  s.encd = reinterpret_cast<float*>(sm + mp.encd);
  s.sums = reinterpret_cast<float*>(sm + mp.sums);
  s.dacc = reinterpret_cast<float*>(sm + mp.dacc);
  s.max = reinterpret_cast<uint32_t*>(sm + mp.misc);
  RingB ring{smem_u32(sm + mp.ring), smem_u32(sm + mp.bars), (uint32_t)mp.n_stages};
  const uint32_t x_full = ring.bars + 16 * kMaxStages;  // the running job's activation tile landed (after the ring's)

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // warp-uniform for ptxas: the role branches hold the wgmma
  const int64_t P_pad = n_tiles * kTileRows;
  const int E = p.n_gemm;
  const int hw1 = p.h[0].n_out * p.h[0].k;
  const int hw2 = p.n_head > 1 ? p.h[1].n_out * p.h[1].k : 0;
  const BlobMap bm = blob_map(p, bp.gb_total);
  unsigned long long* gb = reinterpret_cast<unsigned long long*>(gblob);

  if (tid == 0) {
    ring.init(4 * kWG);
    mbar_init(x_full, 1);
    fence_barrier_init();
    s.max[0] = s.max[1] = 0u;
  }
  // head weights at the chain accumulator's 2^11 scale (the epilogue works on Y = 2048 y, tc_common.cuh split_f16x2_y)
  for (int i = tid; i < hw1; i += kThreadsB) s.headw[i] = blob[p.h[0].w_off + i] * kLoScale;
  for (int i = tid; i < hw2; i += kThreadsB) s.headw[hw1 + i] = blob[p.h[1].w_off + i] * kLoScale;
  for (int i = tid; i < p.enc_cum[0] + 8; i += kThreadsB) s.bgrad[i] = 0.f;
  for (int i = tid; i < kMaxRaysPerTile * 32; i += kThreadsB) s.encd[i] = 0.f;
  for (int i = tid; i < 64 * 28; i += kThreadsB) s.dacc[i] = 0.f;
  for (int i = tid; i < kGBytes / 16; i += kThreadsB) reinterpret_cast<uint4*>(s.g)[i] = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async();
  __syncthreads();

  const int my_tiles = (n_tiles > blockIdx.x) ? (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;

  if (warp >= 4 * kWG) {
    // ===================== weight producer: the chain of event e streams layer t's transposed copies ============
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProdRegs));
    if (warp == 4 * kWG && lane == 0) {
      const uint64_t pol = l2_policy_evict_last();
      for (int it = 0; it < my_tiles; ++it)
        for (int e = 0; e + 1 < E; ++e) {
          const GemmLayer& g = p.g[E - 1 - e];
          const uint8_t* src = reinterpret_cast<const uint8_t*>(blob + g.tcd_off);
          const uint32_t kbytes = 96u * (uint32_t)g.k_h;
          for (int ks = 0; ks < (g.n >> 4); ++ks) ring.fill(src + (size_t)ks * kbytes, 1, kbytes, 0, pol);
        }
    }
  } else {
    // ===================== consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsRegs));
    const int wg = warp >> 2, wt = tid & 127;
    const int r0 = 16 * (wt >> 5) + (lane >> 2);   // warpgroup-local row of accumulator row 0 (row 1: + 8)
    uint32_t x_ph = 0;
    // activation tile of job (it, e, i): hi block, lo block (issued by thread 0 one job ahead)
    auto issue_x = [&](int it, int e, int i) {
      const BwdJob& jq = bp.jobs[e][i];
      const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
      const uint8_t* src = reinterpret_cast<const uint8_t*>(stash + (size_t)P_pad * (jq.src_enc ? p.enc_cum[0] : p.g[jq.src].cum_n)) +
                           (size_t)tile * tile_bytes(jq.n_b);
      const uint32_t hb = (uint32_t)tile_half_bytes(jq.n_b);
      mbar_arrive_expect_tx(x_full, 2 * hb);
      bulk_g2s(smem_u32(s.x), src, hb, x_full);
      bulk_g2s(smem_u32(s.x) + 32768u, src + hb, hb, x_full);
    };
    if (tid == 0 && my_tiles > 0) issue_x(0, 0, 0);

    for (int it = 0; it < my_tiles; ++it) {
      const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
      const int64_t p0 = tile * kTileRows;
      BwdTile tl;
      tl.tr = tile_rays(p0, kTileRows, P, S);
      tl.rs = row_state(p0 + 64 * wg, r0, P, S, tl.tr.first);
      tile_scale(d_raw, p0, P, s.max, it, tl);

      float chain[64];  // G_{t+1} W_{t+1}[:, :128] of this warpgroup's rows (the previous event's chain MMA)
#pragma unroll
      for (int i = 0; i < 64; ++i) chain[i] = 0.f;
      for (int e = 0; e < E; ++e) {
        g_epilogue(p, e, chain, tl, d_raw, stash, P_pad, dirs, dir_stride, s, hw1, wg, r0);
        fence_proxy_async();
        cta_bar();  // the G tile (and the indicator tile) complete
        if (e + 1 < E) chain_mma(chain, ring, s.g, p.g[E - 1 - e].n, wg);

        // ---- the job loop: every consumer thread waits for each job's activation tile once and hands it back once
        const int nj = bp.n_jobs[e];
        for (int i = 0; i < nj; ++i) {
          const BwdJob& jq = bp.jobs[e][i];
          mbar_wait(x_full, x_ph);
          x_ph ^= 1;
          // Once both warpgroups are through, nothing reads the activation tile any more and thread 0 requests the
          // next job's, so that the load overlaps this job's drain instead of following it.
          auto hand_back_x = [&]() {
            cta_bar();
            if (tid == 0) {
              int ni = i + 1, ne = e, nit = it;
              if (ni == nj) {
                ni = 0;
                if (++ne == E) { ne = 0; ++nit; }
              }
              if (nit < my_tiles) issue_x(nit, ne, ni);
            }
          };
          if (!takes_part(p, jq, e, i == 0, wg)) {
            wgrad_job<0, false>(p, jq, e, i == 0, s, tl, gb, bm, wg, r0, hand_back_x);
          } else if (jq.kind == 1) {
            wgrad_job<16, true>(p, jq, e, i == 0, s, tl, gb, bm, wg, r0, hand_back_x);
          } else {
            const int w = jq.n_b;
            if (w == 128) wgrad_job<128, false>(p, jq, e, i == 0, s, tl, gb, bm, wg, r0, hand_back_x);
            else if (w == 64) wgrad_job<64, false>(p, jq, e, i == 0, s, tl, gb, bm, wg, r0, hand_back_x);
            else if (w == 48) wgrad_job<48, false>(p, jq, e, i == 0, s, tl, gb, bm, wg, r0, hand_back_x);
            else if (w == 32) wgrad_job<32, false>(p, jq, e, i == 0, s, tl, gb, bm, wg, r0, hand_back_x);
            else wgrad_job<16, false>(p, jq, e, i == 0, s, tl, gb, bm, wg, r0, hand_back_x);
          }
          if (e == 0 && i == 0 && p.use_viewdirs) {
            cta_bar();  // the per-ray sums of both warpgroups are in place
            dir_accumulate(p, s, tl.tr.n);
          }
        }
      }
    }
  }
  __syncthreads();
  flush_cta(p, s, gb, bm);
}

// gradient blob (fixed point) -> flat (torch-layout) gradient vector: every blob word is added to the one flat element it
// belongs to.  Weight-gradient job blocks follow the accumulator fragment (above make_bwd_plan).
__global__ void unpack_grad_kernel(const __grid_constant__ Plan p, const __grid_constant__ BwdPlan bp,
                                   const unsigned long long* __restrict__ gb, float* __restrict__ flat_grad) {
  const BlobMap sl = blob_map(p, bp.gb_total);
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < sl.words; idx += gridDim.x * blockDim.x) {
    int64_t dst = -1;
    if (idx < bp.gb_total) {
      for (int e = 0; e < p.n_gemm && dst < 0; ++e) {
        const int nj = bp.n_jobs[e];
        for (int i = 0; i < nj; ++i) {
          const BwdJob& j = bp.jobs[e][i];
          if (j.kind != 0) continue;
          const int ncol = ((j.n_b + 15) / 16) * 16, sz = 128 * ncol;
          if (idx < j.gb_off || idx >= j.gb_off + sz) continue;
          const int r = idx - j.gb_off, blk = r >> 6, w = r & 63;
          const int rr = 8 * (blk / (ncol >> 3)) + ((w >> 2) & 7);
          const int col = 8 * (blk % (ncol >> 3)) + 2 * (w & 3) + (w >> 5);
          const GemmLayer& g = p.g[j.dst];
          if (rr < j.nrows && col < j.ncols)
            dst = g.flat_w + (int64_t)rr * (g.k_h + g.enc_real) + j.dst_col0 + col;
          e = p.n_gemm;  // found the block
          break;
        }
      }
    } else if (idx < sl.xd) {
      const int i = idx - sl.xb;
      if (i < p.enc_cum[0]) {
        for (int gi = 0; gi < p.n_gemm; ++gi)
          if (i >= p.g[gi].cum_n && i < p.g[gi].cum_n + p.g[gi].n) dst = p.g[gi].flat_b + (i - p.g[gi].cum_n);
      } else if (p.use_viewdirs) {
        const int j = i - p.enc_cum[0];
        if (j < 3) dst = p.h[1].flat_b + j;
        else if (j == 3) dst = p.h[0].flat_b;
      }
    } else if (idx < sl.xh) {
      const int i = idx - sl.xd, n = i / 28, k = i - 28 * n;
      const GemmLayer& gd = p.g[p.n_gemm - 1];
      if (p.use_viewdirs && n < gd.n && k < p.dim_dir) dst = gd.flat_w + (int64_t)n * (gd.k_h + gd.enc_real) + gd.k_h + k;
    } else if (idx < sl.xh + 1024 && p.use_viewdirs) {
      const int i = idx - sl.xh, hd = i >> 9, c = (i >> 7) & 3, k = i & 127;
      const HeadLayer& h = p.h[hd];
      if (c < h.n_out && k < h.k) dst = h.flat_w + (int64_t)c * h.k + k;
    }
    if (dst < 0) continue;
    flat_grad[dst] += (float)((double)(long long)gb[idx] * (1.0 / 4294967296.0));  // the only writer of this element
  }
}

// the gradient blob, in floats (two per 64-bit word)
int64_t bwd_tc_scratch_floats(const Plan& p) { return 2 * (int64_t)blob_map(p, make_bwd_plan(p).gb_total).words; }

// what the fused backward needs beyond the training forward (tc_supported); `what` names the call and the impl
int bwd_tc_supported(const Plan& p, const char* what) {
  if (!p.use_viewdirs) {
    set_error("%s: the fused backward needs a view-dependent model (fc_rgb / fc_alpha heads); use impl=0", what);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (p.dim_dir > 28) {
    set_error("%s: direction encodings wider than 28 not supported by the fused backward; use impl=0", what);
    return NERFB200_ERR_UNSUPPORTED;
  }
  if (smem_map_b(p).n_stages < 2) {
    set_error("%s: network too deep for the backward's shared-memory budget; use impl=0", what);
    return NERFB200_ERR_UNSUPPORTED;
  }
  return NERFB200_OK;
}

int launch_mlp_bwd_tc(const Plan& p, const float* blob, const float* dirs, int dir_stride, int64_t n_rays, int n_samples,
                      const float* d_raw, const float* stash, float* gblob, float* flat_grad, cudaStream_t s) {
  const int64_t P = n_rays * n_samples;
  const int64_t tiles = (P + kTileRows - 1) / kTileRows;
  const BwdPlan bp = make_bwd_plan(p);
  const BlobMap bm = blob_map(p, bp.gb_total);
  int rc = check_cuda(cudaMemsetAsync(gblob, 0, (size_t)bm.words * 8, s), "mlp_bwd_tc blob memset");
  if (rc) return rc;
  rc = launch_persistent(mlp_bwd_tc_kernel, tiles, kThreadsB, smem_map_b(p).total, s, "mlp_bwd_tc launch", p, blob, dirs,
                         dir_stride, d_raw, stash, P, n_samples, tiles, gblob, bp);
  if (rc) return rc;
  const int blocks = (bm.words + 255) / 256;
  unpack_grad_kernel<<<blocks, 256, 0, s>>>(p, bp, reinterpret_cast<const unsigned long long*>(gblob), flat_grad);
  count_launch();
  return check_cuda(cudaGetLastError(), "unpack_grad launch");
}

}  // namespace nerfb200
