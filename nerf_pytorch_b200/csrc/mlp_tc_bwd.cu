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
// chain's weight copies through a cp.async.bulk ring; the producer gives its registers to the consumers (setmaxnreg), which
// hold the chain accumulator and a job accumulator at once.  Every wgmma is issued in warpgroup-uniform control flow (the
// warp index is broadcast from lane 0), so ptxas keeps the MMAs of a k-loop asynchronous.  Per layer: epilogue (chain
// accumulator + head term, ReLU mask, split -> G tile), chain MMA of the warpgroup's rows, then the layer's
// weight-gradient jobs: A = the G tile (MN-major), B = the activation tile (bulk-copied from the stash one job ahead and
// requested as soon as both warpgroups' MMAs of the running job are complete), the 16-column ray-indicator job that yields the bias gradients and
// the per-ray sums of layers_dir[0], and the two narrow heads' jobs with the roles swapped (A = activation tile, B =
// d_raw = feature rows 64..79 of the first layer's G tile).  Finished weight-gradient accumulators are unscaled,
// converted to 64-bit fixed point and added into the L2-resident gradient blob straight from the registers with
// red.global.add.u64 (the warpgroup goes on to its next MMAs while the adds drain); integer sums do not depend on the
// order of the adds, so the gradients are reproducible bit for bit.
#include "common.cuh"
#include "tc_common.cuh"
#include "wgmma.cuh"

namespace nerfb200 {

namespace tcb {
constexpr int kWG = 2;                            // consumer warpgroups
constexpr int kThreadsB = 128 * (kWG + 1);       // + the producer warpgroup (one thread of it streams the weights)
constexpr int kProdRegs = 24, kConsRegs = 240;   // setmaxnreg split: (24 + 2 x 240) x 128 = 168 x 384 registers
constexpr int kWStage = 96 * 128;                 // one k-step of a 128-wide layer: 3 copies x 2 slabs x 128 x 16 B
constexpr int kMaxWStages = 6;                    // smem_map_b leaves room for all 6 for A0 and A1 (73 KB for A1)
constexpr int kGBytes = 65536;                    // G tile: hi block 32 KB, lo block 32 KB (128 features)
constexpr int kXBytes = 65536;                    // activation tile of the running job
constexpr int kIndBytes = 4096;                   // ray-indicator tile: 128 points x 16 "features" (hi only)
constexpr int kMaxRays = 10;
constexpr int kSmemLimitB = 232448 - 1024;

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
  m.encd = off;   off += kMaxRays * 32 * 4;
  m.sums = off;   off += 64 * 16 * 4;             // per-ray sums of layers_dir[0]'s G (one tile)
  m.dacc = off;   off += 64 * 28 * 4;             // direction-encoding part of dW(layers_dir[0]), whole kernel
  m.misc = off;   off += 256;                     // tile maxima
  m.bars = off;   off += 256;
  off = (off + 1023) & ~1023;
  m.ring = off;
  int ns = (kSmemLimitB - off) / kWStage;
  if (ns > kMaxWStages) ns = kMaxWStages;
  m.n_stages = ns;
  m.total = off + (ns > 0 ? ns : 0) * kWStage;
  return m;
}

// One weight-gradient job: accumulator[n][k] = sum_p A[p][n] * B[p][k] over the tile's 128 points.
struct BwdJob {
  int src_enc;   // B tile: 1 = the xyz-encoding tile, 0 = the stashed output of gemm layer `src`
  int src;
  int n_b;       // columns = width of the B tile (multiple of 16)
  int row0, nrows;  // accumulator rows that carry gradients
  int gb_off;    // offset (int64 words) of this job's block in the gradient blob: 128 rows x n_b words, layout below blob_map
  int dst_head;  // -1: rows are output features of gemm layer `dst`; else head index, rows row0.. are its outputs
  int dst;       // gemm index
  int dst_col0;  // first input column of the destination weight this block covers
  int ncols;     // real columns
  int kind;      // 0: A = G tile, B = activation tile;  1: head job, A = activation tile (rows = its features), B = d_raw tile
};
constexpr int kMaxJobs = 3;

// jobs of event e (layer t = n_gemm - 1 - e); returns their number.  gb offsets are cumulative over the events.
__host__ __device__ inline int bwd_jobs(const Plan& p, int e, BwdJob* out, int* gb_total = nullptr) {
  int gb = 0, n_out = 0;
  for (int ev = 0; ev <= (gb_total ? p.n_gemm - 1 : e); ++ev) {
    const int t = p.n_gemm - 1 - ev;
    const GemmLayer& g = p.g[t];
    int n = 0;
    BwdJob jb[kMaxJobs];
    auto add = [&](int src_enc, int src, int n_b, int row0, int nrows, int dst_head, int dst, int dst_col0, int ncols,
                   int kind) {
      BwdJob& j = jb[n++];
      j.src_enc = src_enc; j.src = src; j.n_b = n_b; j.row0 = row0; j.nrows = nrows;
      j.gb_off = gb; j.dst_head = dst_head; j.dst = dst; j.dst_col0 = dst_col0; j.ncols = ncols; j.kind = kind;
      if (kind == 0) gb += ((n_b + 15) / 16) * 128 * 16;
    };
    if (g.k_h > 0) add(0, g.src, g.k_h, 0, g.n, -1, t, 0, g.k_h, 0);
    if (g.k_enc > 0 && g.enc_sel == 0) add(1, 0, p.enc_tile_w, 0, g.n, -1, t, g.k_h, g.enc_real, 0);
    if (p.use_viewdirs && t == p.n_gemm - 1) {
      // the narrow heads: dW_head[c][k] = sum_p d_raw[p][c] X[p][k] with the activation tile on the M side
      add(0, t, g.n, 0, p.h[1].k, 1, t, 0, 16, 1);                               // fc_rgb reads this layer's output
      add(0, p.h[0].src, p.g[p.h[0].src].n, 0, p.h[0].k, 0, t, 0, 16, 1);        // fc_alpha reads the trunk output
    }
    if (ev == e && out)
      for (int i = 0; i < n; ++i) out[i] = jb[i];
    if (ev == e) n_out = n;
  }
  if (gb_total) *gb_total = gb;
  return n_out;
}

// the job table of a network, built on the host once per launch and passed by value (no per-thread enumeration)
struct BwdPlan {
  int n_jobs[kMaxGemm];
  BwdJob jobs[kMaxGemm][kMaxJobs];
  int gb_total;
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
  for (int e = 0; e < p.n_gemm; ++e) bp.n_jobs[e] = bwd_jobs(p, e, bp.jobs[e]);
  bwd_jobs(p, 0, nullptr, &bp.gb_total);
  return bp;
}

}  // namespace tcb

using namespace tc;
using namespace tcb;

__device__ __forceinline__ void cta_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // both warpgroups

// weight-gradient job of width N (columns of the B tile) for this warpgroup's 64 accumulator rows:
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

__global__ void __launch_bounds__(kThreadsB, 1)
mlp_bwd_tc_kernel(const __grid_constant__ Plan p, const float* __restrict__ blob, const float* __restrict__ rays,
                  int ray_stride, const float* __restrict__ d_raw, const float* __restrict__ stash, int64_t P, int S,
                  int64_t n_tiles, float* __restrict__ gblob,
                  const __grid_constant__ BwdPlan bp) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const SmemMapB mp = smem_map_b(p);
  uint8_t* sG = sm + mp.g;
  uint8_t* sX = sm + mp.x;
  uint8_t* sInd = sm + mp.ind;
  float* s_headw = reinterpret_cast<float*>(sm + mp.headw);
  float* s_bgrad = reinterpret_cast<float*>(sm + mp.bgrad);
  float* s_encd = reinterpret_cast<float*>(sm + mp.encd);
  float* s_sums = reinterpret_cast<float*>(sm + mp.sums);
  float* s_dacc = reinterpret_cast<float*>(sm + mp.dacc);
  uint32_t* s_max = reinterpret_cast<uint32_t*>(sm + mp.misc);      // [2]: tile max of |d_raw| (alternating tiles)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + mp.bars);
  uint64_t* w_full = bars;                      // [kMaxWStages]
  uint64_t* w_empty = bars + kMaxWStages;       // [kMaxWStages]
  uint64_t* x_full = bars + 2 * kMaxWStages;    // the running job's activation tile landed
  const uint32_t n_stages = (uint32_t)mp.n_stages;

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // warp-uniform for ptxas: the role branches hold the wgmma
  const int64_t P_pad = n_tiles * kTileRows;
  const int E = p.n_gemm;
  const int hw1 = p.h[0].n_out * p.h[0].k;
  const int hw2 = p.n_head > 1 ? p.h[1].n_out * p.h[1].k : 0;
  const BlobMap bm = blob_map(p, bp.gb_total);
  unsigned long long* gb = reinterpret_cast<unsigned long long*>(gblob);

  if (tid == 0) {
    for (int i = 0; i < kMaxWStages; ++i) {
      mbar_init(&w_full[i], 1);
      mbar_init(&w_empty[i], 4 * kWG);
    }
    mbar_init(x_full, 1);
    fence_barrier_init();
    s_max[0] = s_max[1] = 0u;
  }
  // head weights at the chain accumulator's 2^11 scale (the epilogue works on Y = 2048 y, tc_common.cuh split_f16x2_y)
  for (int i = tid; i < hw1; i += kThreadsB) s_headw[i] = blob[p.h[0].w_off + i] * kLoScale;
  for (int i = tid; i < hw2; i += kThreadsB) s_headw[hw1 + i] = blob[p.h[1].w_off + i] * kLoScale;
  for (int i = tid; i < p.enc_cum[0] + 8; i += kThreadsB) s_bgrad[i] = 0.f;
  for (int i = tid; i < kMaxRays * 32; i += kThreadsB) s_encd[i] = 0.f;
  for (int i = tid; i < 64 * 28; i += kThreadsB) s_dacc[i] = 0.f;
  for (int i = tid; i < kGBytes / 16; i += kThreadsB) reinterpret_cast<uint4*>(sG)[i] = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async();
  __syncthreads();

  const int my_tiles = (n_tiles > blockIdx.x) ? (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;

  if (warp >= 4 * kWG) {
    // ===================== weight producer: the chain of event e streams layer t's transposed copies ============
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProdRegs));
    if (warp == 4 * kWG && lane == 0) {
      Pipe pp;
      const uint64_t pol = l2_policy_evict_last();
      for (int it = 0; it < my_tiles; ++it)
        for (int e = 0; e + 1 < E; ++e) {
          const GemmLayer& g = p.g[E - 1 - e];
          const uint8_t* src = reinterpret_cast<const uint8_t*>(blob + g.tcd_off);
          const uint32_t kbytes = 96u * (uint32_t)g.k_h;
          for (int ks = 0; ks < (g.n >> 4); ++ks) {
            mbar_wait(&w_empty[pp.stage], pp.phase ^ 1);
            mbar_arrive_expect_tx(&w_full[pp.stage], kbytes);
            bulk_g2s_hint(sm + mp.ring + pp.stage * kWStage, src + (size_t)ks * kbytes, kbytes, &w_full[pp.stage], pol);
            pp.advance(n_stages);
          }
        }
    }
  } else {
    // ===================== consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsRegs));
    const int wg = warp >> 2, wt = tid & 127, q = lane & 3;
    const int r0 = 16 * (wt >> 5) + (lane >> 2);   // warpgroup-local row of accumulator row 0 (row 1: + 8)
    uint32_t x_ph = 0;
    Pipe pp;
    // activation tile of job (it, e, i): hi block, lo block (issued by thread 0 one job ahead)
    auto issue_x = [&](int it, int e, int i) {
      const BwdJob& jq = bp.jobs[e][i];
      const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
      const uint8_t* src = reinterpret_cast<const uint8_t*>(stash + (size_t)P_pad * (jq.src_enc ? p.enc_cum[0] : p.g[jq.src].cum_n)) +
                           (size_t)tile * tile_bytes(jq.n_b);
      const uint32_t hb = (uint32_t)tile_half_bytes(jq.n_b);
      mbar_arrive_expect_tx(x_full, 2 * hb);
      bulk_g2s(sX, src, hb, x_full);
      bulk_g2s(sX + 32768, src + hb, hb, x_full);
    };
    if (tid == 0 && my_tiles > 0) issue_x(0, 0, 0);

    for (int it = 0; it < my_tiles; ++it) {
      const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
      const int64_t p0 = tile * kTileRows;
      const int64_t first_ray = p0 / S;
      const int64_t last_pt = (p0 + kTileRows - 1 < P) ? p0 + kTileRows - 1 : P - 1;
      const int n_rays_tile = (int)(last_pt / S - first_ray) + 1;
      int64_t pt[2];
      bool valid[2];
      int ray_slot[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        pt[i] = p0 + 64 * wg + r0 + 8 * i;
        valid[i] = pt[i] < P;
        if (!valid[i]) pt[i] = P - 1;
        ray_slot[i] = (int)(pt[i] / S - first_ray);
      }
      // ---- tile scale: max |d_raw| -> [4, 8)
      {
        const int rowm = tid & 127;
        const float4 d4 = (p0 + rowm < P && tid < 128) ? reinterpret_cast<const float4*>(d_raw)[p0 + rowm]
                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
        const float m = fmaxf(fmaxf(fabsf(d4.x), fabsf(d4.y)), fmaxf(fabsf(d4.z), fabsf(d4.w)));
        uint32_t mb = __float_as_uint(m);
        mb = __reduce_max_sync(0xffffffffu, mb);
        if (lane == 0) atomicMax(&s_max[it & 1], mb);
        cta_bar();
        if (tid == 0) s_max[(it + 1) & 1] = 0u;  // reset the other slot for the next tile
      }
      const uint32_t ex = (s_max[it & 1] >> 23) & 0xFFu;
      const bool scaled = ex >= 3u && ex <= 254u;
      const float sc = scaled ? __uint_as_float((256u - ex) << 23) : 1.f;
      const float us = (scaled ? __uint_as_float((ex - 2u) << 23) : 1.f) * kActInv;  // activations are stored / 16

      float chain[64];  // G_{t+1} W_{t+1}[:, :128] of this warpgroup's rows (the previous event's chain MMA)
#pragma unroll
      for (int i = 0; i < 64; ++i) chain[i] = 0.f;
      for (int e = 0; e < E; ++e) {
        const int t = E - 1 - e;
        const GemmLayer& g = p.g[t];
        int hsel = -1;
        if (p.h[0].src == t) hsel = 0;
        if (p.n_head > 1 && p.h[1].src == t) hsel = 1;
        const float* hw = hsel == 1 ? s_headw + hw1 : s_headw;
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
                                         (size_t)pt[i] * (g.n >> 5);
              mw[i][m] = valid[i] ? __ldg(mask_row + m) : 0u;
            }
          }
        // d_raw of this thread's rows at the tile scale (re-read per event rather than kept live through the MMAs), and
        // the head outputs' entries of it selected once (a runtime index into dr would put it in local memory)
        float dr[2][4], hd[2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float4 d4 = valid[i] ? reinterpret_cast<const float4*>(d_raw)[pt[i]] : make_float4(0.f, 0.f, 0.f, 0.f);
          dr[i][0] = d4.x * sc; dr[i][1] = d4.y * sc; dr[i][2] = d4.z * sc; dr[i][3] = d4.w * sc;
        }
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int k = (hcol + c) & 3;
            hd[i][c] = k == 0 ? dr[i][0] : k == 1 ? dr[i][1] : k == 2 ? dr[i][2] : dr[i][3];
          }
        // ---------------- epilogue: G_t of this thread's elements -> hi / lo -> the G tile ----------------
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
              *reinterpret_cast<uint32_t*>(sG + off) = hi;
              *reinterpret_cast<uint32_t*>(sG + 32768 + off) = lo;
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
            *reinterpret_cast<uint4*>(sG + tile_piece(r, 8, 128)) = make_uint4(h01, h23, 0u, 0u);
            *reinterpret_cast<uint4*>(sG + 32768 + tile_piece(r, 8, 128)) = make_uint4(l01, l23, 0u, 0u);
#pragma unroll
            for (int fb = 9; fb < 16; ++fb) {
              *reinterpret_cast<uint4*>(sG + tile_piece(r, fb, 128)) = z4;
              *reinterpret_cast<uint4*>(sG + 32768 + tile_piece(r, fb, 128)) = z4;
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
                const uint32_t lo16 = (ray_slot[i] == 2 * k && valid[i]) ? 0x3C00u : 0u;
                const uint32_t hi16 = (ray_slot[i] == 2 * k + 1 && valid[i]) ? 0x3C00u : 0u;
                w[k] = lo16 | (hi16 << 16);
              }
              const int r = 64 * wg + r0 + 8 * i;
              *reinterpret_cast<uint4*>(sInd + tile_piece(r, 0, 16)) = make_uint4(w[0], w[1], w[2], w[3]);
              *reinterpret_cast<uint4*>(sInd + tile_piece(r, 1, 16)) = make_uint4(w[4], w[5], w[6], w[7]);
            }
          }
          if (p.use_viewdirs && tid < n_rays_tile * 3) {
            const int jr = tid / 3, c = tid - 3 * jr;
            const float vv = rays[(first_ray + jr) * ray_stride + 8 + c];
            encode_coord(vv, c, p.inc_dir, 0, p.n_freq_dir, p.freq_dir, s_encd + jr * 32);
          }
        }
        fence_proxy_async();
        cta_bar();  // the G tile (and the indicator tile) complete

        if (e + 1 < E) {
          // ---- chain: chain[p][k] = 2^11 sum_n G_t[p][n] W_t[n][k], N = k_h = 128, K = n: A = this warpgroup's rows of
          // the G tile (K-major), B = the three weight copies from the ring (one k-step per stage)
          const uint64_t a_hi = make_desc(smem_u32(sG) + (uint32_t)wg * 16384u, 128, 2048);
          const uint64_t b_ring = make_desc(smem_u32(sm + mp.ring), 2048, 128);
          uint32_t prev = 0;
          wgmma_fence();
          for (int ks = 0; ks < (g.n >> 4); ++ks) {
            const uint32_t st = pp.stage;
            mbar_wait(&w_full[st], pp.phase);
            const uint64_t b_hs = desc_adv(b_ring, st * (uint32_t)kWStage);
            const uint64_t ah = desc_adv(a_hi, ks * 256u);
            wgmma_f16<128>(chain, ah, b_hs, ks > 0 ? 1 : 0);
            wgmma_f16<128>(chain, desc_adv(ah, 32768u), desc_adv(b_hs, 2 * 2048u), 1);
            wgmma_f16<128>(chain, ah, desc_adv(b_hs, 4 * 2048u), 1);
            wgmma_commit();
            if (ks > 0) {
              wgmma_wait<1>();
              reg_fence(chain);
              if (lane == 0) mbar_arrive(&w_empty[prev]);
            }
            prev = st;
            pp.advance(n_stages);
          }
          wgmma_wait<0>();
          reg_fence(chain);
          if (lane == 0) mbar_arrive(&w_empty[prev]);
        }

        // ---- weight-gradient jobs of this event
        const int nj = bp.n_jobs[e];
        for (int i = 0; i < nj; ++i) {
          const BwdJob& jq = bp.jobs[e][i];
          const int w = jq.n_b;
          const uint32_t fstr = (uint32_t)(w >> 3) * 128u;  // bytes between 8-point blocks of the activation tile
          mbar_wait(x_full, x_ph);
          x_ph ^= 1;
          // Called once per job by every consumer thread as soon as its warpgroup's MMAs are complete: once both
          // warpgroups are through, nothing reads the activation tile any more and thread 0 requests the next job's, so
          // that the load overlaps this job's drain instead of following it.
          auto release_x = [&]() {
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
          if (jq.kind == 1) {
            // head job: A = activation tile (rows = its features, MN-major), B = d_raw (feature rows 64..79 of the G tile)
            if (64 * wg < jq.nrows) {
              float acc[8], dummy[8];
              const uint64_t xa = make_desc(smem_u32(sX) + (uint32_t)wg * 1024u, fstr, 128);
              const uint64_t db = make_desc(smem_u32(sG) + 1024u, 2048, 128);
              // residual products first: A_lo B_hi + A_hi B_lo (job_mma's scheme with B's lo block 32 KB on)
              job_mma<16, false>(acc, dummy, xa, 32768u, 2 * fstr, db, 32768u, 4096u, 0);
              release_x();
              const HeadLayer& h = p.h[jq.dst_head];
#pragma unroll
              for (int jj = 0; jj < 2; ++jj)
#pragma unroll
                for (int ii = 0; ii < 2; ++ii)
#pragma unroll
                  for (int cc = 0; cc < 2; ++cc) {
                    const int k = 64 * wg + r0 + 8 * ii, c = 8 * jj + 2 * q + cc - h.out_col;
                    if (k < h.k && c >= 0 && c < h.n_out)
                      atomicAdd(gb + bm.xh + jq.dst_head * 512 + c * 128 + k, to_fix(acc[4 * jj + 2 * ii + cc] * us));
                  }
            } else {
              release_x();
            }
          } else if (64 * wg < jq.nrows || (i == 0 && e == 0 && p.use_viewdirs)) {
            // (warpgroup 1 of layers_dir[0]'s first job only sums the d_raw rows 64..67 of the indicator product)
            const uint64_t ga = make_desc(smem_u32(sG) + (uint32_t)wg * 1024u, 2048, 128);  // G^T: rows = features
            const uint64_t xb = make_desc(smem_u32(sX), fstr, 128);
            const uint64_t id = make_desc(smem_u32(sInd), 256, 128);
            float acc_i[8];
            unsigned long long* gdst = gb + jq.gb_off;
#define NB_JOB(NN)                                                                                   \
  {                                                                                                  \
    float acc[NN / 2];                                                                               \
    if (i == 0) job_mma<NN, true>(acc, acc_i, ga, 32768u, 4096u, xb, 32768u, 2 * fstr, id);          \
    else job_mma<NN, false>(acc, acc_i, ga, 32768u, 4096u, xb, 32768u, 2 * fstr, id);                \
    release_x();                                                                                     \
    if (64 * wg < jq.nrows) job_drain<NN>(acc, us, gdst, wg);                                        \
  }
            if (w == 128) NB_JOB(128) else if (w == 64) NB_JOB(64) else if (w == 48) NB_JOB(48)
            else if (w == 32) NB_JOB(32) else NB_JOB(16)
#undef NB_JOB
            if (i == 0) {
              // indicator sums of this layer: bias gradient (all rays) and, for layers_dir[0], the direction-encoding
              // part of its weight gradient (per-ray sums x direction encodings, below)
              const float su = us * kActScale;  // the indicator is an exact 1, not an activation / 16
#pragma unroll
              for (int ii = 0; ii < 2; ++ii) {
                const int n = 64 * wg + r0 + 8 * ii;
                float tot = acc_i[2 * ii] + acc_i[2 * ii + 1] + acc_i[4 + 2 * ii] + acc_i[4 + 2 * ii + 1];
                tot += __shfl_xor_sync(0xffffffffu, tot, 1);
                tot += __shfl_xor_sync(0xffffffffu, tot, 2);
                if (q == 0) {
                  if (n < g.n) s_bgrad[g.cum_n + n] += tot * su;
                  if (e == 0 && p.use_viewdirs && n >= 64 && n < 68) s_bgrad[p.enc_cum[0] + n - 64] += tot * su;  // d_rgb, d_sigma sums
                }
                if (e == 0 && p.use_viewdirs && n < 64) {
                  s_sums[n * 16 + 2 * q] = acc_i[2 * ii] * su;
                  s_sums[n * 16 + 2 * q + 1] = acc_i[2 * ii + 1] * su;
                  s_sums[n * 16 + 8 + 2 * q] = acc_i[4 + 2 * ii] * su;
                  s_sums[n * 16 + 9 + 2 * q] = acc_i[4 + 2 * ii + 1] * su;
                }
              }
            }
          } else {
            release_x();
          }
          if (e == 0 && i == 0 && p.use_viewdirs) {
            cta_bar();  // the per-ray sums of both warpgroups are in place
            for (int idx = tid; idx < 64 * p.dim_dir; idx += 128 * kWG) {
              const int n = idx / p.dim_dir, k = idx - n * p.dim_dir;
              float a = 0.f;
              for (int jr = 0; jr < n_rays_tile; ++jr) a = fmaf(s_sums[n * 16 + jr], s_encd[jr * 32 + k], a);
              s_dacc[n * 28 + k] += a;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  // ---- the bias / direction-encoding accumulators of this CTA go to the blob
  for (int i = tid; i < p.enc_cum[0] + 8; i += kThreadsB) atomicAdd(gb + bm.xb + i, to_fix(s_bgrad[i]));
  for (int i = tid; i < 64 * 28; i += kThreadsB) atomicAdd(gb + bm.xd + i, to_fix(s_dacc[i]));
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
          if (rr >= j.row0 && rr < j.row0 + j.nrows && col < j.ncols)
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
int64_t bwd_tc_scratch_floats(const Plan& p) {
  int total = 0;
  bwd_jobs(p, 0, nullptr, &total);
  return 2 * (int64_t)blob_map(p, total).words;
}

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

int launch_mlp_bwd_tc(const Plan& p, const float* blob, const float* rays, int ray_stride, int64_t n_rays, int n_samples,
                      const float* d_raw, const float* stash, float* gblob, float* flat_grad, cudaStream_t s) {
  const int64_t P = n_rays * n_samples;
  const int64_t tiles = (P + kTileRows - 1) / kTileRows;
  const int sms = device_sms();
  const int grid = (int)(tiles < sms ? tiles : sms);
  const BwdPlan bp = make_bwd_plan(p);
  const BlobMap bm = blob_map(p, bp.gb_total);
  int rc = check_cuda(cudaMemsetAsync(gblob, 0, (size_t)bm.words * 8, s), "mlp_bwd_tc blob memset");
  if (rc) return rc;
  const size_t bytes = (size_t)smem_map_b(p).total + 1024;
  rc = check_cuda(cudaFuncSetAttribute(mlp_bwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes),
                  "mlp_bwd_tc smem attribute");
  if (rc) return rc;
  mlp_bwd_tc_kernel<<<grid, kThreadsB, bytes, s>>>(p, blob, rays, ray_stride, d_raw, stash, P, n_samples, tiles, gblob, bp);
  count_launch();
  rc = check_cuda(cudaGetLastError(), "mlp_bwd_tc launch");
  if (rc) return rc;
  const int blocks = (bm.words + 255) / 256;
  unpack_grad_kernel<<<blocks, 256, 0, s>>>(p, bp, reinterpret_cast<const unsigned long long*>(gblob), flat_grad);
  count_launch();
  return check_cuda(cudaGetLastError(), "unpack_grad launch");
}

}  // namespace nerfb200
