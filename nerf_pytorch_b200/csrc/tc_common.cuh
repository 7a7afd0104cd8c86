// tc_common.cuh -- inline-PTX helpers of the Hopper tensor-core path: mbarrier, bulk async copy (TMA engine), the wgmma
// shared-memory matrix descriptor and the fp16 x 2 operand split (the MMAs themselves: wgmma.cuh).
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace nerfb200 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// mbarriers and bulk copies take 32-bit shared-memory addresses (smem_u32): the hot loops keep them in registers instead
// of converting a generic pointer on every call
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// L2 eviction-priority policy for the weight stream: every CTA re-reads the same ~1 MB blob for every tile
// while GBs of stash stream through L2 in training, so the weights are pinned (evict_last) and the
// stash stores are marked streaming (st.global.cs) to keep them from pushing the weights out to HBM.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar), "l"(pol)
      : "memory");
}
// shared -> global bulk store (TMA engine, bulk async-group completion)
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes)
               : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// all committed bulk stores have finished READING their shared-memory source
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}

// wgmma shared-memory matrix descriptor, no swizzle ("interleave" layout type 0): 8-row core matrices (8 x 16 B).
// K-major operand: LBO = bytes between the two K halves of one instruction, SBO = bytes between 8-row groups along M/N;
// MN-major operand: LBO = bytes between 8-deep groups along K, SBO = bytes between 8-wide groups along M/N.
// Bit layout per the PTX ISA (cute::GMMA::GmmaDescriptor): [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4, base offset
// and layout type 0.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
// Advance a descriptor's 14-bit start-address field by `bytes` with one 32-bit add (descriptors are built once per
// layer; the MMA loops only move their start addresses).
__device__ __forceinline__ uint64_t desc_adv(uint64_t d, uint32_t bytes) {
  return (d & 0xFFFFFFFF00000000ull) | (uint64_t)((uint32_t)d + (bytes >> 4));
}
// fp16 x 2 split of a pair of fp32 values: hi = fp16(x), lo = fp16((x - hi) * 2^11); both packed with the FIRST
// value in the low half (= the lower K index of a 16-bit operand).
// The residual is scaled by 2^11 so that it is a NORMAL fp16 number whenever hi is (it would be subnormal below
// |x| = 0.125 otherwise and the split would degrade to 3e-8 absolute resolution): x = hi + lo * 2^-11 carries 22
// significant bits for 6.1e-5 <= |x| < 65504 and resolves 1.5e-11 absolutely below (tests/test_host_cpu.py).
// Conversions do NOT saturate: a value beyond the fp16 range becomes +-inf, the products turn into inf / NaN and
// the render output is visibly non-finite instead of silently clamped.
// Single-accumulator scheme of the chain kernels: the B operand (weights) comes in THREE copies
//     hs = w_hi * 2^11,   h = w_hi,   l = (w - w_hi) * 2^11          (all fp16; |w| < 32 or hs overflows to inf)
// and one k-step issues  a_hi*hs + a_lo*h + a_hi*l  =  2^11 * (a*w)  into ONE fp32 accumulator.
constexpr float kLoScale = 2048.f, kLoInv = 1.f / 2048.f;
constexpr float kActScale = 0.0625f, kActInv = 16.f;  // forward A operands / stash tiles hold activation / 16
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  float h0, h1;
  asm("{\n.reg .b16 a, b;\nmov.b32 {a, b}, %2;\ncvt.f32.f16 %0, a;\ncvt.f32.f16 %1, b;\n}\n" : "=f"(h0), "=f"(h1) : "r"(hi));
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"((x1 - h1) * kLoScale), "f"((x0 - h0) * kLoScale));
}
// The same split from Y = 2048 x (exact scaling): hi = fp16(x), lo = fp16(Y - 2048 hi), one FMA per element instead of
// subtract + multiply.  Bit-identical to split_f16x2(Y0 / 2048, Y1 / 2048): x - hi is exact in fp32.
__device__ __forceinline__ void split_f16x2_y(float Y0, float Y1, float x0, float x1, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  float h0, h1;
  asm("{\n.reg .b16 a, b;\nmov.b32 {a, b}, %2;\ncvt.f32.f16 %0, a;\ncvt.f32.f16 %1, b;\n}\n" : "=f"(h0), "=f"(h1) : "r"(hi));
  const float r0 = fmaf(h0, -kLoScale, Y0), r1 = fmaf(h1, -kLoScale, Y1);
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
}
// hi = fp16(x) alone (same packing): the operand of the single-pass forward, which drops the lo half
__device__ __forceinline__ uint32_t f16x2_hi(float x0, float x1) {
  uint32_t hi;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  return hi;
}
// the three weight copies of one pair (same packing)
__device__ __forceinline__ void split_w3(float w0, float w1, uint32_t& hs, uint32_t& h, uint32_t& l) {
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(w1), "f"(w0));
  float h0, h1;
  asm("{\n.reg .b16 a, b;\nmov.b32 {a, b}, %2;\ncvt.f32.f16 %0, a;\ncvt.f32.f16 %1, b;\n}\n" : "=f"(h0), "=f"(h1) : "r"(h));
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hs) : "f"(h1 * kLoScale), "f"(h0 * kLoScale));
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(l) : "f"((w1 - h1) * kLoScale), "f"((w0 - h0) * kLoScale));
}
// NaN-propagating max (fmaxf would turn the NaN of an out-of-range operand into a plausible 0)
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// ---------------------------------------------------------------------------------------------------------------
// Operand tiles.  A 128-point x (8 F)-feature block of fp16 values is kept as 16 x F core matrices of 128 bytes,
//     T[pb = point / 8][fb = feature / 8][point % 8][feature % 8]            (pb-major, F * 128 bytes per pb)
// and a value x as two such blocks, hi = fp16(x) then lo = fp16((x - hi) 2^11)  (split_f16x2), 16 F 128 bytes apart.
// The SAME bytes serve wgmma as
//   K-major  operand (rows = points,   K = features): SBO = F * 16 (next 8 points),   LBO = 128 (next 8 features)
//   MN-major operand (rows = features, K = points)  : SBO = 128 (next 8 features),    LBO = F * 16 (next 8 points)
// so the training forward writes every layer's activation tile ONCE -- into HBM, straight from the accumulator
// registers that also fill the next layer's shared-memory operand -- and the fused backward (mlp_tc_bwd.cu) bulk-copies
// it back and uses it as the MN-major B operand of the weight-gradient MMAs unchanged.
// ---------------------------------------------------------------------------------------------------------------
__host__ __device__ inline int tile_half_bytes(int n_feat) { return 16 * (n_feat >> 3) * 128; }   // one of hi / lo
__host__ __device__ inline int tile_bytes(int n_feat) { return 2 * tile_half_bytes(n_feat); }      // = 128 * n * 4
// byte offset of the 16-byte piece (point row, features [8 fb, 8 fb + 8)) inside the hi (or lo) block
__host__ __device__ inline int tile_piece(int row, int fb, int n_feat) {
  return (row >> 3) * (n_feat >> 3) * 128 + fb * 128 + (row & 7) * 16;
}
// register -> global reduction without a return value (the thread does not wait for it): *gdst += v, 64-bit integers
__device__ __forceinline__ void red_add_u64(unsigned long long* gdst, unsigned long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(gdst), "l"(v) : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// The persistent kernels (mlp_tc.cu forward, mlp_tc_bwd.cu fused backward): one CTA per SM walks tiles blockIdx.x,
// blockIdx.x + gridDim.x, ...; dynamic shared memory is used from a 1 KB-aligned base, fixed regions first and the weight
// ring in whatever is left of the budget.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kSmemAlign = 1024;
constexpr int kSmemBudget = 232448 - kSmemAlign;  // 227 KB of dynamic shared memory per block minus the alignment slack
constexpr int kMaxStages = 6;                     // weight-ring stages at most (the mbarriers are laid out for this many)
constexpr int kMaxRaysPerTile = 10;               // rays one tile may touch (tc_supported: at least 15 samples per ray)

// stages of `stage_bytes` that fit from `ring` (the 1 KB-aligned end of the fixed regions) to the end of the budget
__host__ __device__ inline int ring_depth(int ring, int stage_bytes) {
  const int ns = (kSmemBudget - ring) / stage_bytes;
  return ns < kMaxStages ? ns : kMaxStages;
}
__device__ __forceinline__ uint8_t* smem_base() {
  extern __shared__ uint8_t smem_raw[];
  return smem_raw + ((kSmemAlign - (smem_u32(smem_raw) & (kSmemAlign - 1))) & (kSmemAlign - 1));
}

// the head that reads gemm layer e's output: 0, 1 or -1
__host__ __device__ inline int head_of(const Plan& p, int e) {
  int hsel = -1;
  if (p.h[0].src == e) hsel = 0;
  if (p.n_head > 1 && p.h[1].src == e) hsel = 1;
  return hsel;
}

// Ray geometry.  Fewer than 2^31 points per call (check_mlp_args), so the divisions are 32-bit instead of emulated
// 64-bit ones.  The rays of the `rows` points from p0 (the last point stands in for points past the end):
struct TileRays {
  int64_t first;
  int n;
};
__device__ __forceinline__ TileRays tile_rays(int64_t p0, int rows, int64_t P, int S) {
  TileRays tr;
  tr.first = (int64_t)((uint32_t)(p0 < P ? p0 : P - 1) / (uint32_t)S);
  const int64_t last_pt = (p0 + rows - 1 < P) ? p0 + rows - 1 : P - 1;
  tr.n = (int)((uint32_t)last_pt / (uint32_t)S) - (int)tr.first + 1;
  return tr;
}
// per-tile state of a consumer thread: its two accumulator rows p0 + r0 and p0 + r0 + 8 (r0 = 16 warp + lane / 4 in the
// warpgroup whose first point is p0); rows past the end are invalid and alias the last point
struct RowState {
  int pt[2];         // a point index fits in an int: fewer than 2^31 points per call
  bool valid[2];
  int ray_slot[2];  // ray - first_ray
};
__device__ __forceinline__ RowState row_state(int64_t p0, int r0, int64_t P, int S, int64_t first_ray) {
  RowState rs;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int64_t pt = p0 + r0 + 8 * i;
    rs.valid[i] = pt < P;
    rs.pt[i] = (int)(pt < P ? pt : P - 1);
    rs.ray_slot[i] = (int)((uint32_t)rs.pt[i] / (uint32_t)S - first_ray);
  }
  return rs;
}
// the same over an occupancy grid's row map (occupancy.cu): rows p0 + r0 (+ 8) of the map; a padding row, or any row of a
// block past the last (live = false), is invalid and stands in for the block's first ray's first point
__device__ __forceinline__ RowState map_row_state(const int* __restrict__ map, int64_t p0, int r0, bool live, int S,
                                                  int64_t first_ray) {
  RowState rs;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = live ? map[p0 + r0 + 8 * i] : -1;
    rs.valid[i] = m >= 0;
    rs.pt[i] = m >= 0 ? m : (int)(first_ray * S);
    rs.ray_slot[i] = (int)((uint32_t)rs.pt[i] / (uint32_t)S - first_ray);
  }
  return rs;
}

// Weight ring: n_stages stages of kStage bytes from `base`, filled by one producer thread with bulk copies from the
// L2-resident blob and read by the consumer warpgroups' MMAs.  full[i] (bars + 8 i, one producer arrival + the bytes):
// stage i has landed; empty[i] (bars + 8 (kMaxStages + i), one arrival per consumer warp): every consumer warp's MMAs
// on it are complete.  Each role walks the ring with its own copy (stage, phase).
template <int kStage>
struct WeightRing {
  uint32_t base, bars, n_stages;
  uint32_t stage = 0, phase = 0;
  uint32_t prev = 0;      // consumer: the stage whose MMAs may still be in flight ...
  bool has_prev = false;  // ... if any (false at the start of each pass over the ring)
  __device__ __forceinline__ uint32_t full(uint32_t s) const { return bars + 8 * s; }
  __device__ __forceinline__ uint32_t empty(uint32_t s) const { return bars + 8 * (kMaxStages + s); }
  __device__ __forceinline__ void init(uint32_t consumer_warps) const {
    for (int i = 0; i < kMaxStages; ++i) {
      mbar_init(full(i), 1);
      mbar_init(empty(i), consumer_warps);
    }
  }
  __device__ __forceinline__ void advance() {
    if (++stage == n_stages) { stage = 0; phase ^= 1; }
  }
  // producer: once every consumer warp has handed the next stage back, fill it with n bulk copies of `bytes`, src_step
  // apart in the blob and packed in the stage (evict_last policy `pol`)
  __device__ __forceinline__ void fill(const uint8_t* src, uint32_t n, uint32_t bytes, size_t src_step, uint64_t pol) {
    const uint32_t f = full(stage), dst = base + stage * kStage;
    mbar_wait(empty(stage), phase ^ 1);
    mbar_arrive_expect_tx(f, n * bytes);
    for (uint32_t i = 0; i < n; ++i) bulk_g2s_hint(dst + i * bytes, src + i * src_step, bytes, f, pol);
    advance();
  }
  // consumer: wait until the next stage has landed; returns its index
  __device__ __forceinline__ uint32_t acquire() const {
    mbar_wait(full(stage), phase);
    return stage;
  }
  // consumer, after committing the MMAs on the acquired stage: hand back the stage before it, if the pass has one,
  // once its MMAs are complete -- wait_group 1 leaves the group just committed in flight
  template <int R>
  __device__ __forceinline__ void release_behind(float (&acc)[R]) {
    if (has_prev) {
      wgmma_wait<1>();
      reg_fence(acc);
      if ((threadIdx.x & 31) == 0) mbar_arrive(empty(prev));
    }
    prev = stage;
    has_prev = true;
    advance();
  }
  // consumer, after the pass's last stage: wait for every MMA and hand back that stage
  template <int R>
  __device__ __forceinline__ void release_last(float (&acc)[R]) {
    wgmma_wait<0>();
    reg_fence(acc);
    if ((threadIdx.x & 31) == 0) mbar_arrive(empty(prev));
    has_prev = false;
  }
};

// Launch a persistent kernel: grid = min(tiles, SMs), `smem` bytes of dynamic shared memory past the aligned base.
template <typename Kernel, typename... Args>
int launch_persistent(Kernel kern, int64_t tiles, int threads, int smem, cudaStream_t s, const char* what,
                      const Args&... args) {
  const int sms = device_sms();
  const int grid = (int)(tiles < sms ? tiles : sms);
  const int bytes = smem + kSmemAlign;
  int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes), what);
  if (rc) return rc;
  kern<<<grid, threads, bytes, s>>>(args...);
  count_launch();
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace tc
}  // namespace nerfb200
