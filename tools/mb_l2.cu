// mb_l2.cu -- micro-benchmarks that size the chain kernels' weight stream (dev tool, not product):
//   (1) cp.async.bulk global(L2-resident) -> shared, all SMs, ring of 4 stages: aggregate GB/s vs chunk size
//   (2) cp.reduce.async.bulk shared -> global .add.f32 and .add.u64 (the backward's fixed-point gradient blob) into a
//       small L2-resident region: aggregate GB/s
//   (3) red.global.add.u64 from the registers of a wgmma accumulator fragment into a 1.31 MB region (fragment-blocked
//       and row-major layouts): aggregate GB/s
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bin/mb_l2 tools/mb_l2.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c)); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile("{\n.reg .pred p;\nW1:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D1;\nbra W1;\nD1:\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

constexpr int kStages = 4;
__global__ void __launch_bounds__(64, 1) stream_kernel(const uint8_t* __restrict__ src, size_t src_bytes, uint32_t chunk, int iters, long long* cyc) {
  extern __shared__ __align__(1024) uint8_t sm[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm);
  uint8_t* ring = sm + 1024;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) mbar_init(&bars[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t0 = clock64();
    size_t off = ((size_t)blockIdx.x * 7919u * chunk) % (src_bytes - chunk);
    off &= ~(size_t)127;
    // prime
    for (int i = 0; i < kStages && i < iters; ++i) {
      mbar_expect(&bars[i], chunk);
      bulk_g2s(ring + (size_t)i * chunk, src + off, chunk, &bars[i]);
      off += chunk; if (off + chunk > src_bytes) off = 0;
    }
    for (int it = 0; it < iters; ++it) {
      const int s = it % kStages; const uint32_t ph = (it / kStages) & 1;
      mbar_wait(&bars[s], ph);
      if (it + kStages < iters) {
        mbar_expect(&bars[s], chunk);
        bulk_g2s(ring + (size_t)s * chunk, src + off, chunk, &bars[s]);
        off += chunk; if (off + chunk > src_bytes) off = 0;
      }
    }
    cyc[blockIdx.x] = clock64() - t0;
  }
}

template <bool kU64>
__global__ void __launch_bounds__(128, 1) reduce_kernel(void* __restrict__ dst_v, size_t dst_bytes, uint32_t chunk, int iters) {
  extern __shared__ __align__(1024) uint8_t sm[];
  uint8_t* dst = reinterpret_cast<uint8_t*>(dst_v);
  if (kU64) {
    unsigned long long* tile = reinterpret_cast<unsigned long long*>(sm);
    for (uint32_t i = threadIdx.x; i < chunk / 8; i += blockDim.x) tile[i] = 1ull;
  } else {
    float* tile = reinterpret_cast<float*>(sm);
    for (uint32_t i = threadIdx.x; i < chunk / 4; i += blockDim.x) tile[i] = 1.0f;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    size_t off = ((size_t)blockIdx.x * 104729u * chunk) % (dst_bytes - chunk);
    off &= ~(size_t)127;
    for (int it = 0; it < iters; ++it) {
      if (kU64)
        asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.u64 [%0], [%1], %2;" ::"l"(dst + off), "r"(smem_u32(sm)), "r"(chunk) : "memory");
      else
        asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(dst + off), "r"(smem_u32(sm)), "r"(chunk) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      if ((it & 3) == 3) asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory");
      off += chunk; if (off + chunk > dst_bytes) off = 0;
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

// (3) red.global.add.u64 straight from registers: two warpgroups per SM, each thread holding the 64 fp32 accumulator
// registers of a wgmma m64n128 fragment (rows 16 warp + lane / 4 (+ 8), columns 8 j + 2 (lane & 3) (+ 1)); a warpgroup
// job adds its 64 x 128 block of words into one of kRedJobs such blocks.  kFrag: the blob stores each 8 x 8 (row-octet,
// column-octet) block contiguously, column parity first, so one warp-wide red covers 256 contiguous bytes; otherwise the
// block is row-major (a warp-wide red touches 8 rows x 4 strided words).
constexpr int kRedJobs = 21;   // 21 x 64 KB = 1.31 MB, one tile's weight gradients in the A1 backward
template <bool kFrag>
__global__ void __launch_bounds__(256, 1) red_kernel(unsigned long long* __restrict__ dst, int iters) {
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, q = lane & 3;
  for (int it = 0; it < iters; ++it) {
    unsigned long long* job = dst + (size_t)((blockIdx.x * 2 + wg + it * 5) % kRedJobs) * 8192;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const size_t w = kFrag ? (size_t)((2 * warp + i) * 16 + j) * 64 + c * 32 + lane
                                 : (size_t)(16 * warp + (lane >> 2) + 8 * i) * 128 + 8 * j + 2 * q + c;
          asm volatile("red.global.add.u64 [%0], %1;" ::"l"(job + w), "l"((unsigned long long)(it + lane + c)) : "memory");
        }
  }
}

int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  printf("%s, SMs %d\n", prop.name, sms);
  uint8_t* src; const size_t src_bytes = 1536 * 1024; cudaMalloc(&src, src_bytes); cudaMemset(src, 1, src_bytes);
  long long* cyc; cudaMalloc(&cyc, sizeof(long long) * 1024);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
  const uint32_t chunks[] = {8192, 12288, 24576, 32768, 49152};
  for (uint32_t chunk : chunks) {
    const int iters = (int)((size_t)256 * 1024 * 1024 / chunk / 4);
    const size_t smem = 1024 + (size_t)kStages * chunk;
    for (int grid : {sms, sms / 2}) {
      stream_kernel<<<grid, 64, smem>>>(src, src_bytes, chunk, 64, cyc);  // warm
      cudaEventRecord(e0);
      stream_kernel<<<grid, 64, smem>>>(src, src_bytes, chunk, iters, cyc);
      cudaEventRecord(e1); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      long long c0; cudaMemcpy(&c0, cyc, 8, cudaMemcpyDeviceToHost);
      const double bytes = (double)grid * iters * chunk;
      printf("stream chunk %6u grid %3d: %.3f ms  %.1f GB/s  (%.1f B/cyc/SM by CTA0 clock, %.0f MHz)\n", chunk, grid, ms, bytes / ms * 1e-6,
             (double)iters * chunk / (double)c0, (double)c0 / ms * 1e-3);
    }
  }
  // the destination is sized like the fine backward's gradient blob (~0.6 MB): L2-resident, every SM adds into it
  void* dst; const size_t dst_bytes = 672 * 1024; cudaMalloc(&dst, dst_bytes); cudaMemset(dst, 0, dst_bytes);
  cudaFuncSetAttribute(reduce_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
  cudaFuncSetAttribute(reduce_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
  for (int u64 = 0; u64 < 2; ++u64)
    for (uint32_t chunk : {8192u, 16384u, 65536u}) {
      auto kern = u64 ? reduce_kernel<true> : reduce_kernel<false>;
      const int iters = (int)((size_t)64 * 1024 * 1024 / chunk);
      kern<<<sms, 128, chunk>>>(dst, dst_bytes, chunk, 16);
      cudaEventRecord(e0);
      kern<<<sms, 128, chunk>>>(dst, dst_bytes, chunk, iters);
      cudaEventRecord(e1); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      printf("reduce-add .%s chunk %6u: %.3f ms  %.1f GB/s aggregate\n", u64 ? "u64" : "f32", chunk, ms,
             (double)sms * iters * chunk / ms * 1e-6);
    }
  unsigned long long* rdst; cudaMalloc(&rdst, (size_t)kRedJobs * 8192 * 8); cudaMemset(rdst, 0, (size_t)kRedJobs * 8192 * 8);
  for (int frag = 1; frag >= 0; --frag) {
    auto kern = frag ? red_kernel<true> : red_kernel<false>;
    const int iters = 512;
    kern<<<sms, 256>>>(rdst, 16);
    cudaEventRecord(e0);
    kern<<<sms, 256>>>(rdst, iters);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("red.global.add.u64 from registers, %s layout: %.3f ms  %.1f GB/s aggregate\n", frag ? "fragment" : "row-major",
           ms, (double)sms * iters * 2 * 65536 / ms * 1e-6);
  }
  printf("err: %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
