// mb_l2.cu -- micro-benchmarks that size the chain kernels' weight stream (dev tool, not product):
//   (1) cp.async.bulk global(L2-resident) -> shared, all SMs, ring of 4 stages: aggregate GB/s vs chunk size
//   (2) cp.reduce.async.bulk shared -> global .add.f32 into a small L2-resident region: aggregate GB/s
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

__global__ void __launch_bounds__(128, 1) reduce_kernel(float* __restrict__ dst, size_t dst_floats, uint32_t chunk, int iters) {
  extern __shared__ __align__(1024) uint8_t sm[];
  float* tile = reinterpret_cast<float*>(sm);
  for (uint32_t i = threadIdx.x; i < chunk / 4; i += blockDim.x) tile[i] = 1.0f;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    size_t off = ((size_t)blockIdx.x * 104729u * (chunk / 4)) % (dst_floats - chunk / 4);
    off &= ~(size_t)31;
    for (int it = 0; it < iters; ++it) {
      asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(dst + off), "r"(smem_u32(tile)), "r"(chunk) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      if ((it & 3) == 3) asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory");
      off += chunk / 4; if (off + chunk / 4 > dst_floats) off = 0;
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  printf("SMs %d\n", sms);
  uint8_t* src; const size_t src_bytes = 1536 * 1024; cudaMalloc(&src, src_bytes); cudaMemset(src, 1, src_bytes);
  long long* cyc; cudaMalloc(&cyc, sizeof(long long) * 1024);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
  cudaFuncSetAttribute(reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
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
  float* dst; const size_t dst_floats = 672 * 1024 / 4; cudaMalloc(&dst, dst_floats * 4); cudaMemset(dst, 0, dst_floats * 4);
  for (uint32_t chunk : {16384u, 65536u}) {
    const int iters = (int)((size_t)64 * 1024 * 1024 / chunk);
    reduce_kernel<<<sms, 128, chunk>>>(dst, dst_floats, chunk, 16);
    cudaEventRecord(e0);
    reduce_kernel<<<sms, 128, chunk>>>(dst, dst_floats, chunk, iters);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("reduce-add chunk %6u: %.3f ms  %.1f GB/s aggregate\n", chunk, ms, (double)sms * iters * chunk / ms * 1e-6);
  }
  printf("err: %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
