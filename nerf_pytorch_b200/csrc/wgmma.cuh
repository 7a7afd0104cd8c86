// wgmma.cuh -- warpgroup MMA wrappers (sm_90a): D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 operands from shared
// memory (matrix descriptors, tc_common.cuh make_desc), fp32 accumulator fragment in registers.  kTA / kTB = 1 reads
// the operand MN-major (transposed).
#pragma once
#include <stdint.h>

namespace nerfb200 {
namespace tc {

#define NB_F8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define NB_F32(o) NB_F8(o), NB_F8(o + 8), NB_F8(o + 16), NB_F8(o + 24)
template <int N, int kTA = 0, int kTB = 0>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t a, uint64_t b, int scale_d);

#define NB_WGMMA_16(TA, TB)                                                                         \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\nwgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "    \
               "{%0,%1,%2,%3,%4,%5,%6,%7}, "                                                                    \
               "%8, %9, p, 1, 1, " #TA ", " #TB ";\n}\n"                                          \
               : NB_F8(0) : "l"(a), "l"(b), "r"(scale_d))
template <> __device__ __forceinline__ void wgmma_f16<16, 0, 0>(float (&d)[8], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_16(0, 0); }
template <> __device__ __forceinline__ void wgmma_f16<16, 1, 1>(float (&d)[8], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_16(1, 1); }
template <> __device__ __forceinline__ void wgmma_f16<16, 0, 1>(float (&d)[8], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_16(0, 1); }
#undef NB_WGMMA_16
#define NB_WGMMA_32(TA, TB)                                                                         \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\nwgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "    \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, "                                                                    \
               "%16, %17, p, 1, 1, " #TA ", " #TB ";\n}\n"                                          \
               : NB_F8(0), NB_F8(8) : "l"(a), "l"(b), "r"(scale_d))
template <> __device__ __forceinline__ void wgmma_f16<32, 0, 0>(float (&d)[16], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_32(0, 0); }
template <> __device__ __forceinline__ void wgmma_f16<32, 1, 1>(float (&d)[16], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_32(1, 1); }
#undef NB_WGMMA_32
#define NB_WGMMA_48(TA, TB)                                                                         \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\nwgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "    \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, "                                                                    \
               "%24, %25, p, 1, 1, " #TA ", " #TB ";\n}\n"                                          \
               : NB_F8(0), NB_F8(8), NB_F8(16) : "l"(a), "l"(b), "r"(scale_d))
template <> __device__ __forceinline__ void wgmma_f16<48, 0, 0>(float (&d)[24], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_48(0, 0); }
template <> __device__ __forceinline__ void wgmma_f16<48, 1, 1>(float (&d)[24], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_48(1, 1); }
#undef NB_WGMMA_48
#define NB_WGMMA_64(TA, TB)                                                                         \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "    \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "                                                                    \
               "%32, %33, p, 1, 1, " #TA ", " #TB ";\n}\n"                                          \
               : NB_F32(0) : "l"(a), "l"(b), "r"(scale_d))
template <> __device__ __forceinline__ void wgmma_f16<64, 0, 0>(float (&d)[32], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_64(0, 0); }
template <> __device__ __forceinline__ void wgmma_f16<64, 1, 1>(float (&d)[32], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_64(1, 1); }
#undef NB_WGMMA_64
#define NB_WGMMA_128(TA, TB)                                                                         \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "    \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "                                                                    \
               "%64, %65, p, 1, 1, " #TA ", " #TB ";\n}\n"                                          \
               : NB_F32(0), NB_F32(32) : "l"(a), "l"(b), "r"(scale_d))
template <> __device__ __forceinline__ void wgmma_f16<128, 0, 0>(float (&d)[64], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_128(0, 0); }
template <> __device__ __forceinline__ void wgmma_f16<128, 1, 1>(float (&d)[64], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_128(1, 1); }
#undef NB_WGMMA_128
#define NB_WGMMA_256(TA, TB)                                                                         \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\nwgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "    \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, "                                                                    \
               "%128, %129, p, 1, 1, " #TA ", " #TB ";\n}\n"                                          \
               : NB_F32(0), NB_F32(32), NB_F32(64), NB_F32(96) : "l"(a), "l"(b), "r"(scale_d))
template <> __device__ __forceinline__ void wgmma_f16<256, 0, 0>(float (&d)[128], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_256(0, 0); }
template <> __device__ __forceinline__ void wgmma_f16<256, 1, 1>(float (&d)[128], uint64_t a, uint64_t b, int scale_d) { NB_WGMMA_256(1, 1); }
#undef NB_WGMMA_256
#undef NB_F32
#undef NB_F8

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }
// the accumulator registers are not to be touched by other instructions while a wgmma on them is in flight
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

}  // namespace tc
}  // namespace nerfb200
