// sm_90a warpgroup MMA wrappers: D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 operands, fp32 accumulators in registers.
// Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l): d[4j + {0,1}] = row 16w + l/4, columns
// 8j + 2(l%4) + {0,1}; d[4j + {2,3}] = the same columns of row 16w + l/4 + 8.
// TA / TB: 0 = operand K-major, 1 = MN-major (the transpose immediates of wgmma.mma_async).
#pragma once
#include <stdint.h>

namespace b200 {

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// accumulator operand lists: WG_R<i> = "%i,...,%(i+7)", WG_D<i> = the matching "+f"(d[..]) constraints

#define WG_R0 "%0,%1,%2,%3,%4,%5,%6,%7"
#define WG_R8 "%8,%9,%10,%11,%12,%13,%14,%15"
#define WG_R16 "%16,%17,%18,%19,%20,%21,%22,%23"
#define WG_R24 "%24,%25,%26,%27,%28,%29,%30,%31"
#define WG_R32 "%32,%33,%34,%35,%36,%37,%38,%39"
#define WG_R40 "%40,%41,%42,%43,%44,%45,%46,%47"
#define WG_R48 "%48,%49,%50,%51,%52,%53,%54,%55"
#define WG_R56 "%56,%57,%58,%59,%60,%61,%62,%63"
#define WG_R64 "%64,%65,%66,%67,%68,%69,%70,%71"
#define WG_R72 "%72,%73,%74,%75,%76,%77,%78,%79"
#define WG_R80 "%80,%81,%82,%83,%84,%85,%86,%87"
#define WG_R88 "%88,%89,%90,%91,%92,%93,%94,%95"
#define WG_R96 "%96,%97,%98,%99,%100,%101,%102,%103"
#define WG_R104 "%104,%105,%106,%107,%108,%109,%110,%111"
#define WG_R112 "%112,%113,%114,%115,%116,%117,%118,%119"
#define WG_R120 "%120,%121,%122,%123,%124,%125,%126,%127"
#define WG_D(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
    "+f"(d[i + 6]), "+f"(d[i + 7])

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32(float* d, uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {" WG_R0 "," WG_R8 "}, %16, %17, p, 1, 1, %19, %20;\n}"
               : WG_D(0), WG_D(8)
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float* d, uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "}, %32, %33, p, 1, 1, %35, %36;\n}"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24)
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float* d, uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "," WG_R32 "," WG_R40 "," WG_R48 "," WG_R56 "}, %64, %65, p, 1, 1, %67, %68;\n}"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24), WG_D(32), WG_D(40), WG_D(48), WG_D(56)
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n160(float* d, uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %82, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n160k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "," WG_R32 "," WG_R40 "," WG_R48 "," WG_R56 "," WG_R64 "," WG_R72 "}, %80, %81, p, 1, 1, %83, %84;\n}"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24), WG_D(32), WG_D(40), WG_D(48), WG_D(56), WG_D(64), WG_D(72)
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n192(float* d, uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %98, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "," WG_R32 "," WG_R40 "," WG_R48 "," WG_R56 "," WG_R64 "," WG_R72 "," WG_R80 "," WG_R88 "}, %96, %97, p, 1, 1, %99, %100;\n}"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24), WG_D(32), WG_D(40), WG_D(48), WG_D(56), WG_D(64), WG_D(72), WG_D(80), WG_D(88)
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256(float* d, uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "," WG_R32 "," WG_R40 "," WG_R48 "," WG_R56 "," WG_R64 "," WG_R72 "," WG_R80 "," WG_R88 "," WG_R96 "," WG_R104 "," WG_R112 "," WG_R120 "}, %128, %129, p, 1, 1, %131, %132;\n}"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24), WG_D(32), WG_D(40), WG_D(48), WG_D(56), WG_D(64), WG_D(72), WG_D(80), WG_D(88), WG_D(96), WG_D(104), WG_D(112), WG_D(120)
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

// A from registers (a[0..3] = the fp16 pairs of the accumulator-shaped 64 x 16 fragment), B MN-major
__device__ __forceinline__ void wgmma_m64n40_rs_bmn(float* d, const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n40k16.f32.f16.f16 {" WG_R0 "," WG_R8 ",%16,%17,%18,%19}, {%20, %21, %22, %23}, %24, 1, 1, 1, 1;"
               : WG_D(0), WG_D(8), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

__device__ __forceinline__ void wgmma_m64n64_rs_bmn(float* d, const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "}, {%32, %33, %34, %35}, %36, 1, 1, 1, 1;"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

__device__ __forceinline__ void wgmma_m64n80_rs_bmn(float* d, const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "," WG_R32 "}, {%40, %41, %42, %43}, %44, 1, 1, 1, 1;"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24), WG_D(32)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

__device__ __forceinline__ void wgmma_m64n160_rs_bmn(float* d, const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n160k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "," WG_R32 "," WG_R40 "," WG_R48 "," WG_R56 "," WG_R64 "," WG_R72 "}, {%80, %81, %82, %83}, %84, 1, 1, 1, 1;"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24), WG_D(32), WG_D(40), WG_D(48), WG_D(56), WG_D(64), WG_D(72)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

__device__ __forceinline__ void wgmma_m64n256_rs_bmn(float* d, const uint32_t (&a)[4], uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {" WG_R0 "," WG_R8 "," WG_R16 "," WG_R24 "," WG_R32 "," WG_R40 "," WG_R48 "," WG_R56 "," WG_R64 "," WG_R72 "," WG_R80 "," WG_R88 "," WG_R96 "," WG_R104 "," WG_R112 "," WG_R120 "}, {%128, %129, %130, %131}, %132, 1, 1, 1, 1;"
               : WG_D(0), WG_D(8), WG_D(16), WG_D(24), WG_D(32), WG_D(40), WG_D(48), WG_D(56), WG_D(64), WG_D(72), WG_D(80), WG_D(88), WG_D(96), WG_D(104), WG_D(112), WG_D(120)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

#undef WG_R0
#undef WG_R8
#undef WG_R16
#undef WG_R24
#undef WG_R32
#undef WG_R40
#undef WG_R48
#undef WG_R56
#undef WG_R64
#undef WG_R72
#undef WG_R80
#undef WG_R88
#undef WG_R96
#undef WG_R104
#undef WG_R112
#undef WG_R120
#undef WG_D

}  // namespace b200
