// Common sm_90a device helpers: mbarrier, TMA (cp.async.bulk.tensor), wgmma shared-memory
// descriptors.  Hand-written inline PTX — no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {

// ----------------------------------------------------------------------------- error state
// C-ABI convention (include/b200_e2eft.h): 0 ok, <0 invalid argument, >0 cudaError_t.
void set_last_error(const char* fmt, ...);
#define B200_CHECK_ARG(cond, ...)                    \
  do {                                               \
    if (!(cond)) {                                   \
      b200::set_last_error(__VA_ARGS__);             \
      return -1;                                     \
    }                                                \
  } while (0)
#define B200_CHECK_LAUNCH(what)                                                    \
  do {                                                                             \
    cudaError_t e__ = cudaGetLastError();                                          \
    if (e__ != cudaSuccess) {                                                      \
      b200::set_last_error("%s: %s", what, cudaGetErrorString(e__));               \
      return (int)e__;                                                             \
    }                                                                              \
  } while (0)

// ----------------------------------------------------------------------------- misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\t"
      "elect.sync R|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  // order generic-proxy smem accesses before later async-proxy ones (TMA writes, wgmma reads)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (error surfaces to the host) instead of hanging the GPU.  No printf here: a
// function call inside a kernel that issues wgmma makes ptxas serialise the whole wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#pragma unroll 1
  for (int i = 0; i < 64; ++i)
    if (mbar_try_wait(bar, parity)) return;           // fast path: no clock reads
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000LL) __trap();      // ~4 s at 2 GHz
  }
}

// ----------------------------------------------------------------------------- TMA loads
// L2 cache-hint policies (createpolicy-encoded constants, as used by CUTLASS TMA::CacheHintSm90)
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0,
                                            int c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0,
                                            int c1, int c2, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(hint)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0,
                                            int c1, int c2, int c3, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "l"(hint)
      : "memory");
}

// ----------------------------------------------------------------------------- wgmma descriptors
// Shared-memory matrix descriptor (64-bit), sm_90 format:
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset>>4 [49,52) base offset = 0      [62,64) layout: 1 = SWIZZLE_128B
// K-major SWIZZLE_128B tile (rows of 64 x 16-bit = 128 B, 8-row groups 1024 B apart): LBO unused (16), SBO = 1024.
// MN-major SWIZZLE_128B tile ([k-row][64 rows] atoms): LBO = byte distance of 64-row atoms, SBO = of 8-k-row groups.
// The swizzle is a function of the absolute smem address, so a start address inside a 1024-byte atom (a k-step of
// +32 B, or a whole 128-byte row further on) needs no base offset.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                    uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// ----------------------------------------------------------------------------- host: tensor maps
// cuTensorMapEncodeTiled is fetched through cudaGetDriverEntryPoint (no -lcuda link dependency).
int encode_tmap(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box,
                const uint32_t* elem_strides, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16);

int sm_count();            // of the CURRENT device (cached per device)
int current_device();      // cudaGetDevice, -1 on error
constexpr int kMaxDevices = 64;   // per-device caches (function attributes are per context: one flag per device and kernel)

}  // namespace b200
