// Pieces shared by the flash attention forward (attention.cu) and backward (attention_bwd.cu) at head widths
// D in {40, 64, 80, 160}: the per-head tensor maps, the exp2 / fp16-pair helpers and the wgmma shapes the kernels use.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace b200 {

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // low half = a, high half = b
  return r;
}

// S (+)= A B^T with both operands K-major in smem: N = 32, 64 or 128 columns (keys in the forward / dQ kernel,
// queries in the dK/dV kernel)
template <int N>
__device__ __forceinline__ void wgmma_ss(float* s, uint64_t da, uint64_t db, int scale_d) {
  static_assert(N == 32 || N == 64 || N == 128, "wgmma_ss width");
  if constexpr (N == 128) wgmma_m64n128<0, 0>(s, da, db, scale_d);
  else if constexpr (N == 64) wgmma_m64n64<0, 0>(s, da, db, scale_d);
  else wgmma_m64n32<0, 0>(s, da, db, scale_d);
}

// O += A B over 16 contraction rows, N = D output columns: A (P or dS) from registers, B ([rows x D] tile: V, K, Q or
// dO) consumed MN-major straight from its TMA tile
template <int D>
__device__ __forceinline__ void wgmma_rs_d(float* o, const uint32_t (&a)[4], uint64_t db) {
  if constexpr (D == 40) wgmma_m64n40_rs_bmn(o, a, db);
  else if constexpr (D == 64) wgmma_m64n64_rs_bmn(o, a, db);
  else if constexpr (D == 80) wgmma_m64n80_rs_bmn(o, a, db);
  else wgmma_m64n160_rs_bmn(o, a, db);
}

// K-major descriptor of k-step k (16 columns) of a SWIZZLE_128B tile whose 64-column atoms are `atom_bytes` apart:
// columns 16 (k % 4) .. of atom k / 4, i.e. +32 B per step inside an atom
__device__ __forceinline__ uint64_t kstep_desc(uint64_t base, int k, int atom_bytes) {
  return base + (k / 4) * (atom_bytes >> 4) + 2 * (k % 4);
}

// 4-d tensor map {D, heads, L, B} over the head slices of a row-strided [B, L, >= heads * D] fp16 buffer (element
// (b, l, h, d) at base + b * bs + l * ls + h * D + d): one head is the innermost dimension, so a 64-column box past D
// reads zeros, never the next head, and rows past L read zeros.  Boxes are 64 columns x `box_rows` rows of one head.
inline int encode_head_tmap(CUtensorMap* tm, const void* base, int D, int heads, int L, int B, long long ls,
                            long long bs, int box_rows) {
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)heads, (uint64_t)L, (uint64_t)B};
  const uint64_t str[3] = {(uint64_t)D * 2, (uint64_t)ls * 2, (uint64_t)bs * 2};
  const uint32_t box[4] = {64, 1, (uint32_t)box_rows, 1};
  return encode_tmap(tm, base, 4, dims, str, box, nullptr);
}

}  // namespace b200
