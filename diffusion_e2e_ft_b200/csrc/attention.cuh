// Pieces shared by the flash attention forward (attention.cu) and backward (attention_bwd.cu, attention_d512_bwd.cu):
// the tensor maps, the exp2 / fp16-pair helpers, the backward's P / dS rounding and the wgmma shapes the kernels use.
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

__device__ __forceinline__ void named_barrier_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// one thread's 64 x 16 A fragment (k-chunk kk) of P and of dS from the accumulator-layout S and dP tiles: element e of
// column group i sits in row r0 + 8 (e / 2), column 8 i + 2 (lane % 4) + e % 2; lse / nd are per element (the dQ
// kernel passes its two rows' values, the dK/dV kernel its two columns').  P = fp16(exp2(fmaf(S, c, -lse))) and
// dS = fp16(fmaf(dP, s, nd) P) with nd = -s delta: the rounding of the GEMM composition (backward._attention_bwd_gemm)
__device__ __forceinline__ void p_ds_pair(float s0, float s1, float dp0, float dp1, float l0, float l1, float n0,
                                          float n1, float c, float sc, bool keep0, bool keep1, uint32_t& pa,
                                          uint32_t& dsa) {
  const float p0 = keep0 ? ex2_approx(fmaf(s0, c, -l0)) : 0.f;
  const float p1 = keep1 ? ex2_approx(fmaf(s1, c, -l1)) : 0.f;
  const __half2 ph = __floats2half2_rn(p0, p1);              // low = p0
  const float2 pf = __half22float2(ph);
  const __half2 dh = __floats2half2_rn(fmaf(dp0, sc, n0) * pf.x, fmaf(dp1, sc, n1) * pf.y);
  pa = *reinterpret_cast<const uint32_t*>(&ph);
  dsa = *reinterpret_cast<const uint32_t*>(&dh);
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

// 3-d tensor map {512, L, B} over a row-strided [B, L, >= 512] fp16 buffer (the single d = 512 head of the VAE
// mid-block, e.g. a column block of the fused [B, L, 1536] QKV projection): 64-column boxes of `box_rows` rows, rows
// past L read as zeros
inline int encode_d512_tmap(CUtensorMap* tm, const void* base, int L, int B, long long ls, long long bs, int box_rows) {
  const uint64_t dims[3] = {512, (uint64_t)L, (uint64_t)B};
  const uint64_t str[2] = {(uint64_t)ls * 2, (uint64_t)bs * 2};
  const uint32_t box[3] = {64, (uint32_t)box_rows, 1};
  return encode_tmap(tm, base, 3, dims, str, box, nullptr);
}

}  // namespace b200
