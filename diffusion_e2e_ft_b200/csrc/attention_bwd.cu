// Flash attention backward on sm_90a for heads of width D in {40, 64, 80, 160}: dQ, dK and dV of
// O = softmax(scale Q K^T) V from Q, K, V, dO, the forward's log2-domain log-sum-exp and delta = rowsum(dO o O),
// without storing P or dS.  Two kernels, no atomics, so the gradients are bitwise reproducible:
//
// attention_bwd_dq_kernel<D>    one warpgroup owns 64 query rows (Q and dO resident in smem, lse / delta in registers)
//                               and walks the K / V tiles through a TMA ring, like attention_kernel<D>.  Per key tile:
//     S  = Q K^T, dP = dO V^T   wgmma, both operands K-major from smem                -> 2 x BK/2 fp32 registers
//     P  = fp16(exp2(fmaf(S, c, -lse)));  dS = fp16(fmaf(dP, s, -s delta) * P)        in registers
//     dQ += dS K                A = dS from registers, K consumed MN-major from its [keys x D] tile
// attention_bwd_dkdv_kernel<D>  one warpgroup owns 64 key rows (K and V resident) and walks the query tiles (Q, dO,
//                               lse and -s delta) through a TMA ring.  Per query tile:
//     S^T = K Q^T, dP^T = V dO^T   so that P^T and dS^T land in the A-operand register layout
//     dV += P^T dO, dK += dS^T Q   B = dO / Q consumed MN-major from their [queries x D] tiles
// The kernels round exactly as the per-image GEMM composition (backward._attention_bwd_gemm) does: c = fp32(scale
// log2 e), P rounded to fp16 before it multiplies pre = fmaf(dP, s, fp32(-s delta)), dS rounded to fp16, fp32
// accumulators, fp16 outputs; only the order of the fp32 sums differs.
//
// Operands are read in place through the {D, heads, L, B} tensor maps of the forward (attention.cuh): 64-column
// SWIZZLE_128B boxes, columns past D and rows past L zero-filled.  Keys past Lk get P = 0 (explicitly: their S is 0,
// not -inf); query rows past Lq see lse = +inf and -s delta = 0, so their P, dP and dS are exactly 0.  Neither is
// ever stored.  Joint attention (kv_segments = 2): query image b walks the keys of b % (B/2) and b % (B/2) + B/2, so a
// key tile of image e takes the queries of both images of its pair.
//
// One consumer warpgroup and one producer warp per CTA (160 threads), so that two CTAs share an SM where registers
// and shared memory allow; tile shapes per D (registers and shared memory from -Xptxas -v in DESIGN §3):
//   dQ:    BK = 64 keys, dQ D/2 + S 32 + dP 32 fp32 registers; 3 stages at D <= 64, 2 at D = 80, 160
//   dK/dV: BQ = 64 queries at D <= 64, 32 at D = 80, 160 (dK + dV are D fp32 registers: 160 at D = 160)
#include "attention.cuh"
#include "../../include/b200_e2eft.h"
#include "../../include/b200_e2eft_attention_bwd.h"

namespace b200 {

constexpr int kBwdRows = 64;                       // query rows (dQ) / key rows (dK/dV) of the CTA's warpgroup
constexpr int kBwdThreads = 128 + 32;              // consumer warpgroup + TMA producer warp

template <int D> struct DqCfg;
template <> struct DqCfg<40> { static constexpr int kBk = 64, kStages = 3, kMinBlocks = 2; };
template <> struct DqCfg<64> { static constexpr int kBk = 64, kStages = 3, kMinBlocks = 2; };
template <> struct DqCfg<80> { static constexpr int kBk = 64, kStages = 2, kMinBlocks = 2; };
template <> struct DqCfg<160> { static constexpr int kBk = 64, kStages = 2, kMinBlocks = 1; };

template <int D> struct DkvCfg;
template <> struct DkvCfg<40> { static constexpr int kBq = 64, kStages = 3, kMinBlocks = 2; };
template <> struct DkvCfg<64> { static constexpr int kBq = 64, kStages = 3, kMinBlocks = 2; };
template <> struct DkvCfg<80> { static constexpr int kBq = 32, kStages = 3, kMinBlocks = 2; };
template <> struct DkvCfg<160> { static constexpr int kBq = 32, kStages = 3, kMinBlocks = 1; };

template <int D>
struct BwdShape {
  static constexpr int kAtoms = (D + 63) / 64;               // 64-column SWIZZLE_128B atoms per row
  static constexpr int kKSteps = (D + 15) / 16;              // k16 steps of a product over D
  static constexpr int kRowAtom = kBwdRows * 128;            // one 64-row atom of a resident tile
  static constexpr int kRowBytes = kAtoms * kRowAtom;        // one resident [64 x D] tile
  // dQ kernel: Q + dO resident, stages x (K + V)
  static constexpr int kBk = DqCfg<D>::kBk;
  static constexpr int kKvAtom = kBk * 128;
  static constexpr int kKvBytes = kAtoms * kKvAtom;
  static constexpr int kDqSmem = 2 * kRowBytes + DqCfg<D>::kStages * 2 * kKvBytes + 256 + 1024;
  // dK/dV kernel: K + V resident, stages x (Q + dO + lse + -s delta)
  static constexpr int kBq = DkvCfg<D>::kBq;
  static constexpr int kQAtom = kBq * 128;
  static constexpr int kQBytes = kAtoms * kQAtom;
  static constexpr int kDkvSmem = 2 * kRowBytes + DkvCfg<D>::kStages * (2 * kQBytes + 2 * kBq * 4) + 256 + 1024;
  static_assert(kDqSmem <= 227 * 1024 && kDkvSmem <= 227 * 1024, "attention backward shared memory");
};

struct AttBwdParams {
  int B, heads, Lq, Lk, kv_segments;
  float scale_log2, scale;
  const float* lse;            // [B][heads][Lq], log2 domain (the forward's)
  const float* delta;          // [B][heads][Lq], rowsum(dO o O)
  __half *dq, *dk, *dv;
  long long dq_bs, dq_ls, dk_bs, dk_ls, dv_bs, dv_ls;
};

// ===================================================================================================== dQ
template <int D>
__global__ void __launch_bounds__(kBwdThreads, DqCfg<D>::kMinBlocks)
attention_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmO,
                        const AttBwdParams p) {
  using S_ = BwdShape<D>;
  constexpr int kBk = S_::kBk, kStages = DqCfg<D>::kStages, kAtoms = S_::kAtoms;
  constexpr int kRowBytes = S_::kRowBytes, kKvBytes = S_::kKvBytes;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                                   // [kAtoms][64 rows x 128 B]
  uint8_t* sO = sQ + kRowBytes;                         // dO, same layout
  uint8_t* sK = sO + kRowBytes;                         // [stages][kAtoms][kBk rows x 128 B]
  uint8_t* sV = sK + kStages * kKvBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kStages * kKvBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = kv_full + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kBwdRows;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int tiles_per_seg = (p.Lk + kBk - 1) / kBk;
  const int n_tiles = tiles_per_seg * p.kv_segments;
  const int half_b = p.kv_segments == 2 ? p.B / 2 : 0;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmO);
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 128);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ===================================================================== TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, 2 * kRowBytes);
      for (int a = 0; a < kAtoms; ++a) {
        tma_load_4d(&tmQ, q_full, sQ + a * S_::kRowAtom, 64 * a, h, q0, b, kEvictFirst);
        tma_load_4d(&tmO, q_full, sO + a * S_::kRowAtom, 64 * a, h, q0, b, kEvictFirst);
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int seg = 0; seg < p.kv_segments; ++seg) {
        const int kb = p.kv_segments == 2 ? (b % half_b) + seg * half_b : b;
        for (int j = 0; j < tiles_per_seg; ++j) {
          mbar_wait(&kv_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&kv_full[stage], 2 * kKvBytes);
          for (int a = 0; a < kAtoms; ++a) {
            tma_load_4d(&tmK, &kv_full[stage], sK + stage * kKvBytes + a * S_::kKvAtom, 64 * a, h, j * kBk, kb,
                        kEvictLast);
            tma_load_4d(&tmV, &kv_full[stage], sV + stage * kKvBytes + a * S_::kKvAtom, 64 * a, h, j * kBk, kb,
                        kEvictLast);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  // ========================================================================= consumer warpgroup
  const int r0 = (warp & 3) * 16 + (lane >> 2);         // accumulator rows r0, r0 + 8 (wgmma.cuh)
  const int cq = 2 * (lane & 3);
  const float c = p.scale_log2, sc = p.scale;
  float lse[2], nd[2];                                   // rows past Lq: P = exp2(-inf) = 0, -s delta = 0
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t = q0 + r0 + 8 * r;
    const long long idx = ((long long)b * p.heads + h) * p.Lq + t;
    lse[r] = t < p.Lq ? p.lse[idx] : INFINITY;
    nd[r] = t < p.Lq ? -sc * p.delta[idx] : 0.f;
  }
  float dq[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dq[i] = 0.f;
  const uint64_t qdesc = make_desc_sw128(smem_u32(sQ), 16, 1024);
  const uint64_t odesc = make_desc_sw128(smem_u32(sO), 16, 1024);
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    const int valid = min(kBk, p.Lk - (j % tiles_per_seg) * kBk);
    float s[kBk / 2], dp[kBk / 2];
    mbar_wait(&kv_full[st], ph);
    const uint32_t kbase = smem_u32(sK + st * kKvBytes);
    {
      const uint64_t kdesc = make_desc_sw128(kbase, 16, 1024);
      const uint64_t vdesc = make_desc_sw128(smem_u32(sV + st * kKvBytes), 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < S_::kKSteps; ++k)
        wgmma_ss<kBk>(s, kstep_desc(qdesc, k, S_::kRowAtom), kstep_desc(kdesc, k, S_::kKvAtom), k != 0);
#pragma unroll
      for (int k = 0; k < S_::kKSteps; ++k)
        wgmma_ss<kBk>(dp, kstep_desc(odesc, k, S_::kRowAtom), kstep_desc(vdesc, k, S_::kKvAtom), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands<kBk / 2>(s);
      wgmma_fence_operands<kBk / 2>(dp);
    }
    uint32_t pa[kBk / 16][4], dsa[kBk / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBk / 16; ++kk) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int i = 2 * kk + hf;
        const int col = 8 * i + cq;                      // keys >= valid do not exist: P = 0
        const bool k0 = col < valid, k1 = col + 1 < valid;
        p_ds_pair(s[4 * i], s[4 * i + 1], dp[4 * i], dp[4 * i + 1], lse[0], lse[0], nd[0], nd[0], c, sc, k0, k1,
                  pa[kk][2 * hf], dsa[kk][2 * hf]);
        p_ds_pair(s[4 * i + 2], s[4 * i + 3], dp[4 * i + 2], dp[4 * i + 3], lse[1], lse[1], nd[1], nd[1], c, sc,
                  k0, k1, pa[kk][2 * hf + 1], dsa[kk][2 * hf + 1]);
      }
    }
    wgmma_fence_operands<D / 2>(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBk / 16; ++kk)         // B = K[16 kk .. 16 kk + 15, :]: MN-major, atoms kKvAtom apart
      wgmma_rs_d<D>(dq, dsa[kk], make_desc_sw128(kbase + kk * 2048, S_::kKvAtom, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands<D / 2>(dq);
    mbar_arrive(&kv_empty[st]);                      // done with K_j / V_j
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t = q0 + r0 + 8 * r;
    if (t >= p.Lq) continue;
    __half* dst = p.dq + (long long)b * p.dq_bs + (long long)t * p.dq_ls + h * D + cq;
#pragma unroll
    for (int i = 0; i < D / 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_half2(dq[4 * i + 2 * r], dq[4 * i + 2 * r + 1]);
  }
}

// ================================================================================================== dK / dV
template <int D>
__global__ void __launch_bounds__(kBwdThreads, DkvCfg<D>::kMinBlocks)
attention_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                          const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmO,
                          const AttBwdParams p) {
  using S_ = BwdShape<D>;
  constexpr int kBq = S_::kBq, kStages = DkvCfg<D>::kStages, kAtoms = S_::kAtoms;
  constexpr int kRowBytes = S_::kRowBytes, kQBytes = S_::kQBytes;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sK = smem;                                   // [kAtoms][64 rows x 128 B]
  uint8_t* sV = sK + kRowBytes;
  uint8_t* sQ = sV + kRowBytes;                         // [stages][kAtoms][kBq rows x 128 B]
  uint8_t* sO = sQ + kStages * kQBytes;                 // dO, same layout
  float* sL = reinterpret_cast<float*>(sO + kStages * kQBytes);   // [stages][kBq] lse, +inf past Lq
  float* sN = sL + kStages * kBq;                                  // [stages][kBq] -s delta, 0 past Lq
  uint64_t* bars = reinterpret_cast<uint64_t*>(sN + kStages * kBq);
  uint64_t* kv_full = bars;
  uint64_t* q_full = bars + 1;
  uint64_t* q_empty = q_full + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * kBwdRows;
  const int h = blockIdx.y;
  const int e = blockIdx.z;                              // the key image
  const int tiles_per_seg = (p.Lq + kBq - 1) / kBq;
  const int n_tiles = tiles_per_seg * p.kv_segments;
  const int half_b = p.kv_segments == 2 ? p.B / 2 : 0;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmO);
    mbar_init(kv_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&q_full[i], 32);                         // every producer lane, after its lse / delta stores
      mbar_init(&q_empty[i], 128);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ===================================================================== producer warp
    if (lane == 0) {
      mbar_arrive_expect_tx(kv_full, 2 * kRowBytes);
      for (int a = 0; a < kAtoms; ++a) {
        tma_load_4d(&tmK, kv_full, sK + a * S_::kRowAtom, 64 * a, h, k0, e, kEvictFirst);
        tma_load_4d(&tmV, kv_full, sV + a * S_::kRowAtom, 64 * a, h, k0, e, kEvictFirst);
      }
    }
    const float sc = p.scale;
    int stage = 0;
    uint32_t phase = 0;
    for (int seg = 0; seg < p.kv_segments; ++seg) {
      const int qb = p.kv_segments == 2 ? (e % half_b) + seg * half_b : e;
      const long long row0 = ((long long)qb * p.heads + h) * p.Lq;
      for (int j = 0; j < tiles_per_seg; ++j) {
        mbar_wait(&q_empty[stage], phase ^ 1);
        for (int i = lane; i < kBq; i += 32) {
          const int t = j * kBq + i;
          sL[stage * kBq + i] = t < p.Lq ? p.lse[row0 + t] : INFINITY;
          sN[stage * kBq + i] = t < p.Lq ? -sc * p.delta[row0 + t] : 0.f;
        }
        if (lane == 0) {
          mbar_arrive_expect_tx(&q_full[stage], 2 * kQBytes);
          for (int a = 0; a < kAtoms; ++a) {
            tma_load_4d(&tmQ, &q_full[stage], sQ + stage * kQBytes + a * S_::kQAtom, 64 * a, h, j * kBq, qb,
                        kEvictLast);
            tma_load_4d(&tmO, &q_full[stage], sO + stage * kQBytes + a * S_::kQAtom, 64 * a, h, j * kBq, qb,
                        kEvictLast);
          }
        } else {
          mbar_arrive(&q_full[stage]);
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  // ========================================================================= consumer warpgroup
  const int r0 = (warp & 3) * 16 + (lane >> 2);         // key rows r0, r0 + 8
  const int cq = 2 * (lane & 3);                         // query columns 8 i + cq, + 1
  const float c = p.scale_log2, sc = p.scale;
  float dk[D / 2], dv[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
  const uint64_t kdesc = make_desc_sw128(smem_u32(sK), 16, 1024);
  const uint64_t vdesc = make_desc_sw128(smem_u32(sV), 16, 1024);
  mbar_wait(kv_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    float s[kBq / 2], dp[kBq / 2];
    mbar_wait(&q_full[st], ph);
    const uint32_t qbase = smem_u32(sQ + st * kQBytes);
    const uint32_t obase = smem_u32(sO + st * kQBytes);
    {
      const uint64_t qdesc = make_desc_sw128(qbase, 16, 1024);
      const uint64_t odesc = make_desc_sw128(obase, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < S_::kKSteps; ++k)
        wgmma_ss<kBq>(s, kstep_desc(kdesc, k, S_::kRowAtom), kstep_desc(qdesc, k, S_::kQAtom), k != 0);
#pragma unroll
      for (int k = 0; k < S_::kKSteps; ++k)
        wgmma_ss<kBq>(dp, kstep_desc(vdesc, k, S_::kRowAtom), kstep_desc(odesc, k, S_::kQAtom), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands<kBq / 2>(s);
      wgmma_fence_operands<kBq / 2>(dp);
    }
    const float* lt = sL + st * kBq;
    const float* nt = sN + st * kBq;
    uint32_t pa[kBq / 16][4], dsa[kBq / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBq / 16; ++kk) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int i = 2 * kk + hf;
        const float2 l2 = *reinterpret_cast<const float2*>(lt + 8 * i + cq);
        const float2 n2 = *reinterpret_cast<const float2*>(nt + 8 * i + cq);
        p_ds_pair(s[4 * i], s[4 * i + 1], dp[4 * i], dp[4 * i + 1], l2.x, l2.y, n2.x, n2.y, c, sc, true, true,
                  pa[kk][2 * hf], dsa[kk][2 * hf]);
        p_ds_pair(s[4 * i + 2], s[4 * i + 3], dp[4 * i + 2], dp[4 * i + 3], l2.x, l2.y, n2.x, n2.y, c, sc, true,
                  true, pa[kk][2 * hf + 1], dsa[kk][2 * hf + 1]);
      }
    }
    wgmma_fence_operands<D / 2>(dv);
    wgmma_fence_operands<D / 2>(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBq / 16; ++kk)         // B = dO / Q[16 kk .. 16 kk + 15, :]: MN-major, atoms kQAtom apart
      wgmma_rs_d<D>(dv, pa[kk], make_desc_sw128(obase + kk * 2048, S_::kQAtom, 1024));
#pragma unroll
    for (int kk = 0; kk < kBq / 16; ++kk)
      wgmma_rs_d<D>(dk, dsa[kk], make_desc_sw128(qbase + kk * 2048, S_::kQAtom, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands<D / 2>(dv);
    wgmma_fence_operands<D / 2>(dk);
    mbar_arrive(&q_empty[st]);                       // done with this query tile
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t = k0 + r0 + 8 * r;
    if (t >= p.Lk) continue;
    __half* dstk = p.dk + (long long)e * p.dk_bs + (long long)t * p.dk_ls + h * D + cq;
    __half* dstv = p.dv + (long long)e * p.dv_bs + (long long)t * p.dv_ls + h * D + cq;
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      *reinterpret_cast<uint32_t*>(dstk + 8 * i) = pack_half2(dk[4 * i + 2 * r], dk[4 * i + 2 * r + 1]);
      *reinterpret_cast<uint32_t*>(dstv + 8 * i) = pack_half2(dv[4 * i + 2 * r], dv[4 * i + 2 * r + 1]);
    }
  }
}

}  // namespace b200

using namespace b200;

namespace {

template <typename K>
int configure_smem(K kernel, int smem, const char* what, bool& configured) {
  if (configured && current_device() >= 0) return 0;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) {
    set_last_error("cudaFuncSetAttribute(%s smem=%d): %s", what, smem, cudaGetErrorString(e));
    return (int)e;
  }
  configured = true;
  return 0;
}

template <int D>
int launch_attention_bwd(const void* q, long long q_bs, long long q_ls, const void* k, long long k_bs, long long k_ls,
                         const void* v, long long v_bs, long long v_ls, const void* dout, long long do_bs,
                         long long do_ls, const AttBwdParams& p, void* stream) {
  using S_ = BwdShape<D>;
  // dQ kernel: Q / dO in 64-row boxes, K / V in BK-row boxes; dK/dV kernel: K / V in 64-row boxes, Q / dO in BQ rows
  CUtensorMap dq_q, dq_k, dq_v, dq_o, kv_q, kv_k, kv_v, kv_o;
  int r = encode_head_tmap(&dq_q, q, D, p.heads, p.Lq, p.B, q_ls, q_bs, kBwdRows);
  if (!r) r = encode_head_tmap(&dq_o, dout, D, p.heads, p.Lq, p.B, do_ls, do_bs, kBwdRows);
  if (!r) r = encode_head_tmap(&dq_k, k, D, p.heads, p.Lk, p.B, k_ls, k_bs, S_::kBk);
  if (!r) r = encode_head_tmap(&dq_v, v, D, p.heads, p.Lk, p.B, v_ls, v_bs, S_::kBk);
  if (!r) r = encode_head_tmap(&kv_q, q, D, p.heads, p.Lq, p.B, q_ls, q_bs, S_::kBq);
  if (!r) r = encode_head_tmap(&kv_o, dout, D, p.heads, p.Lq, p.B, do_ls, do_bs, S_::kBq);
  if (!r) r = encode_head_tmap(&kv_k, k, D, p.heads, p.Lk, p.B, k_ls, k_bs, kBwdRows);
  if (!r) r = encode_head_tmap(&kv_v, v, D, p.heads, p.Lk, p.B, v_ls, v_bs, kBwdRows);
  if (r) return r;
  static bool dq_configured[kMaxDevices] = {false}, kv_configured[kMaxDevices] = {false};   // per device
  const int dev = current_device();
  const int slot = dev < 0 ? 0 : dev;
  r = configure_smem(attention_bwd_dq_kernel<D>, S_::kDqSmem, "attention_bwd_dq_kernel", dq_configured[slot]);
  if (!r) r = configure_smem(attention_bwd_dkdv_kernel<D>, S_::kDkvSmem, "attention_bwd_dkdv_kernel",
                             kv_configured[slot]);
  if (r) return r;
  const dim3 gq((p.Lq + kBwdRows - 1) / kBwdRows, p.heads, p.B);
  attention_bwd_dq_kernel<D><<<gq, kBwdThreads, S_::kDqSmem, (cudaStream_t)stream>>>(dq_q, dq_k, dq_v, dq_o, p);
  B200_CHECK_LAUNCH("attention_bwd_dq_kernel");
  const dim3 gk((p.Lk + kBwdRows - 1) / kBwdRows, p.heads, p.B);
  attention_bwd_dkdv_kernel<D><<<gk, kBwdThreads, S_::kDkvSmem, (cudaStream_t)stream>>>(kv_q, kv_k, kv_v, kv_o, p);
  B200_CHECK_LAUNCH("attention_bwd_dkdv_kernel");
  return 0;
}

}  // namespace

extern "C" int b200_attention_bwd(const void* q, long long q_bs, long long q_ls, const void* k, long long k_bs,
                                  long long k_ls, const void* v, long long v_bs, long long v_ls, const void* dout,
                                  long long do_bs, long long do_ls, const float* lse, const float* delta, void* dq,
                                  long long dq_bs, long long dq_ls, void* dk, long long dk_bs, long long dk_ls,
                                  void* dv, long long dv_bs, long long dv_ls, int B, int heads, int head_dim, int Lq,
                                  int Lk, int kv_segments, float scale, void* stream) {
  B200_CHECK_ARG(head_dim == 40 || head_dim == 64 || head_dim == 80 || head_dim == 160,
                 "b200_attention_bwd: head_dim=%d is not one of 40, 64, 80, 160", head_dim);
  B200_CHECK_ARG(q && k && v && dout && lse && delta && dq && dk && dv, "b200_attention_bwd: null pointer");
  B200_CHECK_ARG(B > 0 && B <= 65535 && heads > 0 && heads <= 65535 && Lq > 0 && Lk > 0,
                 "b200_attention_bwd: bad shape B=%d heads=%d Lq=%d Lk=%d", B, heads, Lq, Lk);
  B200_CHECK_ARG(kv_segments == 1 || (kv_segments == 2 && B % 2 == 0), "b200_attention_bwd: kv_segments=%d B=%d",
                 kv_segments, B);
  B200_CHECK_ARG(q_ls % 8 == 0 && k_ls % 8 == 0 && v_ls % 8 == 0 && do_ls % 8 == 0 && dq_ls % 8 == 0 &&
                     dk_ls % 8 == 0 && dv_ls % 8 == 0 && q_bs % 8 == 0 && k_bs % 8 == 0 && v_bs % 8 == 0 &&
                     do_bs % 8 == 0 && dq_bs % 8 == 0 && dk_bs % 8 == 0 && dv_bs % 8 == 0,
                 "b200_attention_bwd: strides must be multiples of 8 elements");
  B200_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)dout | (uintptr_t)dq | (uintptr_t)dk |
                   (uintptr_t)dv) & 15) == 0,
                 "b200_attention_bwd: pointers must be 16-byte aligned");
  B200_CHECK_ARG((((uintptr_t)lse | (uintptr_t)delta) & 3) == 0, "b200_attention_bwd: lse / delta must be 4-byte aligned");
  AttBwdParams p;
  p.B = B; p.heads = heads; p.Lq = Lq; p.Lk = Lk; p.kv_segments = kv_segments;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.scale = scale;
  p.lse = lse; p.delta = delta;
  p.dq = (__half*)dq; p.dk = (__half*)dk; p.dv = (__half*)dv;
  p.dq_bs = dq_bs; p.dq_ls = dq_ls; p.dk_bs = dk_bs; p.dk_ls = dk_ls; p.dv_bs = dv_bs; p.dv_ls = dv_ls;
  switch (head_dim) {
    case 40: return launch_attention_bwd<40>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, dout, do_bs, do_ls, p, stream);
    case 64: return launch_attention_bwd<64>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, dout, do_bs, do_ls, p, stream);
    case 80: return launch_attention_bwd<80>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, dout, do_bs, do_ls, p, stream);
    default: return launch_attention_bwd<160>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, dout, do_bs, do_ls, p, stream);
  }
}
