// Flash attention backward on sm_90a for the single head of width 512 (VAE mid-block): dQ, dK and dV of
// O = softmax(scale Q K^T) V from Q, K, V, dO, the forward's log2-domain log-sum-exp and delta = rowsum(dO o O),
// without storing P or dS.  The rounding is that of the width-40 .. 160 kernels (attention_bwd.cu, p_ds_pair):
// P = fp16(exp2(fmaf(S, c, -lse))), dS = fp16(fmaf(dP, s, -s delta) P), fp32 accumulators, fp16 outputs.
//
// A 64 x 512 fp32 accumulator is 128 registers per thread over two warpgroups (as the forward holds O), so one CTA
// holds one gradient.  One kernel, templated on the gradient G it produces, with a resident 64-row block (A0, A1) and
// a streamed block of BN rows (B0, B1) per tile:
//   G = dQ   A = (Q, dO) query rows, B = (K, V) key tiles      S  = Q K^T,  dP  = dO V^T,  dQ += dS K
//   G = dK   A = (K, V)  key rows,   B = (Q, dO) query tiles   S^T = K Q^T, dP^T = V dO^T, dK += dS^T Q
//   G = dV   A = K       key rows,   B = (Q, dO) query tiles   S^T = K Q^T,                dV += P^T dO
// so the A operand of the accumulating MMA (P^T / dS^T in the key-stationary kernels) is already in the accumulator
// register layout.  8 products of 2 L^2 512 where 5 are needed: S three times, dP twice.
//
// As in the forward, warpgroup w owns the d-columns 256 w .. 256 w + 255: its half of every reduction over d and its
// 256 output columns.  Per tile j:
//   S_w (, dP_w)        wgmma m64n<BN>k16 x 16 from smem (K-major), the warpgroup's 256 columns
//   S = S_0 + S_1       each warpgroup stores its partial tiles to smem, one named barrier, each adds the other's: both
//                       hold the same S (and dP) and compute the same P and dS redundantly
//   acc_w += X Y_j[:, w]   wgmma m64n256k16 x BN/16, X = dS or P from registers, Y_j = B0 or B1 consumed MN-major
// Keys past Lk get P = 0 (dQ: explicitly); query rows / columns past Lq see lse = +inf and -s delta = 0, so their
// P and dS are exactly 0.  Rows of the resident block past its length are never stored.  No atomics.
//
// Shared memory (BN = 16 for dQ / dK, 32 for dV): A 128 KB (dV: 64 KB) + 2 buffers x (B0 + B1) of BN x 1 KB +
// 2 parities x 2 warpgroups x the partial tiles (S and dP: 2 x 4 KB; dV: S 8 KB) = 224 KB + barriers + 1 KB slack.
// Thread 0 issues the loads.  At the named barrier of tile j both warpgroups are done with tile j - 1, so tile j + 1
// goes into its buffer; the partial tiles are double buffered by tile parity (a warpgroup rewrites parity j after
// barrier j + 1, which its partner passes after reading them).
#include "attention.cuh"
#include "../../include/b200_e2eft.h"
#include "../../include/b200_e2eft_vae_attention.h"

namespace b200 {

enum D5Grad { kGradQ = 0, kGradK = 1, kGradV = 2 };

template <int G>
struct D5BwdShape {
  static constexpr bool kDP = G != kGradV;                 // needs dP, and a second resident block
  static constexpr int kBn = G == kGradV ? 32 : 16;        // streamed rows per tile
  static constexpr int kRes = kDP ? 2 : 1;
  static constexpr int kThreads = 256;
  static constexpr int kRows = 64;                         // resident rows per CTA
  static constexpr int kABox = kRows * 128;                // one 64-row x 64-column box, 8 KB
  static constexpr int kABytes = 8 * kABox;                // 64 rows x 512 columns
  static constexpr int kBBox = kBn * 128;
  static constexpr int kBBytes = 8 * kBBox;
  static constexpr int kXFloats = kRows * kBn;             // one partial tile
  static constexpr int kSmem = kRes * kABytes + 2 * 2 * kBBytes + 2 * 2 * kRes * kXFloats * 4 + 64 + 1024;
  static_assert(kSmem <= 227 * 1024, "attention_d512_bwd shared memory");
};

struct AttD512BwdParams {
  int Lq, Lk;
  float scale_log2, scale;
  const float* lse;            // [B][Lq]
  const float* delta;          // [B][Lq]
  __half* out;                 // dq, dk or dv
  long long o_bs, o_ls;
};

// S (+)= A B^T for 16 keys / queries: m64n16k16, both operands K-major from smem
__device__ __forceinline__ void wgmma_m64n16_ss(float* d, uint64_t da, uint64_t db, int scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(da), "l"(db), "r"(scale_d));
}

template <int N>
__device__ __forceinline__ void d512_wgmma_ss(float* s, uint64_t da, uint64_t db, int scale_d) {
  if constexpr (N == 16) wgmma_m64n16_ss(s, da, db, scale_d);
  else wgmma_m64n32<0, 0>(s, da, db, scale_d);
}

// partial tile X_w = A[:, 256 w ..] B_j[:, 256 w ..]^T over the warpgroup's 4 boxes x 4 k16 steps
template <int BN>
__device__ __forceinline__ void d512_partial(float* x, const uint8_t* a, const uint8_t* bt, int w) {
#pragma unroll
  for (int cc = 0; cc < 4; ++cc) {
    const int box = 4 * w + cc;
    const uint64_t adesc = make_desc_sw128(smem_u32(a + box * (64 * 128)), 16, 1024);
    const uint64_t bdesc = make_desc_sw128(smem_u32(bt + box * (BN * 128)), 16, 1024);
#pragma unroll
    for (int k = 0; k < 4; ++k) d512_wgmma_ss<BN>(x, adesc + 2 * k, bdesc + 2 * k, (cc | k) != 0);
  }
}

template <int G>
__global__ void __launch_bounds__(D5BwdShape<G>::kThreads, 1)
attention_d512_bwd_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                          const __grid_constant__ CUtensorMap tmB0, const __grid_constant__ CUtensorMap tmB1,
                          const AttD512BwdParams p) {
  using S_ = D5BwdShape<G>;
  constexpr int kBn = S_::kBn, kRes = S_::kRes, kXFloats = S_::kXFloats;
  constexpr int kABox = S_::kABox, kABytes = S_::kABytes, kBBox = S_::kBBox, kBBytes = S_::kBBytes;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;                                   // [kRes][8 boxes][64 rows x 128 B]
  uint8_t* sB0 = sA + kRes * kABytes;                   // [2 buffers][8 boxes][kBn rows x 128 B]
  uint8_t* sB1 = sB0 + 2 * kBBytes;
  float* sX = reinterpret_cast<float*>(sB1 + 2 * kBBytes);   // [2 parities][2 warpgroups][kRes][partial tile]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sX + 2 * 2 * kRes * kXFloats);
  uint64_t* a_full = bars;
  uint64_t* b_full = bars + 1;                          // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * S_::kRows;
  const int b = blockIdx.y;
  const int n_rows = G == kGradQ ? p.Lq : p.Lk;         // resident rows
  const int n_cols = G == kGradQ ? p.Lk : p.Lq;         // streamed rows
  const int n_tiles = (n_cols + kBn - 1) / kBn;
  const bool loader = threadIdx.x == 0;
  auto load_b = [&](int j, int buf) {
    mbar_arrive_expect_tx(&b_full[buf], 2 * kBBytes);
    for (int c = 0; c < 8; ++c) {
      tma_load_3d(&tmB0, &b_full[buf], sB0 + buf * kBBytes + c * kBBox, 64 * c, j * kBn, b, kEvictLast);
      tma_load_3d(&tmB1, &b_full[buf], sB1 + buf * kBBytes + c * kBBox, 64 * c, j * kBn, b, kEvictLast);
    }
  };

  if (loader) {
    tma_prefetch_desc(&tmA0);
    if constexpr (S_::kDP) tma_prefetch_desc(&tmA1);
    tma_prefetch_desc(&tmB0);
    tma_prefetch_desc(&tmB1);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(a_full, kRes * kABytes);
    for (int c = 0; c < 8; ++c) {
      tma_load_3d(&tmA0, a_full, sA + c * kABox, 64 * c, row0, b, kEvictFirst);
      if constexpr (S_::kDP) tma_load_3d(&tmA1, a_full, sA + kABytes + c * kABox, 64 * c, row0, b, kEvictFirst);
    }
    load_b(0, 0);
    if (n_tiles > 1) load_b(1, 1);
  }
  __syncthreads();

  const int w = warp >> 2;
  const int t = threadIdx.x & 127;
  const int r0 = (warp & 3) * 16 + (lane >> 2);         // accumulator rows r0, r0 + 8 (wgmma.cuh)
  const int cq = 2 * (lane & 3);                         // columns 8 i + cq, + 1
  const float c = p.scale_log2, sc = p.scale;
  const float* lse_b = p.lse + (long long)b * p.Lq;
  const float* delta_b = p.delta + (long long)b * p.Lq;
  float lse_r[2] = {0.f, 0.f}, nd_r[2] = {0.f, 0.f};    // dQ: per row, rows past Lq: P = 0, -s delta = 0
  if constexpr (G == kGradQ) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = row0 + r0 + 8 * r;
      lse_r[r] = q < p.Lq ? lse_b[q] : INFINITY;
      nd_r[r] = q < p.Lq ? -sc * delta_b[q] : 0.f;
    }
  }
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  mbar_wait(a_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int buf = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    // dK / dV: lse and -s delta of this tile's query columns (read ahead of the MMAs)
    float lc[kBn / 4], nc[kBn / 4];
    if constexpr (G != kGradQ) {
#pragma unroll
      for (int i = 0; i < kBn / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int q = j * kBn + 8 * i + cq + e;
          lc[2 * i + e] = q < p.Lq ? lse_b[q] : INFINITY;
          nc[2 * i + e] = q < p.Lq ? -sc * delta_b[q] : 0.f;
        }
    }
    float s[kBn / 2], dp[kBn / 2];
    mbar_wait(&b_full[buf], ph);
    wgmma_fence();
    d512_partial<kBn>(s, sA, sB0 + buf * kBBytes, w);
    if constexpr (S_::kDP) d512_partial<kBn>(dp, sA + kABytes, sB1 + buf * kBBytes, w);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands<kBn / 2>(s);
    if constexpr (S_::kDP) wgmma_fence_operands<kBn / 2>(dp);
    // S = S_0 + S_1 (dP likewise): thread t of one warpgroup holds the same fragment positions as thread t of the other
    float4* x_own = reinterpret_cast<float4*>(sX + (buf * 2 + w) * kRes * kXFloats);
    const float4* x_other = reinterpret_cast<const float4*>(sX + (buf * 2 + (w ^ 1)) * kRes * kXFloats);
#pragma unroll
    for (int i = 0; i < kBn / 8; ++i) {
      x_own[i * 128 + t] = make_float4(s[4 * i], s[4 * i + 1], s[4 * i + 2], s[4 * i + 3]);
      if constexpr (S_::kDP)
        x_own[(kBn / 8 + i) * 128 + t] = make_float4(dp[4 * i], dp[4 * i + 1], dp[4 * i + 2], dp[4 * i + 3]);
    }
    named_barrier_sync(1, S_::kThreads);
    if (loader && j >= 1 && j + 1 < n_tiles) load_b(j + 1, buf ^ 1);   // tile j - 1's buffer is free
#pragma unroll
    for (int i = 0; i < kBn / 8; ++i) {
      const float4 v = x_other[i * 128 + t];
      s[4 * i] += v.x;
      s[4 * i + 1] += v.y;
      s[4 * i + 2] += v.z;
      s[4 * i + 3] += v.w;
      if constexpr (S_::kDP) {
        const float4 u = x_other[(kBn / 8 + i) * 128 + t];
        dp[4 * i] += u.x;
        dp[4 * i + 1] += u.y;
        dp[4 * i + 2] += u.z;
        dp[4 * i + 3] += u.w;
      } else {
        dp[4 * i] = dp[4 * i + 1] = dp[4 * i + 2] = dp[4 * i + 3] = 0.f;     // dS unused
      }
    }
    uint32_t pa[kBn / 16][4], dsa[kBn / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBn / 16; ++kk) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int i = 2 * kk + hf;
        if constexpr (G == kGradQ) {
          const int key = j * kBn + 8 * i + cq;          // keys >= Lk do not exist: P = 0
          const bool k0 = key < p.Lk, k1 = key + 1 < p.Lk;
          p_ds_pair(s[4 * i], s[4 * i + 1], dp[4 * i], dp[4 * i + 1], lse_r[0], lse_r[0], nd_r[0], nd_r[0], c, sc,
                    k0, k1, pa[kk][2 * hf], dsa[kk][2 * hf]);
          p_ds_pair(s[4 * i + 2], s[4 * i + 3], dp[4 * i + 2], dp[4 * i + 3], lse_r[1], lse_r[1], nd_r[1], nd_r[1],
                    c, sc, k0, k1, pa[kk][2 * hf + 1], dsa[kk][2 * hf + 1]);
        } else {
          p_ds_pair(s[4 * i], s[4 * i + 1], dp[4 * i], dp[4 * i + 1], lc[2 * i], lc[2 * i + 1], nc[2 * i],
                    nc[2 * i + 1], c, sc, true, true, pa[kk][2 * hf], dsa[kk][2 * hf]);
          p_ds_pair(s[4 * i + 2], s[4 * i + 3], dp[4 * i + 2], dp[4 * i + 3], lc[2 * i], lc[2 * i + 1], nc[2 * i],
                    nc[2 * i + 1], c, sc, true, true, pa[kk][2 * hf + 1], dsa[kk][2 * hf + 1]);
        }
      }
    }
    {
      // B = Y_j[16 kk .. 16 kk + 15][256 w ..]: MN-major, the warpgroup's four 64-column boxes kBBox apart (LBO)
      const uint32_t ybase = smem_u32((G == kGradV ? sB1 : sB0) + buf * kBBytes + w * 4 * kBBox);
      wgmma_fence_operands<128>(acc);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBn / 16; ++kk)
        wgmma_m64n256_rs_bmn(acc, G == kGradV ? pa[kk] : dsa[kk], make_desc_sw128(ybase + kk * 2048, kBBox, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands<128>(acc);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + r0 + 8 * r;
    if (row >= n_rows) continue;
    __half* dst = p.out + (long long)b * p.o_bs + (long long)row * p.o_ls + w * 256 + cq;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_half2(acc[4 * i + 2 * r], acc[4 * i + 2 * r + 1]);
  }
}

// delta[b][l] = sum_d a[b][l][d] c[b][l][d] over 512 columns: one warp per row, 16 columns per lane
__global__ void __launch_bounds__(256)
rowdot_d512_kernel(const __half* a, long long a_bs, long long a_ls, const __half* c, long long c_bs, long long c_ls,
                   int B, int L, float* out) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (long long)B * L) return;
  const long long bb = row / L, l = row % L;
  const __half* ar = a + bb * a_bs + l * a_ls;
  const __half* cr = c + bb * c_bs + l * c_ls;
  float acc = 0.f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint4 x = *reinterpret_cast<const uint4*>(ar + 256 * h + 8 * lane);
    const uint4 y = *reinterpret_cast<const uint4*>(cr + 256 * h + 8 * lane);
    const __half2* xh = reinterpret_cast<const __half2*>(&x);
    const __half2* yh = reinterpret_cast<const __half2*>(&y);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 xf = __half22float2(xh[i]), yf = __half22float2(yh[i]);
      acc = fmaf(xf.x, yf.x, acc);
      acc = fmaf(xf.y, yf.y, acc);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[row] = acc;
}

}  // namespace b200

using namespace b200;

namespace {

template <int G>
int launch_d512_bwd(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b0, const CUtensorMap& b1,
                    const AttD512BwdParams& p, int B, void* stream) {
  using S_ = D5BwdShape<G>;
  static bool configured_dev[kMaxDevices] = {false};    // per device: function attributes live in the context
  const int dev = current_device();
  bool& configured = configured_dev[dev < 0 ? 0 : dev];
  if (!configured || dev < 0) {
    cudaError_t e = cudaFuncSetAttribute(attention_d512_bwd_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         S_::kSmem);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(attention_d512_bwd_kernel<%d> smem=%d): %s", G, S_::kSmem,
                     cudaGetErrorString(e));
      return (int)e;
    }
    configured = true;
  }
  const dim3 grid(((G == kGradQ ? p.Lq : p.Lk) + S_::kRows - 1) / S_::kRows, B);
  attention_d512_bwd_kernel<G><<<grid, S_::kThreads, S_::kSmem, (cudaStream_t)stream>>>(a0, a1, b0, b1, p);
  B200_CHECK_LAUNCH("attention_d512_bwd_kernel");
  return 0;
}

bool strides_ok(std::initializer_list<long long> ls, std::initializer_list<long long> bs) {
  for (long long x : ls)
    if (x % 8 != 0 || x < 512) return false;
  for (long long x : bs)
    if (x % 8 != 0 || x < 0) return false;
  return true;
}

}  // namespace

extern "C" int b200_rowdot_d512(const void* a, long long a_bs, long long a_ls, const void* c, long long c_bs,
                                long long c_ls, int B, int L, float* delta, void* stream) {
  B200_CHECK_ARG(a && c && delta, "b200_rowdot_d512: null pointer");
  B200_CHECK_ARG(B > 0 && B <= 65535 && L > 0, "b200_rowdot_d512: bad shape B=%d L=%d", B, L);
  B200_CHECK_ARG(strides_ok({a_ls, c_ls}, {a_bs, c_bs}),
                 "b200_rowdot_d512: strides must be multiples of 8 elements, row strides >= 512, batch strides >= 0");
  B200_CHECK_ARG((((uintptr_t)a | (uintptr_t)c) & 15) == 0 && ((uintptr_t)delta & 3) == 0,
                 "b200_rowdot_d512: a / c must be 16-byte aligned, delta 4-byte aligned");
  const long long rows = (long long)B * L;
  rowdot_d512_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)a, a_bs, a_ls, (const __half*)c, c_bs, c_ls, B, L, delta);
  B200_CHECK_LAUNCH("rowdot_d512_kernel");
  return 0;
}

extern "C" int b200_attention_d512_bwd(const void* q, long long q_bs, long long q_ls, const void* k, long long k_bs,
                                       long long k_ls, const void* v, long long v_bs, long long v_ls, const void* dout,
                                       long long do_bs, long long do_ls, const float* lse, const float* delta,
                                       void* dq, long long dq_bs, long long dq_ls, void* dk, long long dk_bs,
                                       long long dk_ls, void* dv, long long dv_bs, long long dv_ls, int B, int Lq,
                                       int Lk, float scale, void* stream) {
  B200_CHECK_ARG(q && k && v && dout && lse && delta && dq && dk && dv, "b200_attention_d512_bwd: null pointer");
  B200_CHECK_ARG(B > 0 && B <= 65535 && Lq > 0 && Lk > 0, "b200_attention_d512_bwd: bad shape B=%d Lq=%d Lk=%d", B,
                 Lq, Lk);
  B200_CHECK_ARG(strides_ok({q_ls, k_ls, v_ls, do_ls, dq_ls, dk_ls, dv_ls}, {q_bs, k_bs, v_bs, do_bs, dq_bs, dk_bs, dv_bs}),
                 "b200_attention_d512_bwd: strides must be multiples of 8 elements, row strides >= 512, batch "
                 "strides >= 0");
  B200_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)dout | (uintptr_t)dq | (uintptr_t)dk |
                   (uintptr_t)dv) & 15) == 0,
                 "b200_attention_d512_bwd: pointers must be 16-byte aligned");
  B200_CHECK_ARG((((uintptr_t)lse | (uintptr_t)delta) & 3) == 0,
                 "b200_attention_d512_bwd: lse / delta must be 4-byte aligned");
  // resident blocks in 64-row boxes; streamed tiles in 16-row (dQ, dK) and 32-row (dV) boxes
  CUtensorMap q64, o64, k16, v16, k64, v64, q16, o16, q32, o32;
  int r = encode_d512_tmap(&q64, q, Lq, B, q_ls, q_bs, 64);
  if (!r) r = encode_d512_tmap(&o64, dout, Lq, B, do_ls, do_bs, 64);
  if (!r) r = encode_d512_tmap(&k16, k, Lk, B, k_ls, k_bs, 16);
  if (!r) r = encode_d512_tmap(&v16, v, Lk, B, v_ls, v_bs, 16);
  if (!r) r = encode_d512_tmap(&k64, k, Lk, B, k_ls, k_bs, 64);
  if (!r) r = encode_d512_tmap(&v64, v, Lk, B, v_ls, v_bs, 64);
  if (!r) r = encode_d512_tmap(&q16, q, Lq, B, q_ls, q_bs, 16);
  if (!r) r = encode_d512_tmap(&o16, dout, Lq, B, do_ls, do_bs, 16);
  if (!r) r = encode_d512_tmap(&q32, q, Lq, B, q_ls, q_bs, 32);
  if (!r) r = encode_d512_tmap(&o32, dout, Lq, B, do_ls, do_bs, 32);
  if (r) return r;
  AttD512BwdParams p;
  p.Lq = Lq; p.Lk = Lk;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.scale = scale;
  p.lse = lse; p.delta = delta;
  p.out = (__half*)dq; p.o_bs = dq_bs; p.o_ls = dq_ls;
  r = launch_d512_bwd<kGradQ>(q64, o64, k16, v16, p, B, stream);
  if (r) return r;
  p.out = (__half*)dk; p.o_bs = dk_bs; p.o_ls = dk_ls;
  r = launch_d512_bwd<kGradK>(k64, v64, q16, o16, p, B, stream);
  if (r) return r;
  p.out = (__half*)dv; p.o_bs = dv_bs; p.o_ls = dv_ls;
  return launch_d512_bwd<kGradV>(k64, k64, q32, o32, p, B, stream);
}
