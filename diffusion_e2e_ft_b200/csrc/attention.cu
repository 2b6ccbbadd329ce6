// Flash attention on sm_90a: softmax(Q K^T * scale) V, no mask.  attention_kernel<D> (UNet heads of width D in
// {40, 64, 80, 160}) first, attention_d512_kernel (the single-head VAE mid-block) below.
//
// Warp-specialised, WG x 64 query rows per CTA: warp 4 WG = TMA producer (the Q tiles once, K/V tiles through a
// STAGES-deep smem ring), warps 0 .. 4 WG - 1 = WG consumer warpgroups, each owning 64 query rows with S, P and O in
// registers.  Per key tile j (BK keys) and warpgroup w:
//   S = Q_w K_j^T        wgmma m64n<BK>k16 x ceil(D/16), both operands from smem (K-major)  -> BK/2 fp32 registers
//   m, l, O *= alpha     online softmax; a row lives in the 4 lanes of a quad, so the row max / sum take 2 shuffles
//   P = exp2(S*c - m*c)  fp16, repacked in registers straight into the A-operand fragment layout
//   O += P V_j           wgmma m64n<D>k16 x BK/16, A = P from registers, V consumed MN-major from its [keys x d] tile
// The warpgroups run independently; while one exponentiates, the tensor core serves the others.
// Joint attention (GeoWizard): kv_segments = 2 walks the K/V tiles of batch b%(B/2) then
// b%(B/2)+B/2 — the concatenated K/V of attention.py:482-491 is never materialised.
//
// Operand tiles: Q / K / V are read in place through a 4-d tensor map {D, heads, L, B} whose innermost dimension is
// one head, in 64-column SWIZZLE_128B boxes: ceil(D/64) atoms per row, the columns past D zero-filled by TMA (a head
// slice of width 40 / 80 / 160 is 80 / 160 / 320 bytes, so the next head is never read).  The zero columns add
// nothing to Q K^T; the P V product is N = D wide and never reads them.
// Tile shape per D (the O accumulator is D/2 fp32 registers per thread, a K or V tile BK x ceil(D/64) x 128 bytes).
// A 416-thread CTA (13 warps, allocated as 16) may use 128 registers per thread, a 288-thread one (9 warps, as 12) 168:
//   D = 40, 64   3 warpgroups, 128-key tiles, 3 stages   (Q 24 KB + K/V 96 KB; S 64 + P 32 + O <= 32 registers)
//   D = 80       3 warpgroups,  64-key tiles, 3 stages   (Q 48 KB + K/V 96 KB; 128-key tiles spill at 128 registers)
//   D = 160      2 warpgroups,  64-key tiles, 3 stages   (Q 48 KB + K/V 144 KB; O 80 + S 32 + P 16 registers)
#include "attention.cuh"
#include "../../include/b200_e2eft.h"
#include "../../include/b200_e2eft_vae_attention.h"

namespace b200 {

constexpr int kBq = 64;                          // query rows per warpgroup

template <int D> struct AttCfg;
template <> struct AttCfg<40> { static constexpr int kWG = 3, kBk = 128, kStages = 3; };
template <> struct AttCfg<64> { static constexpr int kWG = 3, kBk = 128, kStages = 3; };
template <> struct AttCfg<80> { static constexpr int kWG = 3, kBk = 64, kStages = 3; };
template <> struct AttCfg<160> { static constexpr int kWG = 2, kBk = 64, kStages = 3; };

template <int D>
struct AttShape : AttCfg<D> {
  using AttCfg<D>::kWG;
  using AttCfg<D>::kBk;
  using AttCfg<D>::kStages;
  static constexpr int kAtoms = (D + 63) / 64;               // 64-column SWIZZLE_128B atoms per row
  static constexpr int kKSteps = (D + 15) / 16;              // k16 steps of Q K^T
  static constexpr int kThreads = 128 * kWG + 32;            // + the TMA producer warp
  static constexpr int kQAtom = kBq * 128;                   // one 64-row atom of a Q tile
  static constexpr int kKvAtom = kBk * 128;                  // one BK-row atom of a K or V tile
  static constexpr int kQBytes = kAtoms * kQAtom;
  static constexpr int kKvBytes = kAtoms * kKvAtom;
  static constexpr int kSmem = kWG * kQBytes + kStages * 2 * kKvBytes + 1024 + 1024;
  static_assert(kSmem <= 227 * 1024, "attention shared memory");
};

struct AttParams {
  int B, heads, Lq, Lk, kv_segments;
  float scale_log2;
  __half* out;
  long long o_bs, o_ls;
  float* lse;                  // optional [B][heads][Lq]: log2-domain log-sum-exp of the scaled scores (backward pass)
};

template <int D>
__global__ void __launch_bounds__(AttShape<D>::kThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const AttParams p) {
  using S_ = AttShape<D>;
  constexpr int kWG = S_::kWG, kBk = S_::kBk, kStages = S_::kStages, kAtoms = S_::kAtoms;
  constexpr int kQBytes = S_::kQBytes, kKvBytes = S_::kKvBytes;
  // 1024-byte alignment (SWIZZLE_128B atoms) by pointer arithmetic on the __shared__ array itself, so
  // the compiler keeps the shared address space (LDS/STS, no aliasing with global stores)
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                                   // [kWG][kAtoms][64 rows x 128 B]
  uint8_t* sK = sQ + kWG * kQBytes;                     // [stages][kAtoms][kBk rows x 128 B]
  uint8_t* sV = sK + kStages * kKvBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kStages * kKvBytes);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;
  uint64_t* v_full = k_full + kStages;
  uint64_t* kv_empty = v_full + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * (kWG * kBq);
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int tiles_per_seg = (p.Lk + kBk - 1) / kBk;
  const int n_tiles = tiles_per_seg * p.kv_segments;
  const int half_b = p.kv_segments == 2 ? p.B / 2 : 0;

  if (warp == 4 * kWG && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 128 * kWG);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4 * kWG) {
    // ===================================================================== TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, kWG * kQBytes);
      for (int w = 0; w < kWG; ++w)
        for (int a = 0; a < kAtoms; ++a)
          tma_load_4d(&tmQ, q_full, sQ + w * kQBytes + a * S_::kQAtom, 64 * a, h, q0 + w * kBq, b, kEvictFirst);
      int stage = 0;
      uint32_t phase = 0;
      for (int seg = 0; seg < p.kv_segments; ++seg) {
        const int kb = p.kv_segments == 2 ? (b % half_b) + seg * half_b : b;
        for (int j = 0; j < tiles_per_seg; ++j) {
          mbar_wait(&kv_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&k_full[stage], kKvBytes);
          for (int a = 0; a < kAtoms; ++a)
            tma_load_4d(&tmK, &k_full[stage], sK + stage * kKvBytes + a * S_::kKvAtom, 64 * a, h, j * kBk, kb,
                        kEvictLast);
          mbar_arrive_expect_tx(&v_full[stage], kKvBytes);
          for (int a = 0; a < kAtoms; ++a)
            tma_load_4d(&tmV, &v_full[stage], sV + stage * kKvBytes + a * S_::kKvAtom, 64 * a, h, j * kBk, kb,
                        kEvictLast);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  // ======================================================================= consumer warpgroups
  const int w = warp >> 2;
  // accumulator fragment: this thread holds rows r0 = 16 (warp & 3) + lane / 4 and r0 + 8 of the warpgroup's 64, columns
  // 8 i + 2 (lane % 4) + {0, 1}: s[4i], s[4i+1] for row r0, s[4i+2], s[4i+3] for row r0 + 8
  const int r0 = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const float c = p.scale_log2;
  const uint64_t qdesc = make_desc_sw128(smem_u32(sQ + w * kQBytes), 16, 1024);
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    const int jj = j % tiles_per_seg;
    const int valid = min(kBk, p.Lk - jj * kBk);
    float s[kBk / 2];
    mbar_wait(&k_full[st], ph);
    {
      const uint64_t kdesc = make_desc_sw128(smem_u32(sK + st * kKvBytes), 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < S_::kKSteps; ++k)        // k-step k: columns 16 (k % 4) .. of atom k / 4 (+32 B per step)
        wgmma_ss<kBk>(s, kstep_desc(qdesc, k, S_::kQAtom), kstep_desc(kdesc, k, S_::kKvAtom), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands<kBk / 2>(s);
    }
    if (valid < kBk) {                               // ragged last key tile: columns >= valid do not exist
#pragma unroll
      for (int i = 0; i < kBk / 8; ++i) {
        const int col = 8 * i + cq;
        if (col >= valid) { s[4 * i] = -INFINITY; s[4 * i + 2] = -INFINITY; }
        if (col + 1 >= valid) { s[4 * i + 1] = -INFINITY; s[4 * i + 3] = -INFINITY; }
      }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kBk / 8; ++i) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * i], s[4 * i + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * i + 2], s[4 * i + 3]));
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m[r], mx[r]);
      alpha[r] = ex2_approx((m[r] - m_new) * c);     // m = -inf on the first tile -> 0
      m[r] = m_new;
      mc[r] = m_new * c;
    }
    // P = exp2(S c - m c) as fp16 A fragments: k-chunk kk (keys 16 kk .. 16 kk + 15) = accumulator columns 8 (2 kk) ..
    uint32_t pa[kBk / 16][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < kBk / 16; ++kk) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int i = 2 * kk + hf;
        const float p0 = ex2_approx(fmaf(s[4 * i], c, -mc[0]));
        const float p1 = ex2_approx(fmaf(s[4 * i + 1], c, -mc[0]));
        const float p2 = ex2_approx(fmaf(s[4 * i + 2], c, -mc[1]));
        const float p3 = ex2_approx(fmaf(s[4 * i + 3], c, -mc[1]));
        rs[0] += p0 + p1;
        rs[1] += p2 + p3;
        pa[kk][2 * hf] = pack_half2(p0, p1);         // a0 / a2: row r0, a1 / a3: row r0 + 8
        pa[kk][2 * hf + 1] = pack_half2(p2, p3);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l[r] = fmaf(l[r], alpha[r], rs[r]);
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o[4 * i] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
    mbar_wait(&v_full[st], ph);
    {
      const uint32_t vbase = smem_u32(sV + st * kKvBytes);
      wgmma_fence_operands<D / 2>(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBk / 16; ++kk)       // B = V[16 kk .. 16 kk + 15, :]: MN-major, 2 groups of 8 key rows
        wgmma_rs_d<D>(o, pa[kk], make_desc_sw128(vbase + kk * 2048, S_::kKvAtom, 1024));   // atoms kKvAtom apart
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands<D / 2>(o);
    }
    mbar_arrive(&kv_empty[st]);                      // this warpgroup is done with K_j / V_j
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qrow = q0 + w * kBq + r0 + 8 * r;
    if (qrow >= p.Lq) continue;
    if (p.lse != nullptr && (lane & 3) == 0)       // P_ij = exp2(S_ij * c - lse): what the backward pass recomputes P from
      p.lse[((long long)b * p.heads + h) * p.Lq + qrow] = fmaf(m[r], c, log2f(l[r]));
    const float inv = 1.0f / l[r];
    __half* dst = p.out + (long long)b * p.o_bs + (long long)qrow * p.o_ls + h * D + cq;
#pragma unroll
    for (int i = 0; i < D / 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_half2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
  }
}

// ============================================================================= head_dim 512 (VAE mid-block)
// Flash attention for one head of width 512: softmax(Q K^T * scale) V with S and P never leaving the SM.
//
// 64 query rows per CTA (grid = ceil(Lq / 64) x B), two warpgroups and no producer warp: warpgroup w owns the
// d-columns 256 w .. 256 w + 255, both as its share of the Q K^T reduction and as its 256 output columns.
// Per key tile j (32 keys):
//   S_w = Q[:, w] K_j[:, w]^T   wgmma m64n32k16 x 16 from smem (K-major)       -> 16 fp32 registers per thread
//   S = S_0 + S_1               each warpgroup stores its partial tile to smem, one named barrier, each adds the
//                               other's: both warpgroups hold bit-identical S (fp32 addition commutes), so they run
//                               the same online softmax redundantly and agree on m, l and P
//   P = exp2(S*c - m*c)         fp16, packed in registers into the A-operand fragments (as the d64 kernel)
//   O_w += P V_j[:, w]          wgmma m64n256k16 x 2, A = P from registers, V consumed MN-major
// Q, K and V arrive by TMA in 64-column SWIZZLE_128B boxes (8 boxes per 512-wide row block).  K and V are double
// buffered; thread 0 issues the loads.  At the named barrier of tile j both warpgroups have finished S_j and P V_{j-1},
// so K_{j+2} and V_{j+1} go into the buffers those freed.  The partial-S tiles are double buffered by tile parity: a
// warpgroup overwrites its tile of parity j only after barrier j+1, which its partner passes after reading it.
// Budget per thread: O 128 + S 16 + P 8 fp32/b32 registers (+ m, l, addressing); 256 threads may use 255 each.
// (A separate producer warp would make the CTA 288 threads, which the register file serves as 384: 168 each.)
// Shared memory: Q 64 KB (resident) + 2 x K 32 KB + 2 x V 32 KB + 2 x 2 partial-S tiles of 8 KB = 224 KB + barriers
// + 1 KB alignment slack, of the 227 KB an sm_90 CTA may use.
// With `lse` set, warpgroup 0 also stores each row's log2-domain log-sum-exp m c + log2(l) (attention_kernel<D>'s
// convention), which attention_d512_bwd.cu recomputes P from; O is computed and stored the same way either way.
constexpr int kD5 = 512;
constexpr int kD5WG = 2;                          // warpgroups
constexpr int kD5Cols = kD5 / kD5WG;             // output columns per warpgroup
constexpr int kD5Threads = 128 * kD5WG;
constexpr int kD5Bq = 64;                         // query rows per CTA
constexpr int kD5Bk = 32;                         // keys per tile
constexpr int kD5Box = kD5Bq * 64 * 2;            // one 64-row x 64-column fp16 TMA box of Q, 8 KB
constexpr int kD5QBytes = (kD5 / 64) * kD5Box;    // 64 rows x 512 columns, 64 KB
constexpr int kD5KBox = kD5Bk * 64 * 2;           // one 32-key x 64-column box of K or V, 4 KB
constexpr int kD5KvBytes = (kD5 / 64) * kD5KBox;  // 32 keys x 512 columns, 32 KB
constexpr int kD5XFloats = kD5Bq * kD5Bk;         // one partial S tile
constexpr int kD5Smem = kD5QBytes + 4 * kD5KvBytes + 2 * kD5WG * kD5XFloats * 4 + 64 + 1024;
static_assert(kD5Smem <= 227 * 1024, "attention_d512 shared memory");

struct AttD512Params {
  int Lq, Lk;
  float scale_log2;
  __half* out;
  long long o_bs, o_ls;
  float* lse;                  // optional [B][Lq]
};

__device__ __forceinline__ void d512_load_kv(const CUtensorMap* tm, uint64_t* bar, uint8_t* dst, int key0, int b) {
  mbar_arrive_expect_tx(bar, kD5KvBytes);
  for (int c = 0; c < kD5 / 64; ++c) tma_load_3d(tm, bar, dst + c * kD5KBox, 64 * c, key0, b, kEvictNormal);
}

__global__ void __launch_bounds__(kD5Threads, 1)
attention_d512_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const AttD512Params p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                                   // [8 boxes][64 rows][64 columns]
  uint8_t* sK = sQ + kD5QBytes;                         // [2 buffers][8 boxes][32 keys][64 columns]
  uint8_t* sV = sK + 2 * kD5KvBytes;
  float* sX = reinterpret_cast<float*>(sV + 2 * kD5KvBytes);   // [2 parities][kD5WG][partial S tile]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sX + 2 * kD5WG * kD5XFloats);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;                          // [2]
  uint64_t* v_full = bars + 3;                          // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kD5Bq;
  const int b = blockIdx.y;
  const int n_tiles = (p.Lk + kD5Bk - 1) / kD5Bk;
  const bool loader = threadIdx.x == 0;

  if (loader) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < 5; ++i) mbar_init(&bars[i], 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(q_full, kD5QBytes);
    for (int c = 0; c < kD5 / 64; ++c) tma_load_3d(&tmQ, q_full, sQ + c * kD5Box, 64 * c, q0, b, kEvictFirst);
    d512_load_kv(&tmK, &k_full[0], sK, 0, b);
    if (n_tiles > 1) d512_load_kv(&tmK, &k_full[1], sK + kD5KvBytes, kD5Bk, b);
    d512_load_kv(&tmV, &v_full[0], sV, 0, b);
  }
  __syncthreads();

  const int w = warp >> 2;
  const int t = threadIdx.x & 127;
  const int r0 = (warp & 3) * 16 + (lane >> 2);     // accumulator fragment rows r0, r0 + 8 (see wgmma.cuh)
  const int cq = 2 * (lane & 3);
  float o[kD5Cols / 2];
#pragma unroll
  for (int i = 0; i < kD5Cols / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const float c = p.scale_log2;
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int buf = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    const int valid = min(kD5Bk, p.Lk - j * kD5Bk);
    float s[kD5Bk / 2];
    mbar_wait(&k_full[buf], ph);
    wgmma_fence();
#pragma unroll
    for (int cc = 0; cc < kD5Cols / 64; ++cc) {
      const int box = w * (kD5Cols / 64) + cc;
      const uint64_t qdesc = make_desc_sw128(smem_u32(sQ + box * kD5Box), 16, 1024);
      const uint64_t kdesc = make_desc_sw128(smem_u32(sK + buf * kD5KvBytes + box * kD5KBox), 16, 1024);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n32<0, 0>(s, qdesc + 2 * k, kdesc + 2 * k, (cc | k) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands<kD5Bk / 2>(s);
    // S = S_0 + S_1: thread t of one warpgroup holds the same fragment positions as thread t of the other
    float4* x_own = reinterpret_cast<float4*>(sX + (buf * kD5WG + w) * kD5XFloats);
    const float4* x_other = reinterpret_cast<const float4*>(sX + (buf * kD5WG + (w ^ 1)) * kD5XFloats);
#pragma unroll
    for (int i = 0; i < kD5Bk / 8; ++i) x_own[i * 128 + t] = make_float4(s[4 * i], s[4 * i + 1], s[4 * i + 2], s[4 * i + 3]);
    named_barrier_sync(1, kD5Threads);
    if (loader) {                                    // K buffer `buf` and V buffer `buf ^ 1` are free now
      if (j + 2 < n_tiles) d512_load_kv(&tmK, &k_full[buf], sK + buf * kD5KvBytes, (j + 2) * kD5Bk, b);
      if (j + 1 < n_tiles) d512_load_kv(&tmV, &v_full[buf ^ 1], sV + (buf ^ 1) * kD5KvBytes, (j + 1) * kD5Bk, b);
    }
#pragma unroll
    for (int i = 0; i < kD5Bk / 8; ++i) {
      const float4 v = x_other[i * 128 + t];
      s[4 * i] += v.x;
      s[4 * i + 1] += v.y;
      s[4 * i + 2] += v.z;
      s[4 * i + 3] += v.w;
    }
    if (valid < kD5Bk) {                             // ragged last key tile: columns >= valid do not exist
#pragma unroll
      for (int i = 0; i < kD5Bk / 8; ++i) {
        const int col = 8 * i + cq;
        if (col >= valid) { s[4 * i] = -INFINITY; s[4 * i + 2] = -INFINITY; }
        if (col + 1 >= valid) { s[4 * i + 1] = -INFINITY; s[4 * i + 3] = -INFINITY; }
      }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kD5Bk / 8; ++i) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * i], s[4 * i + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * i + 2], s[4 * i + 3]));
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m[r], mx[r]);
      alpha[r] = ex2_approx((m[r] - m_new) * c);     // m = -inf on the first tile -> 0
      m[r] = m_new;
      mc[r] = m_new * c;
    }
    uint32_t pa[kD5Bk / 16][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < kD5Bk / 16; ++kk) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int i = 2 * kk + hf;
        const float p0 = ex2_approx(fmaf(s[4 * i], c, -mc[0]));
        const float p1 = ex2_approx(fmaf(s[4 * i + 1], c, -mc[0]));
        const float p2 = ex2_approx(fmaf(s[4 * i + 2], c, -mc[1]));
        const float p3 = ex2_approx(fmaf(s[4 * i + 3], c, -mc[1]));
        rs[0] += p0 + p1;
        rs[1] += p2 + p3;
        pa[kk][2 * hf] = pack_half2(p0, p1);
        pa[kk][2 * hf + 1] = pack_half2(p2, p3);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l[r] = fmaf(l[r], alpha[r], rs[r]);
#pragma unroll
    for (int i = 0; i < kD5Cols / 8; ++i) {
      o[4 * i] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
    mbar_wait(&v_full[buf], ph);
    {
      // B = V[16 kk .. 16 kk + 15][256 w ..]: MN-major, the four 64-column boxes of this warpgroup 4 KB apart (LBO)
      const uint32_t vbase = smem_u32(sV + buf * kD5KvBytes + w * (kD5Cols / 64) * kD5KBox);
      wgmma_fence_operands<kD5Cols / 2>(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kD5Bk / 16; ++kk)
        wgmma_m64n256_rs_bmn(o, pa[kk], make_desc_sw128(vbase + kk * 2048, kD5KBox, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands<kD5Cols / 2>(o);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qrow = q0 + r0 + 8 * r;
    if (qrow >= p.Lq) continue;                      // rows past Lq came from TMA zero fill
    if (p.lse != nullptr && w == 0 && (lane & 3) == 0)   // both warpgroups hold the same m and l
      p.lse[(long long)b * p.Lq + qrow] = fmaf(m[r], c, log2f(l[r]));
    const float inv = 1.0f / l[r];
    __half* dst = p.out + (long long)b * p.o_bs + (long long)qrow * p.o_ls + w * kD5Cols + cq;
#pragma unroll
    for (int i = 0; i < kD5Cols / 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_half2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
  }
}

}  // namespace b200

using namespace b200;


namespace {

template <int D>
int launch_attention(const void* q, long long q_bs, long long q_ls, const void* k, long long k_bs, long long k_ls,
                     const void* v, long long v_bs, long long v_ls, const AttParams& p, void* stream) {
  using S_ = AttShape<D>;
  CUtensorMap tq, tk, tv;
  int r = encode_head_tmap(&tq, q, D, p.heads, p.Lq, p.B, q_ls, q_bs, kBq);
  if (!r) r = encode_head_tmap(&tk, k, D, p.heads, p.Lk, p.B, k_ls, k_bs, S_::kBk);
  if (!r) r = encode_head_tmap(&tv, v, D, p.heads, p.Lk, p.B, v_ls, v_bs, S_::kBk);
  if (r) return r;
  static bool configured_dev[kMaxDevices] = {false};      // per device: function attributes live in the context
  const int dev_ = current_device();
  bool& configured = configured_dev[dev_ < 0 ? 0 : dev_];
  if (!configured || dev_ < 0) {
    cudaError_t e = cudaFuncSetAttribute(attention_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, S_::kSmem);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(attention head_dim=%d smem=%d): %s", D, S_::kSmem, cudaGetErrorString(e));
      return (int)e;
    }
    configured = true;
  }
  dim3 grid((p.Lq + S_::kWG * kBq - 1) / (S_::kWG * kBq), p.heads, p.B);
  attention_kernel<D><<<grid, S_::kThreads, S_::kSmem, (cudaStream_t)stream>>>(tq, tk, tv, p);
  B200_CHECK_LAUNCH("attention_kernel");
  return 0;
}

}  // namespace

extern "C" int b200_attention(const void* q, long long q_bs, long long q_ls, const void* k, long long k_bs,
                              long long k_ls, const void* v, long long v_bs, long long v_ls, void* out, long long o_bs,
                              long long o_ls, int B, int heads, int head_dim, int Lq, int Lk, int kv_segments,
                              float scale, float* lse, void* stream) {
  B200_CHECK_ARG(head_dim == 40 || head_dim == 64 || head_dim == 80 || head_dim == 160,
                 "b200_attention: head_dim=%d is not one of 40, 64, 80, 160", head_dim);
  B200_CHECK_ARG(q && k && v && out, "b200_attention: null pointer");
  B200_CHECK_ARG(B > 0 && B <= 65535 && heads > 0 && heads <= 65535 && Lq > 0 && Lk > 0,
                 "b200_attention: bad shape B=%d heads=%d Lq=%d Lk=%d", B, heads, Lq, Lk);
  B200_CHECK_ARG(kv_segments == 1 || (kv_segments == 2 && B % 2 == 0), "b200_attention: kv_segments=%d B=%d", kv_segments, B);
  B200_CHECK_ARG(q_ls % 8 == 0 && k_ls % 8 == 0 && v_ls % 8 == 0 && o_ls % 8 == 0 && q_bs % 8 == 0 &&
                     k_bs % 8 == 0 && v_bs % 8 == 0 && o_bs % 8 == 0,
                 "b200_attention: strides must be multiples of 8 elements");
  B200_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15) == 0,
                 "b200_attention: pointers must be 16-byte aligned");
  AttParams p;
  p.B = B; p.heads = heads; p.Lq = Lq; p.Lk = Lk; p.kv_segments = kv_segments;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = (__half*)out; p.o_bs = o_bs; p.o_ls = o_ls;
  p.lse = lse;
  switch (head_dim) {
    case 40: return launch_attention<40>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, p, stream);
    case 64: return launch_attention<64>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, p, stream);
    case 80: return launch_attention<80>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, p, stream);
    default: return launch_attention<160>(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, p, stream);
  }
}

extern "C" int b200_attention_d64(const void* q, long long q_bs, long long q_ls, const void* k,
                                  long long k_bs, long long k_ls, const void* v, long long v_bs,
                                  long long v_ls, void* out, long long o_bs, long long o_ls, int B,
                                  int heads, int Lq, int Lk, int kv_segments, float scale, float* lse,
                                  void* stream) {
  return b200_attention(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, out, o_bs, o_ls, B, heads, 64, Lq, Lk,
                        kv_segments, scale, lse, stream);
}

extern "C" int b200_attention_d512_lse(const void* q, long long q_bs, long long q_ls, const void* k, long long k_bs,
                                       long long k_ls, const void* v, long long v_bs, long long v_ls, void* out,
                                       long long o_bs, long long o_ls, int B, int Lq, int Lk, float scale, float* lse,
                                       void* stream) {
  B200_CHECK_ARG(q && k && v && out, "b200_attention_d512: null pointer");
  B200_CHECK_ARG(B > 0 && B <= 65535 && Lq > 0 && Lk > 0, "b200_attention_d512: bad shape B=%d Lq=%d Lk=%d", B, Lq, Lk);
  B200_CHECK_ARG(q_ls % 8 == 0 && k_ls % 8 == 0 && v_ls % 8 == 0 && o_ls % 8 == 0 && q_bs % 8 == 0 &&
                     k_bs % 8 == 0 && v_bs % 8 == 0 && o_bs % 8 == 0,
                 "b200_attention_d512: strides must be multiples of 8 elements");
  B200_CHECK_ARG(q_ls >= kD5 && k_ls >= kD5 && v_ls >= kD5 && o_ls >= kD5 && q_bs >= 0 && k_bs >= 0 && v_bs >= 0 &&
                     o_bs >= 0,
                 "b200_attention_d512: row strides must be >= 512 elements, batch strides >= 0");
  B200_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15) == 0,
                 "b200_attention_d512: pointers must be 16-byte aligned");
  B200_CHECK_ARG(((uintptr_t)lse & 3) == 0, "b200_attention_d512: lse must be 4-byte aligned");
  CUtensorMap tq, tk, tv;
  int r = encode_d512_tmap(&tq, q, Lq, B, q_ls, q_bs, kD5Bq);
  if (!r) r = encode_d512_tmap(&tk, k, Lk, B, k_ls, k_bs, kD5Bk);
  if (!r) r = encode_d512_tmap(&tv, v, Lk, B, v_ls, v_bs, kD5Bk);
  if (r) return r;
  static bool configured_dev[kMaxDevices] = {false};
  const int dev_ = current_device();
  bool& configured = configured_dev[dev_ < 0 ? 0 : dev_];
  if (!configured || dev_ < 0) {
    cudaError_t e = cudaFuncSetAttribute(attention_d512_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kD5Smem);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(attention_d512 smem=%d): %s", kD5Smem, cudaGetErrorString(e));
      return (int)e;
    }
    configured = true;
  }
  AttD512Params p;
  p.Lq = Lq; p.Lk = Lk;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = (__half*)out; p.o_bs = o_bs; p.o_ls = o_ls;
  p.lse = lse;
  dim3 grid((Lq + kD5Bq - 1) / kD5Bq, B);
  attention_d512_kernel<<<grid, kD5Threads, kD5Smem, (cudaStream_t)stream>>>(tq, tk, tv, p);
  B200_CHECK_LAUNCH("attention_d512_kernel");
  return 0;
}

extern "C" int b200_attention_d512(const void* q, long long q_bs, long long q_ls, const void* k, long long k_bs,
                                   long long k_ls, const void* v, long long v_bs, long long v_ls, void* out,
                                   long long o_bs, long long o_ls, int B, int Lq, int Lk, float scale, void* stream) {
  return b200_attention_d512_lse(q, q_bs, q_ls, k, k_bs, k_ls, v, v_bs, v_ls, out, o_bs, o_ls, B, Lq, Lk, scale,
                                 nullptr, stream);
}
