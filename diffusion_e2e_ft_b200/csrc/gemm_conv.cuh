// wgmma GEMM + im2col-free implicit-GEMM convolution for sm_90a.
//
//   D[M,N] = epilogue( A[M,K] * W[N,K]^T )        fp16 operands, fp32 accumulate in registers
//
// * A/W tiles are staged by TMA (cp.async.bulk.tensor, SWIZZLE_128B) into a multi-stage smem ring.
// * LINEAR mode: A is a 3-D tensor (K, rows, batch).
// * CONV mode:   A is the NHWC activation itself, a 4-D tensor (C, W, H, N).  An M-tile is a
//   bw x bh patch of output pixels of one image; k-block (tap, c-block) is fetched with the box
//   (64, bw, bh, 1) at coordinates (c0, w0*s+dx, h0*s+dy, n) — the halo / padding comes from TMA
//   out-of-bounds zero fill, the stride from the tensor map's element strides.  No im2col buffer.
//   Optional second source A2 (same pixel tiling, 1x1) appends k-blocks: this fuses the
//   ResnetBlock2D 1x1 `conv_shortcut` into conv2's accumulation.
// * Two consumer warpgroups (warps 0-7) each issue wgmma m64nBLOCK_Nk16 for one 64-row half of the 128-row tile,
//   accumulating in registers; warps 8-11 are the producer warpgroup, of which one lane issues the TMA loads.  The
//   producer warpgroup gives up registers (setmaxnreg.dec 40) so the consumers can hold the 128 accumulator registers
//   of a 256-wide tile plus the epilogue's working set without spilling (setmaxnreg.inc 232).
// * Epilogue, vectorised swapped orientation (VEC): straight from the accumulator registers.  Each warp owns 16 rows
//   (channels) of the tile and turns them, 32 columns (pixels) at a time, into per-pixel channel runs through a small
//   per-warp smem tile.  No CTA barrier and no use of the operand ring, so the producer fills the ring with the next
//   tile's operands while the epilogue runs.
// * Epilogue, every other instantiation: the accumulators are staged as fp32 into the (then idle) operand ring and the
//   same 8 warps run the epilogue from there: thread (warp & 3, lane) owns accumulator row 32 (warp & 3) + lane, the two
//   warps of a row quadrant take alternate 32-column chunks.  The producer starts the next tile's loads once every
//   epilogue thread has released the ring.
// * Persistent: grid = min(#tiles, #SMs), static round-robin tile schedule (n fastest).
#pragma once
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"

namespace b200 {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;       // 64 x fp16 = one 128-byte swizzle row
constexpr int kMmaK = 16;
constexpr int kGemmThreads = 384;   // warps 0-7: two MMA + epilogue warpgroups, warps 8-11: producer warpgroup
constexpr int kEpiWarps = 8;
constexpr int kConsumerThreads = 32 * kEpiWarps;
// per-thread register budgets after the role split: 128 * 40 + 256 * 232 <= 384 * 168 (the launch allocation)
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
constexpr int kMaxTaps = 9;

enum EpiAct { ACT_NONE = 0, ACT_SILU = 1, ACT_GEGLU = 2, ACT_GELU = 3, ACT_EXP2 = 4 };   // EXP2: P = exp2(alpha S - lse)

struct GemmParams {
  int M, N, num_k_blocks;
  int batch, m_tiles, n_tiles;
  int a_batched, b_batched;    // operand has a batch dimension (else shared across the batch)
  int act_mn, w_mn;            // LINEAR: the activation / weight operand is stored [K][rows] (MN-major, e.g. dY for a weight
                               // gradient dY^T X) and is fed to the MMA as is — no transposition pass.  smem layout per
                               // stage: rows / 64 boxes of [64 k-rows][64 rows x 2 B], 8192 B apart (descriptor LBO 8192,
                               // SBO 1024)
  // ---- conv geometry (conv != 0)
  int conv;
  int Ho, Wo;                  // conv-output grid the M tiles walk over
  int bw, bh, tiles_w, tiles_h;
  int col_pitch;               // accumulator column q of a conv tile = pixel (q / col_pitch, q % col_pitch): bw normally,
                               // bw + 2 in halo mode (the two halo columns of every patch row ride along as dead columns)
  int halo_n;                  // halo mode: N of the per-tap MMA = round_up64((bw + 2) * bh)
  int cin_blocks, num_taps, in_stride;
  int tap_dy[kMaxTaps], tap_dx[kMaxTaps];
  int k2_blocks;               // trailing k-blocks read from A2 (1x1 shortcut)
  // output pixel mapping: pixel (ho,wo) -> (ho*out_mul+out_oy, wo*out_mul+out_ox) in OHxOW
  int out_mul, out_oy, out_ox, OH, OW;
  // ---- epilogue
  void* out;
  long long ldo, out_batch_stride;
  int out_f32;
  int vec_ok;                  // 16-byte vector stores/loads are aligned (ldo, ld_res % 8 == 0)
  int out_nchw;                // conv only: write fp32/fp16 NCHW (small Cout) instead of NHWC
  const float* bias;           // [N] (or [M] when bias_row)
  int bias_row;
  long long bias_bs;           // bias_row: element offset of the bias vector per batch index
  const float* rowvec;         // per-image vector, indexed [img*ld_rowvec + col]
  long long ld_rowvec;
  int res_mul;                 // residual operand multiplies (out = act(acc+bias) * residual) instead of adding
  const void* residual;        // same dtype as out
  long long ld_res, res_batch_stride;
  int act;
  float alpha;                 // scale applied to the accumulator before bias
  __half* out2;                // optional second output: fp16 copy of `out` (same layout) for a following GEMM/conv operand
  double* chan_stats;          // optional [img][N][2] per-channel (sum, sum of squares) of the stored values: shifted
                               // fp32 partial sums per thread (no cancellation for |mean| >> std), fp64 atomics
  int rows_per_img;            // LINEAR + chan_stats: img = row / rows_per_img (tiles never straddle images)
  int debug;                   // perf experiments: 1 = no epilogue stores, 2 = no A loads, 4 = no B loads, 8 = no MMAs, 16 = empty epilogue
};

// floats per pixel row of the vectorised epilogue's per-warp [32 pixels][16 channels] transpose tile: 16-byte aligned,
// and 20 makes both the fragment stores and the 16-byte pixel-row loads bank-conflict-free
constexpr int kSwapPitch = 20;

// HALO (conv3x3, stride 1, swapped orientation): the activation patch of a tile — (bh+2) x (bw+2) pixels x 64 channels —
// is loaded ONCE per 64-channel block and all nine taps are issued as row-shifted views of it (wgmma descriptors with a
// 128-byte-granular start address), instead of nine separate bw x bh boxes: 9x -> (bh+2)(bw+2)/(bh*bw) ~ 1.5x of
// L2 -> smem activation traffic.
constexpr int kHaloMaxPatchPix = 400;                       // (bw+2)*(bh+2) <= 400: 64x4, 96x2, 48x5, 32x8 tiles
constexpr int kHaloPatchBytes = kHaloMaxPatchPix * 128;     // one 64-channel slab of the patch (50 KB, 1024-aligned)
constexpr int kHaloWStages = 5;                             // 128 x 64 weight tiles in flight (16 KB each)

template <int BLOCK_N, bool SWAP = false, bool HALO = false>
struct GemmSmem {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarrierBytes = 1024;
  // normal: per-epilogue-warp 32x33 fp32 transpose tile + per-warp row tables (out / residual offsets, row bias)
  // swapped: pixel-offset tables [2 acc][out|res][BLOCK_N] + flags, then per-warp 32 x kSwapPitch fp32 transpose tiles
  static constexpr int kSwapTabBytes = 4 * BLOCK_N * 4 + 256;
  static constexpr int kStagingBytes = SWAP ? kSwapTabBytes + kEpiWarps * 32 * kSwapPitch * 4 : kEpiWarps * 32 * 33 * 4;
  static constexpr int kRowMetaBytes = SWAP ? 0 : kEpiWarps * 640;
  static constexpr int kEpiBytes = kStagingBytes + kRowMetaBytes;
  static constexpr int kBudget = 227 * 1024 - 1024 /*align slack*/ - kBarrierBytes - kEpiBytes;
  static constexpr int kStages = HALO ? kHaloWStages : ((kBudget / kStageBytes) > 8 ? 8 : (kBudget / kStageBytes));
  static constexpr int kOperandBytes = HALO ? kHaloWStages * kABytes + 2 * kHaloPatchBytes : kStages * kStageBytes;
  static constexpr int kTotalBytes = kOperandBytes + kEpiBytes + kBarrierBytes + 1024;
  static_assert(kTotalBytes <= 227 * 1024, "shared memory budget");
  // fp32 accumulator tile staged for the epilogue in the operand area; the odd-ish pitch keeps both the fragment
  // stores (8 rows x 4 column pairs per warp) and the row reads (32 rows per warp) at <= 2-way bank conflicts
  static constexpr int kAccPitch = BLOCK_N + 9;
  static constexpr int kAccBytes = kBlockM * kAccPitch * 4;
  static_assert(kAccBytes <= kOperandBytes, "the accumulator tile must fit the operand ring");
};

template <typename OutT>
__device__ __forceinline__ void store_chunk8(OutT* dst, const float* v);
template <>
__device__ __forceinline__ void store_chunk8<float>(float* dst, const float* v) {
  reinterpret_cast<float4*>(dst)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(dst)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
template <>
__device__ __forceinline__ void store_chunk8<__half>(__half* dst, const float* v) {
  __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
  __half2 h2 = __floats2half2_rn(v[4], v[5]), h3 = __floats2half2_rn(v[6], v[7]);
  uint4 u;
  u.x = *reinterpret_cast<uint32_t*>(&h0);
  u.y = *reinterpret_cast<uint32_t*>(&h1);
  u.z = *reinterpret_cast<uint32_t*>(&h2);
  u.w = *reinterpret_cast<uint32_t*>(&h3);
  *reinterpret_cast<uint4*>(dst) = u;
}
template <typename OutT>
__device__ __forceinline__ void load_chunk8(const OutT* src, float* v);
template <>
__device__ __forceinline__ void load_chunk8<float>(const float* src, float* v) {
  float4 a = reinterpret_cast<const float4*>(src)[0], b = reinterpret_cast<const float4*>(src)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <>
__device__ __forceinline__ void load_chunk8<__half>(const __half* src, float* v) {
  uint4 u = *reinterpret_cast<const uint4*>(src);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __half22float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// erf-GELU with erf from Abramowitz & Stegun 7.1.26 (|abs err| <= 1.5e-7): 2 MUFU + ~10 FMA per element
// instead of the ~45-instruction two-branch libdevice erff.
__device__ __forceinline__ float gelu_erf_f(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float e = __expf(-z * z);
  const float erf_abs = fmaf(-poly * t, e, 1.0f);          // erf(|x|/sqrt2)
  const float erf_v = copysignf(erf_abs, x);
  return 0.5f * x * (1.0f + erf_v);
}

// CW consecutive staged accumulator values of one row
template <int CW>
__device__ __forceinline__ void acc_ld(const float* src, uint32_t (&r)[CW]) {
#pragma unroll
  for (int j = 0; j < CW; ++j) r[j] = __float_as_uint(src[j]);
}

// D (+)= A B^T for one 64-row half of the tile: wgmma m64nNk16 with the operand majorness as immediates
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_n(float* d, uint64_t da, uint64_t db, int scale_d) {
  if constexpr (N == 32) wgmma_m64n32<TA, TB>(d, da, db, scale_d);
  else if constexpr (N == 64) wgmma_m64n64<TA, TB>(d, da, db, scale_d);
  else if constexpr (N == 128) wgmma_m64n128<TA, TB>(d, da, db, scale_d);
  else if constexpr (N == 160) wgmma_m64n160<TA, TB>(d, da, db, scale_d);
  else if constexpr (N == 192) wgmma_m64n192<TA, TB>(d, da, db, scale_d);
  else {
    static_assert(N == 256, "tile width without a wgmma wrapper");
    wgmma_m64n256<TA, TB>(d, da, db, scale_d);
  }
}
template <int N>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db, int scale_d, bool a_mn, bool b_mn) {
  if (!a_mn && !b_mn) wgmma_n<N, 0, 0>(d, da, db, scale_d);
  else if (!a_mn) wgmma_n<N, 0, 1>(d, da, db, scale_d);
  else if (!b_mn) wgmma_n<N, 1, 0>(d, da, db, scale_d);
  else wgmma_n<N, 1, 1>(d, da, db, scale_d);
}
// halo mode: N = halo_n (a multiple of 64, <= 256), both operands K-major
__device__ __forceinline__ void wgmma_halo(float* d, uint64_t da, uint64_t db, int scale_d, int n) {
  if (n <= 64) wgmma_n<64, 0, 0>(d, da, db, scale_d);
  else if (n <= 128) wgmma_n<128, 0, 0>(d, da, db, scale_d);
  else if (n <= 192) wgmma_n<192, 0, 0>(d, da, db, scale_d);
  else wgmma_n<256, 0, 0>(d, da, db, scale_d);
}

// SWAP = false: accumulator rows = 128 pixels, columns = BLOCK_N output channels.
// SWAP = true : operands swapped — rows = 128 output channels (weights are the M operand), columns =
//               BLOCK_N pixels (activations are the N operand).  Used when Cout % 128 == 0: a 128-channel
//               layer then issues 128x256 MMAs (half the operand smem traffic and half the per-k-block
//               barrier round trips of 128x128), and since rows = channels the NHWC stores of one
//               accumulator column are contiguous — no smem transpose in the epilogue.
// VEC (swapped orientation only): the vectorised epilogue (smem transpose, 16-byte accesses, statistics carried across
// tiles) INSTEAD of the direct lane = channel one; a template parameter so that each instantiation carries one epilogue
// only — with both compiled in, the small-K GEMMs of the transformer blocks (epilogue-bound) lose time to spills and
// instruction-cache misses.
template <int BLOCK_N, typename OutT, bool SWAP, bool GEGLU, bool HALO = false, bool VEC = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  static_assert(!HALO || (SWAP && !GEGLU && BLOCK_N == 256 && VEC), "halo mode: swapped orientation, 256 accumulator columns");
  static_assert(!VEC || SWAP, "the vectorised epilogue belongs to the swapped orientation");
  using S = GemmSmem<BLOCK_N, SWAP, HALO>;
  constexpr int kStages = S::kStages;
  // 1024-byte alignment (SWIZZLE_128B atoms) by pointer arithmetic on the __shared__ array itself, so
  // the compiler keeps the shared address space (LDS/STS, no aliasing with global stores)
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;                                // HALO: the weight-tile ring
  uint8_t* smem_b = smem + kStages * S::kABytes;         // HALO: the two patch buffers
  uint8_t* stage_smem = smem + S::kOperandBytes;
  uint8_t* rowmeta_smem = stage_smem + S::kStagingBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kOperandBytes + S::kEpiBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;
  uint64_t* acc_empty = bars + 2 * kStages;            // every epilogue thread is done with the staged accumulators
  uint64_t* patch_full = bars + 2 * kStages + 1;        // HALO only
  uint64_t* patch_empty = patch_full + 2;
  float* acc_smem = reinterpret_cast<float*>(smem);     // [kBlockM][kAccPitch] fp32, in the operand ring between tiles

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.batch * p.m_tiles * p.n_tiles;
  // bytes each stage receives: the activation box of a conv tile may hold fewer pixels than the tile
  const uint32_t act_bytes = p.conv ? (uint32_t)(p.bw * p.bh * kBlockK * 2)
                                    : (uint32_t)((SWAP ? BLOCK_N : kBlockM) * kBlockK * 2);
  const uint32_t w_bytes = (uint32_t)((SWAP ? kBlockM : BLOCK_N) * kBlockK * 2);
  const uint32_t a_bytes = SWAP ? w_bytes : act_bytes;
  const uint32_t b_bytes = SWAP ? act_bytes : w_bytes;

  if (warp == kEpiWarps && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.k2_blocks) tma_prefetch_desc(&tmA2);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumerThreads);
    }
    mbar_init(acc_empty, kConsumerThreads);
    if constexpr (HALO) {
      for (int i = 0; i < 2; ++i) {
        mbar_init(&patch_full[i], 1);
        mbar_init(&patch_empty[i], kConsumerThreads);
      }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kEpiWarps) {
    // ======================================================================= TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp != kEpiWarps) return;
    // VEC epilogues never touch the ring, so only the staged epilogues hold the producer back at a tile boundary
    uint32_t aphase = 0;
    if constexpr (HALO) {
      if (lane == 0) {
        int ws = 0, pb = 0;
        uint32_t wphase = 0, pphase = 0;
        const uint32_t patch_bytes = (uint32_t)((p.bw + 2) * (p.bh + 2) * kBlockK * 2);
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
          const int n_blk = tile % p.n_tiles;                       // channel tile (fastest: neighbours share the patch in L2)
          const int m_blk = tile / p.n_tiles;
          const int tw = m_blk % p.tiles_w;
          const int r2 = m_blk / p.tiles_w;
          const int th = r2 % p.tiles_h;
          const int img = r2 / p.tiles_h;
          const int h0 = th * p.bh, w0 = tw * p.bw;
          if constexpr (!VEC) {
            mbar_wait(acc_empty, aphase ^ 1);                // the accumulators of the previous tile left the ring
            aphase ^= 1;
          }
          for (int blk = 0; blk < p.cin_blocks + p.k2_blocks; ++blk) {
            const bool main = blk < p.cin_blocks;
            mbar_wait(&patch_empty[pb], pphase ^ 1);
            mbar_arrive_expect_tx(&patch_full[pb], (p.debug & 2) ? 0u : patch_bytes);
            // one box = the whole (bh+2) x (bw+2) halo patch of this 64-channel block; image borders = OOB zero fill
            if (p.debug & 2) {
            } else if (main)
              tma_load_4d(&tmA, &patch_full[pb], smem_b + pb * kHaloPatchBytes, blk * kBlockK, w0 - 1, h0 - 1, img,
                          kEvictNormal);
            else
              tma_load_4d(&tmA2, &patch_full[pb], smem_b + pb * kHaloPatchBytes, (blk - p.cin_blocks) * kBlockK, w0 - 1,
                          h0 - 1, img, kEvictNormal);
            const int ntaps = main ? p.num_taps : 1;                // the 1x1 shortcut operand only feeds the centre tap
            for (int t = 0; t < ntaps; ++t) {
              const int kcol = main ? (t * p.cin_blocks + blk) : (p.num_taps * p.cin_blocks + (blk - p.cin_blocks));
              mbar_wait(&empty_bar[ws], wphase ^ 1);
              mbar_arrive_expect_tx(&full_bar[ws], (p.debug & 4) ? 0u : (uint32_t)S::kABytes);
              if (!(p.debug & 4))
                tma_load_3d(&tmB, &full_bar[ws], smem_a + ws * S::kABytes, kcol * kBlockK, n_blk * kBlockM, 0, kEvictLast);
              if (++ws == kStages) { ws = 0; wphase ^= 1; }
            }
            pb ^= 1;
            if (pb == 0) pphase ^= 1;
          }
        }
      }
    } else
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int tap_blocks = p.num_k_blocks - p.k2_blocks;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_blk = tile % p.n_tiles;
        int rest = tile / p.n_tiles;
        const int m_blk = rest % p.m_tiles;
        const int b = rest / p.m_tiles;
        int img = 0, h0 = 0, w0 = 0;
        if (p.conv) {
          const int tw = m_blk % p.tiles_w;
          const int r2 = m_blk / p.tiles_w;
          const int th = r2 % p.tiles_h;
          img = r2 / p.tiles_h;
          h0 = th * p.bh;
          w0 = tw * p.bw;
        }
        if constexpr (!VEC) {
          mbar_wait(acc_empty, aphase ^ 1);                  // the accumulators of the previous tile left the ring
          aphase ^= 1;
        }
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], ((p.debug & 2) ? 0u : a_bytes) + ((p.debug & 4) ? 0u : b_bytes));
          void* sa = smem_a + stage * S::kABytes;
          void* sb = smem_b + stage * S::kBBytes;
          void* s_act = SWAP ? sb : sa;            // activations: M operand normally, N operand when swapped
          void* s_w = SWAP ? sa : sb;
          constexpr int kActRows = SWAP ? BLOCK_N : kBlockM;
          constexpr int kWRows = SWAP ? kBlockM : BLOCK_N;
          if (!(p.debug & 2)) {
            if (p.conv) {
              if (kb < tap_blocks) {
                const int tap = kb / p.cin_blocks;
                const int cb = kb - tap * p.cin_blocks;
                tma_load_4d(&tmA, &full_bar[stage], s_act, cb * kBlockK, w0 * p.in_stride + p.tap_dx[tap],
                            h0 * p.in_stride + p.tap_dy[tap], img, kEvictNormal);
              } else {
                tma_load_4d(&tmA2, &full_bar[stage], s_act, (kb - tap_blocks) * kBlockK, w0, h0, img,
                            kEvictNormal);
              }
            } else if (p.act_mn) {
#pragma unroll 1
              for (int j = 0; j < kActRows / 64; ++j)
                tma_load_3d(&tmA, &full_bar[stage], (uint8_t*)s_act + j * 8192, m_blk * kActRows + j * 64, kb * kBlockK,
                            p.a_batched ? b : 0, kEvictNormal);
            } else {
              tma_load_3d(&tmA, &full_bar[stage], s_act, kb * kBlockK, m_blk * kActRows, p.a_batched ? b : 0,
                          kEvictNormal);
            }
          }
          if (!(p.debug & 4)) {
            if (p.w_mn) {
#pragma unroll 1
              for (int j = 0; j < kWRows / 64; ++j)
                tma_load_3d(&tmB, &full_bar[stage], (uint8_t*)s_w + j * 8192, n_blk * kWRows + j * 64, kb * kBlockK,
                            p.b_batched ? b : 0, kEvictLast);
            } else {
              tma_load_3d(&tmB, &full_bar[stage], s_w, kb * kBlockK, n_blk * kWRows, p.b_batched ? b : 0,
                          kEvictLast);
            }
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ======================================================================= MMA + epilogue warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int wg = warp >> 2;                        // MMA rows 64 wg .. 64 wg + 63 of the 128-row tile
    int stage = 0, ws = 0, pb = 0;
    uint32_t phase = 0, wphase = 0, pphase = 0;
    // Main loop of this CTA's next tile; returns with this warpgroup's fp32 accumulators in d (layout in wgmma.cuh).
    // One k-block of MMAs stays in flight: a ring slot is released once the MMAs after it have been issued.
    auto mma_main = [&](float (&d)[BLOCK_N / 2]) {
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) d[i] = 0.f;
      if constexpr (HALO) {
        const uint32_t a_base = smem_u32(smem_a) + wg * 8192, patch_base = smem_u32(smem_b);
        // One MMA per (tap, k-step): its N = halo_n accumulator columns are halo_n CONSECUTIVE patch pixels starting
        // at (dy, dx), i.e. bh output rows of bw pixels with the two halo pixels of every patch row riding along as dead
        // columns (masked in the epilogue).  N stays large: the weight slice is fetched once per 128-256 columns.
        const int pitch = p.bw + 2;
        int prev_ws = -1, prev_pb = -1;
        for (int blk = 0; blk < p.cin_blocks + p.k2_blocks; ++blk) {
          const bool main = blk < p.cin_blocks;
          mbar_wait(&patch_full[pb], pphase);
          const uint32_t pbase = patch_base + pb * kHaloPatchBytes;
          const int ntaps = main ? p.num_taps : 1;
          for (int t = 0; t < ntaps; ++t) {
            // patch offsets (0..2) of tap t: any tap set inside the 3x3 neighbourhood, in any order (forward convs,
            // flipped-tap data gradients, the 2x2 phases of nearest-2x + conv)
            const int dy = main ? p.tap_dy[t] + 1 : 1, dx = main ? p.tap_dx[t] + 1 : 1;
            mbar_wait(&full_bar[ws], wphase);
            const uint64_t adesc = make_desc_sw128(a_base + ws * S::kABytes, 16, 1024);
            // B rows = patch pixels (dy * pitch + dx) ...: a 128-byte-granular start inside the SWIZZLE_128B tile
            const uint64_t bdesc = make_desc_sw128(pbase + (uint32_t)((dy * pitch + dx) * 128), 16, 1024);
            wgmma_fence_operands<BLOCK_N / 2>(d);
            wgmma_fence();
            if (!(p.debug & 8)) {
#pragma unroll
              for (int k = 0; k < kBlockK / kMmaK; ++k)
                wgmma_halo(d, adesc + 2 * k, bdesc + 2 * k, (blk | t | k) != 0, p.halo_n);
            }
            wgmma_commit();
            wgmma_fence_operands<BLOCK_N / 2>(d);
            wgmma_wait<1>();
            if (prev_ws >= 0) mbar_arrive(&empty_bar[prev_ws]);
            if (prev_pb >= 0) mbar_arrive(&patch_empty[prev_pb]);
            prev_ws = ws;
            prev_pb = t == ntaps - 1 ? pb : -1;
            if (++ws == kStages) { ws = 0; wphase ^= 1; }
          }
          pb ^= 1;
          if (pb == 0) pphase ^= 1;
        }
        wgmma_wait<0>();
        wgmma_fence_operands<BLOCK_N / 2>(d);
        mbar_arrive(&empty_bar[prev_ws]);
        mbar_arrive(&patch_empty[prev_pb]);
      } else {
        const uint32_t a_base = smem_u32(smem_a) + wg * 8192, b_base = smem_u32(smem_b);
        // MMA operand A = weights when SWAP, activations otherwise; either may be MN-major (stored [K][rows])
        const bool a_mn = SWAP ? (p.w_mn != 0) : (p.act_mn != 0);
        const bool b_mn = SWAP ? (p.act_mn != 0) : (p.w_mn != 0);
        int prev = -1;
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          // K-major: rows of 128 B, k-step = +32 B inside the swizzle row.  MN-major: [k-row][64 rows] atoms 8192 B apart
          // (LBO), 8-k-row groups 1024 B apart (SBO), k-step = 16 k-rows = +2048 B.  Either way the 64-row half of this
          // warpgroup starts 8192 B into the A tile.
          const uint64_t adesc = make_desc_sw128(a_base + stage * S::kABytes, a_mn ? 8192 : 16, 1024);
          const uint64_t bdesc = make_desc_sw128(b_base + stage * S::kBBytes, b_mn ? 8192 : 16, 1024);
          const uint64_t astep = a_mn ? 128 : 2, bstep = b_mn ? 128 : 2;        // in 16-byte units
          wgmma_fence_operands<BLOCK_N / 2>(d);
          wgmma_fence();
          if (!(p.debug & 8)) {
#pragma unroll
            for (int k = 0; k < kBlockK / kMmaK; ++k)
              wgmma_tile<BLOCK_N>(d, adesc + astep * k, bdesc + bstep * k, (kb | k) != 0, a_mn, b_mn);
          }
          wgmma_commit();
          wgmma_fence_operands<BLOCK_N / 2>(d);
          wgmma_wait<1>();
          if (prev >= 0) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_operands<BLOCK_N / 2>(d);
        mbar_arrive(&empty_bar[prev]);
      }
    };
    // Main loop of this CTA's next tile; returns with the fp32 accumulators in acc_smem (row-major, kAccPitch).
    auto mma_tile = [&]() {
      float d[BLOCK_N / 2];
      mma_main(d);
      // both warpgroups' MMAs have retired (they read the ring) before it is overwritten with the accumulators
      asm volatile("bar.sync 1, 256;" ::: "memory");
      {
        float* dst = acc_smem + (wg * 64 + (warp & 3) * 16 + (lane >> 2)) * S::kAccPitch + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          dst[8 * j] = d[4 * j];
          dst[8 * j + 1] = d[4 * j + 1];
          dst[8 * S::kAccPitch + 8 * j] = d[4 * j + 2];
          dst[8 * S::kAccPitch + 8 * j + 1] = d[4 * j + 3];
        }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
    };
    // this thread's reads of the staged accumulators are done: the ring may take the next tile's TMA loads
    auto release_acc = [&]() {
      fence_proxy_async_smem();
      mbar_arrive(acc_empty);
    };
    // Each thread reads one staged accumulator ROW (32 consecutive columns per chunk).  Writing that
    // straight to global memory touches 32 different 128-byte lines per store instruction, so every
    // 32x32 chunk is transposed through a padded smem tile first: afterwards lane = column, and each
    // residual load / output store of a row segment is one fully coalesced 128-byte (fp32) access.
    const int quad = warp & 3;                       // row quadrant of the tile
    const int row_in_tile = quad * 32 + lane;
    const int eg = warp >> 2;                        // epilogue group: which half of the chunks
    const int ew = warp;                             // epilogue warp index 0..7
    const float* t_row = acc_smem + row_in_tile * S::kAccPitch;
    if constexpr (SWAP) {
      // ------------------------------------------------------------------ swapped: lane = channel
      OutT* __restrict__ out = reinterpret_cast<OutT*>(p.out);
      const OutT* __restrict__ res = reinterpret_cast<const OutT*>(p.residual);
      const float* __restrict__ bias = p.bias;
      uint32_t* tab = reinterpret_cast<uint32_t*>(stage_smem);     // [2 acc][out|res][BLOCK_N] pixel offsets
      const int et = threadIdx.x;                                  // 0..255 within the epilogue warps
      int acc = 0;                                                 // which of the two pixel-offset tables
      // Fused GroupNorm statistics of the vectorised path: per-lane shifted partial sums of this lane's four channels,
      // carried ACROSS the tiles this persistent CTA processes for the same (image, channel tile) and merged into the
      // global fp64 accumulators only when that key changes.  One atomic per tile and channel — tens of thousands of
      // tiles hammering the same 2 x Cout addresses of an image — serialise on those addresses; a CTA sees many
      // consecutive tiles of an image, so carrying the sums divides the atomics by that count.
      float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
      int scnt = 0;
      long long skey = -1;                                         // (image * N + first channel) the sums belong to
      auto flush_stats = [&]() {
        // plain sums in fp64 (each lane has its own shift), folded over the eight lanes that share a channel quad
        // (lane & 3 = quad, see the vectorised epilogue below)
        double d1[4], d2[4];
        const double n = (double)scnt;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double shd = (double)sh[k], a = (double)s1[k];
          d1[k] = a + n * shd;
          d2[k] = (double)s2[k] + 2.0 * shd * a + n * shd * shd;
#pragma unroll
          for (int m = 4; m < 32; m <<= 1) {
            d1[k] += __shfl_xor_sync(0xffffffffu, d1[k], m);
            d2[k] += __shfl_xor_sync(0xffffffffu, d2[k], m);
          }
        }
        if ((lane >> 2) == 0 && skey >= 0) {
          double* dst = p.chan_stats + skey * 2;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            atomicAdd(dst + 2 * k, d1[k]);
            atomicAdd(dst + 2 * k + 1, d2[k]);
          }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) s1[k] = s2[k] = sh[k] = 0.f;
        scnt = 0;
      };
      // Vectorised path: the offsets of a tile's pixels RELATIVE to its first pixel are the same for every tile, so the
      // table is built once per CTA (rebuilding it per tile costs integer divisions and a 256-thread barrier); per tile
      // only a 64-bit base and the (rows, columns) still inside the image change.
      uint32_t* s_rel_out = tab;                                   // [BLOCK_N]
      uint32_t* s_rel_res = tab + BLOCK_N;                         // [BLOCK_N]
      uint32_t* s_dhdw = tab + 2 * BLOCK_N;                        // [BLOCK_N]  (dh << 16 | dw), dh = 0xFFFF: dead column
      if constexpr (VEC) {
        for (int pi = et; pi < BLOCK_N; pi += 32 * kEpiWarps) {
          int dh = 0, dw = pi;
          if (p.conv) {
            dh = pi / p.col_pitch;
            dw = pi - dh * p.col_pitch;
            if (dw >= p.bw || dh >= p.bh) dh = 0xFFFF;
          }
          const long long rel = p.conv ? ((long long)dh * p.out_mul * p.OW + (long long)dw * p.out_mul) : (long long)pi;
          s_rel_out[pi] = dh == 0xFFFF ? 0u : (uint32_t)(rel * p.ldo);
          s_rel_res[pi] = dh == 0xFFFF ? 0u : (uint32_t)(rel * p.ld_res);
          s_dhdw[pi] = ((uint32_t)dh << 16) | (uint32_t)(dw & 0xFFFF);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_blk = tile % p.n_tiles;                        // channel tile
        int rest = tile / p.n_tiles;
        const int m_blk = rest % p.m_tiles;                        // pixel tile
        const int b = rest / p.m_tiles;
        int img = 0, th = 0, tw = 0;
        if (p.conv) {
          tw = m_blk % p.tiles_w;
          const int r2 = m_blk / p.tiles_w;
          th = r2 % p.tiles_h;
          img = r2 / p.tiles_h;
        }
        uint32_t* t_out = tab + acc * (2 * BLOCK_N);
        uint32_t* t_res = t_out + BLOCK_N;
        uint32_t* t_flag = tab + 4 * BLOCK_N + acc * 8;              // per 32-pixel chunk: all rows valid
        if constexpr (!VEC) {
        for (int pi = et; pi < BLOCK_N; pi += 32 * kEpiWarps) {
          bool ok;
          long long orow;
          if (p.conv) {
            const int dh = pi / p.col_pitch;
            const int dw = pi - dh * p.col_pitch;
            const int ho = th * p.bh + dh, wo = tw * p.bw + dw;
            ok = (dh < p.bh) && (dw < p.bw) && (ho < p.Ho) && (wo < p.Wo);
            orow = ((long long)img * p.OH + (ho * p.out_mul + p.out_oy)) * p.OW + (wo * p.out_mul + p.out_ox);
          } else {
            const long long r = (long long)m_blk * BLOCK_N + pi;
            ok = r < p.M;
            orow = r;
          }
          t_out[pi] = ok ? (uint32_t)(orow * p.ldo) : 0xFFFFFFFFu;
          t_res[pi] = (uint32_t)(orow * p.ld_res);
          const unsigned okmask = __ballot_sync(0xffffffffu, ok);   // a warp covers one 32-pixel chunk
          if ((et & 31) == 0) t_flag[pi >> 5] = (okmask == 0xffffffffu);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");             // table visible to the 8 epilogue warps
        }
        const int ch = n_blk * kBlockM + row_in_tile;
        const bool ch_ok = ch < p.N;
        float add = 0.f;
        if (ch_ok) {
          if (bias) add += bias[ch];
          if (p.rowvec) add += p.rowvec[(long long)img * p.ld_rowvec + ch];
        }
        OutT* __restrict__ out_b = out + (long long)b * p.out_batch_stride + ch;
        const OutT* __restrict__ res_b = res ? res + (long long)b * p.res_batch_stride + ch : nullptr;
        __half* __restrict__ out2_b = p.out2 ? p.out2 + (long long)b * p.out_batch_stride + ch : nullptr;
        if (!p.conv && p.chan_stats) img = (int)(((long long)m_blk * BLOCK_N) / p.rows_per_img);
        float st1 = 0.f, st2 = 0.f, st_shift = 0.f;     // sums of (v - shift), (v - shift)^2 over this thread's pixels
        int st_cnt = 0;

        if constexpr (VEC) {
          // ---------------------------------------------------------------- vectorised path (16-byte accesses)
          // Straight from the accumulator registers: warp w holds tile rows (channels) 16 w .. 16 w + 15 for all columns
          // (pixels), lane l two channels of column pairs (wgmma.cuh).  NHWC wants, per pixel, runs of consecutive
          // channels, so each 16 x 32 chunk goes through the warp's [32 pixels][kSwapPitch] smem tile (STS.32 from the
          // fragment, LDS.128 back): afterwards lane (pr, q = lane % 4) owns channels 4q..4q+3 of pixels pr, pr+8, pr+16,
          // pr+24, and each residual load / output store moves 16 bytes (fp32) or 8 bytes (fp16) per lane — eight
          // 64-byte (fp32) or 32-byte (fp16) pixel runs of whole sectors per warp instruction.  pr pairs pixels p and
          // p + 4 in every group of 8 lanes, which keeps the 16-byte loads conflict-free at pitch 20.
          float* stgw = reinterpret_cast<float*>(stage_smem + S::kSwapTabBytes) + warp * (32 * kSwapPitch);
          const int q = lane & 3, pr = (lane >> 3) + 4 * ((lane >> 2) & 1);
          const int chq = n_blk * kBlockM + warp * 16 + 4 * q;          // first of this lane's four channels
          const bool cq_ok = chq < p.N;                                 // N % 4 == 0 on this path
          float add4[4] = {0.f, 0.f, 0.f, 0.f};
          if (cq_ok) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              if (bias) add4[k] += bias[chq + k];
              if (p.rowvec) add4[k] += p.rowvec[(long long)img * p.ld_rowvec + chq + k];
            }
          }
          // first pixel of the tile (64-bit) and how many rows / columns of it are inside the image
          long long pix0;
          int lim_h, lim_w;
          if (p.conv) {
            const int h0 = th * p.bh, w0 = tw * p.bw;
            pix0 = ((long long)img * p.OH + (h0 * p.out_mul + p.out_oy)) * p.OW + (w0 * p.out_mul + p.out_ox);
            lim_h = min(p.bh, p.Ho - h0);
            lim_w = min(p.bw, p.Wo - w0);
          } else {
            pix0 = (long long)m_blk * BLOCK_N;
            lim_h = 1;
            lim_w = (int)min((long long)BLOCK_N, (long long)p.M - pix0);
          }
          OutT* __restrict__ out_q = out + (long long)b * p.out_batch_stride + pix0 * p.ldo + chq;
          const OutT* __restrict__ res_q = res ? res + (long long)b * p.res_batch_stride + pix0 * p.ld_res + chq : nullptr;
          __half* __restrict__ out2_q = p.out2 ? p.out2 + (long long)b * p.out_batch_stride + pix0 * p.ldo + chq : nullptr;
          using Vec = typename std::conditional<std::is_same<OutT, float>::value, float4, uint2>::type;
          if (p.chan_stats) skey = cq_ok ? (long long)img * p.N + chq : -1;   // invalid channel quads keep key -1
          float frag[BLOCK_N / 2];
          mma_main(frag);
          // conv tiles may use fewer than BLOCK_N accumulator columns (bw * bh pixels)
          const int ncols = p.conv ? min(BLOCK_N, (p.col_pitch * p.bh + 31) & ~31) : BLOCK_N;
          if (!(p.debug & 16)) {
            // unrolled over the chunks: every fragment register index is then a compile-time constant (a loop-carried
            // index would move frag to local memory)
#pragma unroll
            for (int c = 0; c < BLOCK_N; c += 32) {
              if (c >= ncols) break;
              uint32_t oo[4];
              Vec rres[4];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const uint32_t dd = s_dhdw[c + 8 * i + pr];
                const bool ok = cq_ok && (int)(dd >> 16) < lim_h && (int)(dd & 0xFFFFu) < lim_w;
                oo[i] = ok ? s_rel_out[c + 8 * i + pr] : 0xFFFFFFFFu;
              }
              if (res_q != nullptr) {                // residual rows first: their latency hides behind the transpose
#pragma unroll
                for (int i = 0; i < 4; ++i)
                  if (oo[i] != 0xFFFFFFFFu) rres[i] = *reinterpret_cast<const Vec*>(res_q + s_rel_res[c + 8 * i + pr]);
              }
              // fragment columns c .. c + 31 (frag[4j .. 4j + 3], j = c / 8 .. c / 8 + 3) into the tile: pixel
              // 8 (j % 4) + 2 (lane % 4) + {0, 1}, channel lane / 4 + {0, 8}
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int j = c / 8 + jj;
                float* dst = stgw + (8 * jj + 2 * (lane & 3)) * kSwapPitch + (lane >> 2);
                dst[0] = frag[4 * j];
                dst[kSwapPitch] = frag[4 * j + 1];
                dst[8] = frag[4 * j + 2];
                dst[kSwapPitch + 8] = frag[4 * j + 3];
              }
              __syncwarp();
              // phase A: accumulator * alpha + bias (+ residual) for the lane's 4 pixels x 4 channels
              float v[4][4];
              auto res4 = [&](int i, float* r4) {          // the residual / multiplicative operand of pixel i as fp32
                if constexpr (std::is_same<OutT, float>::value) {
                  r4[0] = rres[i].x; r4[1] = rres[i].y; r4[2] = rres[i].z; r4[3] = rres[i].w;
                } else {
                  const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&rres[i].x));
                  const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&rres[i].y));
                  r4[0] = f0.x; r4[1] = f0.y; r4[2] = f1.x; r4[3] = f1.y;
                }
              };
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float4 t4 = *reinterpret_cast<const float4*>(stgw + (8 * i + pr) * kSwapPitch + 4 * q);
                v[i][0] = fmaf(t4.x, p.alpha, add4[0]); v[i][1] = fmaf(t4.y, p.alpha, add4[1]);
                v[i][2] = fmaf(t4.z, p.alpha, add4[2]); v[i][3] = fmaf(t4.w, p.alpha, add4[3]);
                if (res_q != nullptr && !p.res_mul && oo[i] != 0xFFFFFFFFu) {
                  float r4[4];
                  res4(i, r4);
#pragma unroll
                  for (int k = 0; k < 4; ++k) v[i][k] += r4[k];
                }
              }
              // phase B: activations, one contiguous block that a plain conv skips with a single branch (SiLU / GELU bodies
              // interleaved into the unrolled pixel loop bloat it with instruction-fetch stalls)
              if (p.act == ACT_SILU) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                  for (int k = 0; k < 4; ++k) v[i][k] = silu_f(v[i][k]);
              } else if (p.act == ACT_GELU) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                  for (int k = 0; k < 4; ++k) v[i][k] = gelu_erf_f(v[i][k]);
              }
              // phase C: multiplicative operand, stores, statistics
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const bool ok = oo[i] != 0xFFFFFFFFu;
                if (res_q != nullptr && p.res_mul && ok) {
                  float r4[4];
                  res4(i, r4);
#pragma unroll
                  for (int k = 0; k < 4; ++k) v[i][k] *= r4[k];
                }
                __half2 h01 = __floats2half2_rn(v[i][0], v[i][1]), h23 = __floats2half2_rn(v[i][2], v[i][3]);
                uint2 hv;
                hv.x = *reinterpret_cast<uint32_t*>(&h01);
                hv.y = *reinterpret_cast<uint32_t*>(&h23);
                if (ok && !(p.debug & 1)) {
                  if constexpr (std::is_same<OutT, float>::value) {
                    *reinterpret_cast<float4*>(out_q + oo[i]) = make_float4(v[i][0], v[i][1], v[i][2], v[i][3]);
                    if (out2_q != nullptr) *reinterpret_cast<uint2*>(out2_q + oo[i]) = hv;
                  } else {
                    *reinterpret_cast<uint2*>(out_q + oo[i]) = hv;
                  }
                }
                if (p.chan_stats && ok) {
                  float w4[4] = {v[i][0], v[i][1], v[i][2], v[i][3]};
                  if constexpr (!std::is_same<OutT, float>::value) {      // statistics of the values as stored
                    const float2 f0 = __half22float2(h01), f1 = __half22float2(h23);
                    w4[0] = f0.x; w4[1] = f0.y; w4[2] = f1.x; w4[3] = f1.y;
                  }
                  if (scnt == 0) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) sh[k] = w4[k];
                  }
#pragma unroll
                  for (int k = 0; k < 4; ++k) {
                    const float d = w4[k] - sh[k];
                    s1[k] += d;
                    s2[k] = fmaf(d, d, s2[k]);
                  }
                  ++scnt;
                }
              }
              __syncwarp();                          // the tile is rewritten by the next chunk
            }
          }
          if (p.chan_stats) {
            // merge the carried sums when this CTA's next tile belongs to another (image, channel tile), or at its last
            // tile (warp-uniform).  Flushing here rather than after the tile loop keeps the whole consumer path inside
            // the setmaxnreg.inc region, where ptxas allocates up to kConsumerRegs.
            const int nt = tile + gridDim.x;
            bool same = false;
            if (nt < total_tiles) {
              const int nn = nt % p.n_tiles, nm = (nt / p.n_tiles) % p.m_tiles;
              const int nimg = p.conv ? nm / p.tiles_w / p.tiles_h : (int)(((long long)nm * BLOCK_N) / p.rows_per_img);
              same = nn == n_blk && nimg == img;
            }
            if (!same && __any_sync(0xffffffffu, scnt > 0)) flush_stats();
          }
          continue;
        }
        mma_tile();
        if (!(p.debug & 16)) {
#pragma unroll 1
          for (int c = eg * 32; c < BLOCK_N; c += 64) {
            uint32_t roff[32];
#pragma unroll
            for (int q4 = 0; q4 < 8; ++q4) {
              const uint4 t4 = reinterpret_cast<const uint4*>(t_out + c)[q4];
              roff[4 * q4] = t4.x; roff[4 * q4 + 1] = t4.y; roff[4 * q4 + 2] = t4.z; roff[4 * q4 + 3] = t4.w;
            }
            OutT rres[32];                 // kept in the storage type: converting right after each load would
            if (res_b != nullptr) {        // serialise the loads
#pragma unroll
              for (int q4 = 0; q4 < 8; ++q4) {
                const uint4 t4 = reinterpret_cast<const uint4*>(t_res + c)[q4];
                const uint32_t o4[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const int j = 4 * q4 + e;
                  rres[j] = (ch_ok && roff[j] != 0xFFFFFFFFu) ? res_b[o4[e]] : (OutT)0.f;
                }
              }
            }
            uint32_t r[32];
            acc_ld(t_row + c, r);
            float vals[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) vals[j] = fmaf(__uint_as_float(r[j]), p.alpha, add);
            if (res_b != nullptr && !p.res_mul) {
#pragma unroll
              for (int j = 0; j < 32; ++j) vals[j] += (float)rres[j];
            }
            if (p.act == ACT_SILU) {
#pragma unroll
              for (int j = 0; j < 32; ++j) vals[j] = silu_f(vals[j]);
            } else if (p.act == ACT_GELU) {
#pragma unroll
              for (int j = 0; j < 32; ++j) vals[j] = gelu_erf_f(vals[j]);
            }
            if (res_b != nullptr && p.res_mul) {
#pragma unroll
              for (int j = 0; j < 32; ++j) vals[j] *= (float)rres[j];
            }
            const bool full = t_flag[c >> 5] != 0 && ch_ok;          // interior chunk: no per-element predicates
            if (!(p.debug & 1)) {
              if (full) {
#pragma unroll
                for (int j = 0; j < 32; ++j) out_b[roff[j]] = (OutT)vals[j];
                if (out2_b != nullptr) {
#pragma unroll
                  for (int j = 0; j < 32; ++j) out2_b[roff[j]] = __float2half_rn(vals[j]);
                }
              } else {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  if (ch_ok && roff[j] != 0xFFFFFFFFu) out_b[roff[j]] = (OutT)vals[j];
                if (out2_b != nullptr) {
#pragma unroll
                  for (int j = 0; j < 32; ++j)
                    if (ch_ok && roff[j] != 0xFFFFFFFFu) out2_b[roff[j]] = __float2half_rn(vals[j]);
                }
              }
            }
            if (p.chan_stats) {
              if (c == eg * 32) st_shift = (float)(OutT)vals[0];      // any finite value near the data works as the shift
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                const bool ok = roff[j] != 0xFFFFFFFFu;
                const float d = ok ? (float)(OutT)vals[j] - st_shift : 0.f;
                st1 += d;
                st2 = fmaf(d, d, st2);
                st_cnt += ok ? 1 : 0;
              }
            }
          }
        }
        if (p.chan_stats && ch_ok && st_cnt) {
          double* dst = p.chan_stats + ((long long)img * p.N + ch) * 2;
          const double sh = (double)st_shift, n = (double)st_cnt, s1 = (double)st1;
          atomicAdd(dst, s1 + n * sh);
          atomicAdd(dst + 1, (double)st2 + 2.0 * sh * s1 + n * sh * sh);
        }
        release_acc();
        acc ^= 1;
      }
    } else {
    float (*stg)[33] = reinterpret_cast<float (*)[33]>(stage_smem + ew * (32 * 33 * 4));
    // per-warp row tables (16-byte aligned): element offsets of each of the warp's 32 rows relative to the
    // batch base (0xFFFFFFFF = row outside the tensor), same for the residual, and the per-row bias
    uint32_t* s_off_out = reinterpret_cast<uint32_t*>(rowmeta_smem + ew * 640);
    uint32_t* s_off_res = s_off_out + 32;
    float* s_bias_r = reinterpret_cast<float*>(s_off_res + 32);
    OutT* __restrict__ out = reinterpret_cast<OutT*>(p.out);
    const OutT* __restrict__ res = reinterpret_cast<const OutT*>(p.residual);
    const float* __restrict__ bias = p.bias;
    constexpr int kOutCols = BLOCK_N;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n_blk = tile % p.n_tiles;
      int rest = tile / p.n_tiles;
      const int m_blk = rest % p.m_tiles;
      const int b = rest / p.m_tiles;
      // ---- this thread's row -> output offsets (published to the warp through smem)
      bool row_ok;
      long long orow;   // linear output row index (pixel index for conv)
      long long opix = 0;
      int img = 0;
      if (p.conv) {
        const int tw = m_blk % p.tiles_w;
        const int r2 = m_blk / p.tiles_w;
        const int th = r2 % p.tiles_h;
        img = r2 / p.tiles_h;
        const int dh = row_in_tile / p.bw;
        const int dw = row_in_tile - dh * p.bw;
        const int ho = th * p.bh + dh, wo = tw * p.bw + dw;
        row_ok = (dh < p.bh) && (ho < p.Ho) && (wo < p.Wo);
        opix = (long long)(ho * p.out_mul + p.out_oy) * p.OW + (wo * p.out_mul + p.out_ox);
        orow = (long long)img * p.OH * p.OW + opix;
      } else {
        const int r = m_blk * kBlockM + row_in_tile;
        row_ok = r < p.M;
        orow = r;
        if (p.chan_stats) img = (m_blk * kBlockM) / p.rows_per_img;
      }
      const float* __restrict__ rv = p.rowvec ? p.rowvec + (long long)img * p.ld_rowvec : nullptr;
      __syncwarp();
      s_off_out[lane] = row_ok ? (uint32_t)(orow * p.ldo) : 0xFFFFFFFFu;
      s_off_res[lane] = (uint32_t)(orow * p.ld_res);
      s_bias_r[lane] = (bias && p.bias_row && row_ok) ? bias[(long long)b * p.bias_bs + orow] : 0.f;
      __syncwarp();
      OutT* __restrict__ out_b = out + (long long)b * p.out_batch_stride;
      const OutT* __restrict__ res_b = res ? res + (long long)b * p.res_batch_stride : nullptr;
      __half* __restrict__ out2_b = p.out2 ? p.out2 + (long long)b * p.out_batch_stride : nullptr;

      mma_tile();

      if (p.debug & 16) {
      } else if (p.out_nchw) {
        if (eg == 0) {
        // tiny Cout (<= 8): thread = pixel, consecutive lanes = consecutive pixels -> already coalesced
        uint32_t r[16];
        acc_ld(t_row, r);
        if (row_ok) {
          const long long plane = (long long)p.OH * p.OW;
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            if (e < p.N) {
              float v = __uint_as_float(r[e]) * p.alpha;
              if (bias) v += bias[e];
              if (rv) v += rv[e];
              if (p.act == ACT_SILU) v = silu_f(v);
              out[((long long)img * p.N + e) * plane + opix] = (OutT)v;
            }
          }
        }
        }
      } else {
        constexpr bool geglu = GEGLU;                               // compile-time: keeps registers < 168
        const int width = geglu ? kOutCols / 2 : kOutCols;          // output columns this tile produces
        const int ncol0 = n_blk * width;
        const int n_out = geglu ? p.N / 2 : p.N;
        // one 32-row x CW-column chunk (CW = 32, or 16 for the tail of an 80/16-wide GEGLU tile)
        auto do_chunk = [&](int c, auto cw_tag) {
          constexpr int CW = decltype(cw_tag)::value;
          const int col = ncol0 + c + lane;
          const bool col_ok = lane < CW && col < n_out;
          // row offsets of this warp's 32 rows: 8 broadcast 16-byte loads
          uint32_t roff[32];
#pragma unroll
          for (int q4 = 0; q4 < 8; ++q4) {
            const uint4 t4 = reinterpret_cast<const uint4*>(s_off_out)[q4];
            roff[4 * q4] = t4.x; roff[4 * q4 + 1] = t4.y; roff[4 * q4 + 2] = t4.z; roff[4 * q4 + 3] = t4.w;
          }
          // residual rows for this chunk: 32 independent coalesced loads in flight per warp, issued
          // before the accumulator load / transpose so their latency is hidden
          OutT rres[geglu ? 1 : 32];
          if constexpr (!geglu) if (res_b != nullptr) {
#pragma unroll
            for (int q4 = 0; q4 < 8; ++q4) {
              const uint4 t4 = reinterpret_cast<const uint4*>(s_off_res)[q4];
              const uint32_t o4[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int rr = 4 * q4 + e;
                rres[rr] = (col_ok && roff[rr] != 0xFFFFFFFFu) ? res_b[o4[e] + col] : (OutT)0.f;
              }
            }
          }
          uint32_t r[CW];
          acc_ld(t_row + c, r);
          float gact[geglu ? 32 : 1];
          if constexpr (geglu) {
            // gate half first: transpose it, add its bias and apply erf-GELU with lane = column (batched,
            // branch-free); the value half then goes through the normal transposed path below
            uint32_t g[CW];
            acc_ld(t_row + width + c, g);
#pragma unroll
            for (int e = 0; e < CW; ++e) stg[lane][e] = __uint_as_float(g[e]);
            __syncwarp();
            const float bg = (lane < CW) ? bias[n_blk * kOutCols + width + c + lane] : 0.f;
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) gact[rr] = gelu_erf_f(stg[rr][lane] + bg);
            __syncwarp();
          }
#pragma unroll
          for (int e = 0; e < CW; ++e) stg[lane][e] = __uint_as_float(r[e]);
          __syncwarp();
          // ---- transposed phase: lane = column; all smem reads first, then branch-free math + predicated stores
          float vals[32];
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) vals[rr] = stg[rr][lane];
          if constexpr (geglu) {
            const float bv = (lane < CW) ? bias[n_blk * kOutCols + c + lane] : 0.f;
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) vals[rr] = (vals[rr] + bv) * gact[rr];
          } else {
            float add = 0.f;
            if (col_ok) {
              if (bias && !p.bias_row) add += bias[col];
              if (rv) add += rv[col];
            }
            if (p.bias_row) {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) vals[rr] = fmaf(vals[rr], p.alpha, add + s_bias_r[rr]);
            } else {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) vals[rr] = fmaf(vals[rr], p.alpha, add);
            }
            if (res_b != nullptr && !p.res_mul) {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) vals[rr] += (float)rres[rr];
            }
            if (p.act == ACT_SILU) {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) vals[rr] = silu_f(vals[rr]);
            } else if (p.act == ACT_GELU) {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) vals[rr] = gelu_erf_f(vals[rr]);
            } else if (p.act == ACT_EXP2) {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) vals[rr] = exp2f(vals[rr]);
            }
            if (res_b != nullptr && p.res_mul) {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) vals[rr] *= (float)rres[rr];
            }
          }
          if (!(p.debug & 1)) {
#pragma unroll
            for (int rr = 0; rr < 32; ++rr)
              if (col_ok && roff[rr] != 0xFFFFFFFFu) out_b[roff[rr] + col] = (OutT)vals[rr];
            if (out2_b != nullptr) {
#pragma unroll
              for (int rr = 0; rr < 32; ++rr)
                if (col_ok && roff[rr] != 0xFFFFFFFFu) out2_b[roff[rr] + col] = __float2half_rn(vals[rr]);
            }
          }
          if (p.chan_stats) {
            float st1 = 0.f, st2 = 0.f;
            int st_cnt = 0;
            const float st_shift = (float)(OutT)vals[0];
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) {
              const bool ok = roff[rr] != 0xFFFFFFFFu;
              const float d = ok ? (float)(OutT)vals[rr] - st_shift : 0.f;
              st1 += d;
              st2 = fmaf(d, d, st2);
              st_cnt += ok ? 1 : 0;
            }
            if (col_ok && st_cnt) {
              double* dst = p.chan_stats + ((long long)img * n_out + col) * 2;
              const double sh = (double)st_shift, n = (double)st_cnt, s1 = (double)st1;
              atomicAdd(dst, s1 + n * sh);
              atomicAdd(dst + 1, (double)st2 + 2.0 * sh * s1 + n * sh * sh);
            }
          }
          __syncwarp();
        };
#pragma unroll 1
        for (int c = eg * 32; c < width; c += 64) {
          if (c + 32 <= width) do_chunk(c, std::integral_constant<int, 32>{});
          else do_chunk(c, std::integral_constant<int, 16>{});
        }
      }
      release_acc();
    }
    }  // !SWAP
  }
}

}  // namespace b200
