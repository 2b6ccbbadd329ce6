// Host side of the wgmma GEMM / implicit-GEMM conv: tensor-map construction, tile-shape
// selection, launch.  C-ABI entry points are declared in include/b200_e2eft.h.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "gemm_conv.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

static thread_local char g_err[512] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int encode_tmap(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides,
                CUtensorMapDataType dtype) {
  EncodeTiledFn fn = get_encode();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return -2;
  }
  cuuint64_t d[5], s[4];
  cuuint32_t b[5], e[5];
  for (int i = 0; i < rank; ++i) {
    d[i] = dims[i];
    b[i] = box[i];
    e[i] = elem_strides ? elem_strides[i] : 1;
  }
  for (int i = 0; i < rank - 1; ++i) s[i] = strides_bytes[i];
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(gptr), d, s, b, e,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error(
        "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] strides [%llu %llu %llu] "
        "box [%u %u %u %u] ptr %p",
        (int)r, rank, (unsigned long long)d[0], (unsigned long long)(rank > 1 ? d[1] : 0),
        (unsigned long long)(rank > 2 ? d[2] : 0), (unsigned long long)(rank > 3 ? d[3] : 0),
        (unsigned long long)s[0], (unsigned long long)(rank > 2 ? s[1] : 0),
        (unsigned long long)(rank > 3 ? s[2] : 0), b[0], rank > 1 ? b[1] : 0, rank > 2 ? b[2] : 0,
        rank > 3 ? b[3] : 0, gptr);
    return -3;
  }
  return 0;
}

int current_device() {
  int dev = 0;
  return cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < kMaxDevices ? dev : -1;
}

int sm_count() {
  static int n[kMaxDevices] = {0};          // immutable once written; a racing first call writes the same value
  const int dev = current_device();
  if (dev < 0) return 132;
  if (!n[dev]) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;
  }
  return n[dev];
}

// Debug record of the last gemm_conv_kernel launch (b200_debug_last_launch): which instantiation ran and on which tile
// geometry, so tests can assert the path and tile they mean to cover.  Written by launch_one only; never read on the
// launch path.  Field order: include/b200_e2eft.h.
constexpr int kLastLaunchFields = 16;
static int g_last_launch[kLastLaunchFields] = {0};

// ------------------------------------------------------------------------------------------
template <int BN, typename OutT, bool SWAP, bool GEGLU = false, bool HALO = false, bool VEC = false>
static int launch_one(const CUtensorMap& a, const CUtensorMap& a2, const CUtensorMap& b,
                      const GemmParams& p, cudaStream_t st) {
  using S = GemmSmem<BN, SWAP, HALO>;
  static bool configured_dev[kMaxDevices] = {false};      // the attribute belongs to the (device) context
  const int dev = current_device();
  bool& configured = configured_dev[dev < 0 ? 0 : dev];
  auto kern = gemm_conv_kernel<BN, OutT, SWAP, GEGLU, HALO, VEC>;
  if (!configured || dev < 0) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotalBytes);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(smem=%d): %s", S::kTotalBytes, cudaGetErrorString(e));
      return (int)e;
    }
    configured = true;
  }
  int tiles = p.batch * p.m_tiles * p.n_tiles;
  int grid = tiles < sm_count() ? tiles : sm_count();
  // fused statistics are carried across a CTA's tiles while (image, channel tile) stays the same: with the channel tile
  // fastest in the tile index, a grid that is a multiple of n_tiles keeps every CTA on ONE channel tile
  if (SWAP && p.chan_stats && p.n_tiles > 1 && grid > p.n_tiles) grid -= grid % p.n_tiles;
  {
    const int rec[kLastLaunchFields] = {p.conv, HALO, SWAP, BN, VEC, GEGLU, (int)std::is_same<OutT, float>::value,
                                        p.bw, p.bh, p.halo_n, p.tiles_w, p.tiles_h, p.m_tiles, p.n_tiles, grid,
                                        p.chan_stats != nullptr};
    memcpy(g_last_launch, rec, sizeof(rec));
  }
  kern<<<grid, kGemmThreads, S::kTotalBytes, st>>>(a, a2, b, p);
  B200_CHECK_LAUNCH("gemm_conv_kernel");
  return 0;
}

template <typename OutT>
static int launch_bn(int bn, bool swap, const CUtensorMap& a, const CUtensorMap& a2, const CUtensorMap& b,
                     const GemmParams& p, cudaStream_t st) {
  if (swap) {
    switch (bn) {
      case 64: return p.vec_ok ? launch_one<64, OutT, true, false, false, true>(a, a2, b, p, st)
                               : launch_one<64, OutT, true>(a, a2, b, p, st);
      case 128: return p.vec_ok ? launch_one<128, OutT, true, false, false, true>(a, a2, b, p, st)
                                : launch_one<128, OutT, true>(a, a2, b, p, st);
      case 256: return p.vec_ok ? launch_one<256, OutT, true, false, false, true>(a, a2, b, p, st)
                                : launch_one<256, OutT, true>(a, a2, b, p, st);
    }
  } else if (p.act == ACT_GEGLU) {
    if constexpr (std::is_same<OutT, __half>::value) {
      switch (bn) {
        case 64: return launch_one<64, OutT, false, true>(a, a2, b, p, st);
        case 128: return launch_one<128, OutT, false, true>(a, a2, b, p, st);
        case 160: return launch_one<160, OutT, false, true>(a, a2, b, p, st);
        case 256: return launch_one<256, OutT, false, true>(a, a2, b, p, st);
      }
    }
    set_last_error("GEGLU epilogue needs fp16 output and a tile width in {64,128,160,256} (got %d)", bn);
    return -1;
  } else {
    switch (bn) {
      case 32: return launch_one<32, OutT, false>(a, a2, b, p, st);
      case 64: return launch_one<64, OutT, false>(a, a2, b, p, st);
      case 128: return launch_one<128, OutT, false>(a, a2, b, p, st);
      case 160: return launch_one<160, OutT, false>(a, a2, b, p, st);
      case 256: return launch_one<256, OutT, false>(a, a2, b, p, st);
    }
  }
  set_last_error("unsupported tile width %d (swap=%d)", bn, (int)swap);
  return -1;
}

// Per-k-block time of a 128 x n MMA tile in SM cycles: 4n tensor cycles (K=64 at 2048 dense fp16 FMA per SM and
// cycle), floored by a ~365-cycle producer / consumer barrier round trip per k-block (an estimate, not measured here).
static double kblock_cycles(int n) { return n * 4.0 > 365.0 ? n * 4.0 : 365.0; }
static double tiles_cost(long long tiles, int n) {
  long long waves = (tiles + sm_count() - 1) / sm_count();
  return (double)waves * (kblock_cycles(n) + 40.0);
}

static int g_force_bn = 0;
static int g_debug = 0;
static int g_swap_mode = 1;   // 1 = automatic (swap operands when Cout % 128 == 0), 0 = never
static int g_halo_mode = 1;   // 1 = automatic (halo-resident patch for stride-1 3x3 convs), 0 = never
static int g_last_path = 0;   // 0 = per-tap boxes / GEMM, 1 = halo-resident conv (tests assert the path they mean to cover)

// Tile geometry of the halo-resident conv: bh rows x bw columns of output pixels.  The per-tap MMA covers
// N = round_up64((bw + 2) * bh) consecutive patch pixels (one of the wgmma widths 64 / 128 / 192 / 256), of which bw * bh are real outputs;
// the patch ((bh + 2) rows of bw + 2 pixels, plus the tail the last taps read past it) must fit kHaloMaxPatchPix rows.
static bool pick_halo_tile(int Ho, int Wo, int* bw_out, int* bh_out) {
  double best = 0.0;
  int bbw = 0, bbh = 0;
  for (int bw = 8; bw <= 254 && bw <= Wo; ++bw) {
    for (int bh = 1; bh <= 32 && bh <= Ho; ++bh) {
      const int pitch = bw + 2;
      const int n = (pitch * bh + 63) / 64 * 64;
      if (n > 256) break;
      if ((bh + 2) * pitch + (n - pitch * bh) + 2 > kHaloMaxPatchPix) continue;
      const double ew = (double)Wo / ((double)((Wo + bw - 1) / bw) * bw);
      const double eh = (double)Ho / ((double)((Ho + bh - 1) / bh) * bh);
      double score = ew * eh * (double)(bw * bh) / n;                     // useful fraction of the MMA columns
      score *= 0.9 + 0.1 * n / 256.0;                                     // fewer, fuller tiles
      score *= 1.0 - 0.03 * ((double)(bw + 2) * (bh + 2) / (bw * bh) - 1.0);   // halo traffic
      if (score > best + 1e-9) { best = score; bbw = bw; bbh = bh; }
    }
  }
  *bw_out = bbw; *bh_out = bbh;
  return bbw != 0 && best >= 0.78;
}

}  // namespace b200

using namespace b200;

extern "C" const char* b200_last_error_string(void) { return b200::last_error(); }
extern "C" void b200_debug_force_block_n(int bn) { b200::g_force_bn = bn; }
extern "C" void b200_debug_set_flags(int f) { b200::g_debug = f; }
extern "C" void b200_debug_set_swap(int m) { b200::g_swap_mode = m; }
extern "C" void b200_debug_set_halo(int m) { b200::g_halo_mode = m; }
extern "C" int b200_debug_last_path(void) { return b200::g_last_path; }
extern "C" int b200_debug_last_launch(int* out, int n) {
  if (!out || n <= 0) return kLastLaunchFields;
  const int k = n < kLastLaunchFields ? n : kLastLaunchFields;
  memcpy(out, b200::g_last_launch, k * sizeof(int));
  return kLastLaunchFields;
}
extern "C" int b200_abi_version(void) { return 17; }
// Tile width used by the GEGLU epilogue for a packed width N (= 2 x output width); weights must be
// packed per tile as [value half | gate half] with this width.
extern "C" int b200_geglu_block_n(int N) {
  return (N % 160 == 0) ? 160 : (N % 256 == 0 ? 256 : (N % 128 == 0 ? 128 : (N % 64 == 0 ? 64 : 0)));
}

extern "C" int b200_linear(const void* A, long long lda, long long a_batch_stride, const void* W,
                           long long ldw, long long w_batch_stride, int M, int N, int K, int batch,
                           const float* bias, int bias_row, const void* residual, long long ld_res,
                           long long res_batch_stride, void* out, long long ldo,
                           long long out_batch_stride, int out_f32, int act, float alpha,
                           double* chan_stats, int rows_per_img, void* out2_f16, int res_mul, int a_mn, int w_mn,
                           long long bias_batch_stride, void* stream) {
  B200_CHECK_ARG(A && W && out, "b200_linear: null pointer");
  B200_CHECK_ARG(!(a_mn || w_mn) || act != ACT_GEGLU, "b200_linear: MN-major operands are not combined with GEGLU");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0 && batch > 0, "b200_linear: bad shape M=%d N=%d K=%d batch=%d", M, N, K, batch);
  B200_CHECK_ARG(lda % 8 == 0 && ldw % 8 == 0, "b200_linear: lda/ldw must be multiples of 8 elements (16 B)");
  B200_CHECK_ARG(((uintptr_t)A & 15) == 0 && ((uintptr_t)W & 15) == 0 && ((uintptr_t)out & 15) == 0,
                 "b200_linear: pointers must be 16-byte aligned");
  B200_CHECK_ARG(act != ACT_GEGLU || ldo % 8 == 0, "b200_linear: GEGLU needs ldo %% 8 == 0");
  B200_CHECK_ARG(act != ACT_GEGLU || (N % 16 == 0 && bias), "b200_linear: GEGLU needs bias and N%%16==0");
  B200_CHECK_ARG(batch == 1 || (a_batch_stride % 8 == 0 && (w_batch_stride % 8 == 0)),
                 "b200_linear: batch strides must be multiples of 8 elements");

  B200_CHECK_ARG(!chan_stats || (batch == 1 && rows_per_img > 0 && rows_per_img % 64 == 0 && M % rows_per_img == 0 &&
                                 act != ACT_GEGLU && !bias_row),
                 "b200_linear: chan_stats needs batch=1, rows_per_img %% 64 == 0, M %% rows_per_img == 0");
  B200_CHECK_ARG((long long)M * ldo < 0xFFFFFFFFll && (long long)M * (ld_res > 0 ? ld_res : 1) < 0xFFFFFFFFll,
                 "b200_linear: per-batch output larger than 2^32 elements");
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N;
  p.num_k_blocks = (K + kBlockK - 1) / kBlockK;
  p.batch = batch;
  p.m_tiles = (M + kBlockM - 1) / kBlockM;
  p.a_batched = (a_batch_stride != 0 && batch > 1);
  p.b_batched = (w_batch_stride != 0 && batch > 1);
  // tile shape: normal (rows = 128 pixels, bn channels) vs swapped (rows = 128 channels, bn pixels)
  const bool can_swap = g_swap_mode && N >= 128 && act != ACT_GEGLU && !bias_row;
  bool swap = false;
  int bn = 0;
  double best = 1e30;
  if (act == ACT_GEGLU) {
    bn = b200_geglu_block_n(N);
    B200_CHECK_ARG(bn != 0, "b200_linear: GEGLU N=%d not tileable", N);
  } else {
    const int nc[5] = {256, 160, 128, 64, 32};
    const bool normal_ok = !chan_stats || rows_per_img % kBlockM == 0;   // stats: a row tile stays inside one image
    for (int i = 0; i < 5 && normal_ok; ++i) {
      if (g_force_bn && nc[i] != g_force_bn) continue;
      if (w_mn && nc[i] % 64 != 0) continue;                              // MN-major tiles are built from 64-row atoms
      double c = tiles_cost((long long)p.m_tiles * batch * ((N + nc[i] - 1) / nc[i]), nc[i]);
      if (c < best - 1e-9) { best = c; bn = nc[i]; swap = false; }
    }
    if (can_swap || (chan_stats && !normal_ok && N >= 128)) {
      const int pc[3] = {256, 128, 64};
      for (int i = 0; i < 3; ++i) {
        if (g_force_bn && pc[i] != g_force_bn) continue;
        if (chan_stats && rows_per_img % pc[i] != 0) continue;
        if (a_mn && pc[i] % 64 != 0) continue;
        double c = tiles_cost((long long)batch * ((M + pc[i] - 1) / pc[i]) * ((N + 127) / 128), pc[i]) * 0.85;  // cheaper epilogue, fewer barrier round trips
        if (c < best - 1e-9) { best = c; bn = pc[i]; swap = true; }
      }
    }
    B200_CHECK_ARG(bn != 0, "b200_linear: no tile shape for N=%d (forced %d)", N, g_force_bn);
  }
  if (swap) {
    p.m_tiles = (M + bn - 1) / bn;
    p.n_tiles = (N + 127) / 128;
  } else {
    p.n_tiles = (N + bn - 1) / bn;
  }
  p.out = out; p.ldo = ldo; p.out_batch_stride = out_batch_stride; p.out_f32 = out_f32;
  p.bias = bias; p.bias_row = bias_row;
  p.residual = residual; p.ld_res = ld_res; p.res_batch_stride = res_batch_stride; p.res_mul = res_mul;
  p.act = act; p.alpha = alpha; p.debug = g_debug;
  p.chan_stats = chan_stats; p.rows_per_img = rows_per_img; p.out2 = (__half*)out2_f16;
  p.act_mn = a_mn; p.w_mn = w_mn;
  p.bias_bs = bias_batch_stride;
  p.out_mul = 1;
  // swapped epilogue: 16-byte (fp32) / 8-byte (fp16) accesses over runs of 4 channels
  {
    const uintptr_t omask = out_f32 ? 15 : 7;
    // linear layers: the transposing epilogue only pays off where it carries the fused statistics across tiles; for the
    // small-K GEMMs of the transformer blocks the direct lane = channel stores are cheaper
    p.vec_ok = swap && (chan_stats != nullptr || (g_debug & 128)) && !(g_debug & 64) && N % 4 == 0 && ldo % 4 == 0 &&
               out_batch_stride % 4 == 0 && ((uintptr_t)out & omask) == 0 &&
               (!residual || (ld_res % 4 == 0 && res_batch_stride % 4 == 0 && ((uintptr_t)residual & omask) == 0)) &&
               (!out2_f16 || ((uintptr_t)out2_f16 & 7) == 0);
  }

  CUtensorMap ta, tb;
  if (a_mn) {                 // A stored [K][M]: innermost dimension = rows (M), boxes of 64 rows x 64 k
    uint64_t dims[3] = {(uint64_t)M, (uint64_t)K, (uint64_t)(p.a_batched ? batch : 1)};
    uint64_t str[2] = {(uint64_t)lda * 2, (uint64_t)(p.a_batched ? a_batch_stride : (long long)K * lda) * 2};
    uint32_t box[3] = {64, kBlockK, 1};
    int r = encode_tmap(&ta, A, 3, dims, str, box, nullptr);
    if (r) return r;
  } else {
    uint64_t dims[3] = {(uint64_t)K, (uint64_t)M, (uint64_t)(p.a_batched ? batch : 1)};
    uint64_t str[2] = {(uint64_t)lda * 2, (uint64_t)(p.a_batched ? a_batch_stride : (long long)M * lda) * 2};
    uint32_t box[3] = {kBlockK, (uint32_t)(swap ? bn : kBlockM), 1};
    int r = encode_tmap(&ta, A, 3, dims, str, box, nullptr);
    if (r) return r;
  }
  if (w_mn) {                 // W stored [K][N]
    uint64_t dims[3] = {(uint64_t)N, (uint64_t)K, (uint64_t)(p.b_batched ? batch : 1)};
    uint64_t str[2] = {(uint64_t)ldw * 2, (uint64_t)(p.b_batched ? w_batch_stride : (long long)K * ldw) * 2};
    uint32_t box[3] = {64, kBlockK, 1};
    int r = encode_tmap(&tb, W, 3, dims, str, box, nullptr);
    if (r) return r;
  } else {
    uint64_t dims[3] = {(uint64_t)K, (uint64_t)N, (uint64_t)(p.b_batched ? batch : 1)};
    uint64_t str[2] = {(uint64_t)ldw * 2, (uint64_t)(p.b_batched ? w_batch_stride : (long long)N * ldw) * 2};
    uint32_t box[3] = {kBlockK, (uint32_t)(swap ? kBlockM : bn), 1};
    int r = encode_tmap(&tb, W, 3, dims, str, box, nullptr);
    if (r) return r;
  }
  cudaStream_t st = (cudaStream_t)stream;
  return out_f32 ? launch_bn<float>(bn, swap, ta, ta, tb, p, st) : launch_bn<__half>(bn, swap, ta, ta, tb, p, st);
}

// Choose the (bw, bh) output-pixel patch of an M tile: bw*bh <= 128, maximise useful rows.
static double pick_patch(int Ho, int Wo, int stride, int target, int* bw_out, int* bh_out) {
  double best = -1;
  int bbw = 1, bbh = 1;
  for (int bw = 1; bw <= target && bw <= Wo; ++bw) {
    if (bw * stride > 256) break;
    int bh = target / bw;
    if (bh > Ho) bh = Ho;
    if (bh * stride > 256) bh = 256 / stride;
    if (bh < 1) continue;
    long long tw = (Wo + bw - 1) / bw, th = (Ho + bh - 1) / bh;
    double eff = (double)Ho * Wo / (double)(tw * th * target);
    // prefer wider rows on ties (longer contiguous TMA rows / stores)
    if (eff > best + 1e-9 || (eff > best - 1e-9 && bw > bbw)) {
      best = eff; bbw = bw; bbh = bh;
    }
  }
  *bw_out = bbw; *bh_out = bbh;
  return best;
}

extern "C" int b200_conv2d_nhwc(const void* X, int NB, int H, int W, int Cin, const void* X2, int C2,
                                const void* Wp, int Cout, int num_taps, const int* tap_dy,
                                const int* tap_dx, int stride, int Ho, int Wo, int out_mul, int out_oy,
                                int out_ox, const float* bias, const float* rowvec,
                                long long ld_rowvec, const void* residual, void* out, int out_f32,
                                int out_nchw, int act, double* chan_stats, void* out2_f16, void* stream) {
  B200_CHECK_ARG(X && Wp && out, "b200_conv2d_nhwc: null pointer");
  B200_CHECK_ARG(Cin % 64 == 0, "b200_conv2d_nhwc: Cin=%d must be a multiple of 64 (use im2col path)", Cin);
  B200_CHECK_ARG(C2 % 64 == 0, "b200_conv2d_nhwc: C2=%d must be a multiple of 64", C2);
  B200_CHECK_ARG(num_taps >= 1 && num_taps <= kMaxTaps, "b200_conv2d_nhwc: num_taps=%d", num_taps);
  B200_CHECK_ARG(stride >= 1 && stride <= 2 && out_mul >= 1, "b200_conv2d_nhwc: stride=%d out_mul=%d", stride, out_mul);
  B200_CHECK_ARG(NB > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && Cout > 0, "b200_conv2d_nhwc: bad shape");
  B200_CHECK_ARG(((uintptr_t)X & 15) == 0 && ((uintptr_t)Wp & 15) == 0 && ((uintptr_t)out & 15) == 0,
                 "b200_conv2d_nhwc: pointers must be 16-byte aligned");
  B200_CHECK_ARG(act != ACT_GEGLU, "b200_conv2d_nhwc: GEGLU epilogue is linear-only");
  B200_CHECK_ARG(!out_nchw || (!residual && Cout <= 8), "b200_conv2d_nhwc: out_nchw needs Cout <= 8 and no residual");

  B200_CHECK_ARG((long long)NB * Ho * out_mul * Wo * out_mul * Cout < 0xFFFFFFFFll,
                 "b200_conv2d_nhwc: output larger than 2^32 elements");
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.conv = 1;
  p.N = Cout;
  p.batch = 1;
  p.Ho = Ho; p.Wo = Wo;
  const bool can_swap = g_swap_mode && Cout >= 128 && !out_nchw;
  // ---- halo-resident path: stride-1 "same" 3x3 convs in the swapped orientation
  {
    bool taps_ok = stride == 1 && Ho == H && Wo == W && !(X2 && out_mul != 1);
    for (int i = 0; i < num_taps && taps_ok; ++i)
      taps_ok = tap_dy[i] >= -1 && tap_dy[i] <= 1 && tap_dx[i] >= -1 && tap_dx[i] <= 1;
    int hbw = 0, hbh = 0;
    // epilogue-bound launches (fp32 output + fp32 residual over a short K = 9 * Cin <= 1152: 8 B read + 4-6 B written per
    // output element against ~1 us of MMA per tile) gain nothing from cheaper operand loads and lose ~10 % to the dead
    // halo columns their epilogue still walks
    const bool epi_bound = out_f32 && residual && num_taps * Cin <= 1152 && !X2;
    const bool halo_vec = !(g_debug & 64) && (Cout % 4 == 0) && (!residual || ((uintptr_t)residual & 15) == 0) &&
                          (!out2_f16 || ((uintptr_t)out2_f16 & 7) == 0);      // the halo kernel has the vectorised epilogue only
    if (can_swap && g_halo_mode && taps_ok && !g_force_bn && halo_vec && (!epi_bound || g_halo_mode == 2) &&
        pick_halo_tile(Ho, Wo, &hbw, &hbh)) {
      p.bw = hbw; p.bh = hbh;
      p.col_pitch = hbw + 2;
      p.halo_n = ((hbw + 2) * hbh + 63) / 64 * 64;
      p.tiles_w = (Wo + hbw - 1) / hbw;
      p.tiles_h = (Ho + hbh - 1) / hbh;
      p.m_tiles = NB * p.tiles_w * p.tiles_h;
      p.n_tiles = (Cout + 127) / 128;
      p.M = NB * Ho * Wo;
      p.cin_blocks = Cin / 64;
      p.num_taps = num_taps;
      for (int i = 0; i < num_taps; ++i) { p.tap_dy[i] = tap_dy[i]; p.tap_dx[i] = tap_dx[i]; }
      p.in_stride = 1;
      p.k2_blocks = X2 ? C2 / 64 : 0;
      p.num_k_blocks = num_taps * p.cin_blocks + p.k2_blocks;
      p.out_mul = out_mul; p.out_oy = out_oy; p.out_ox = out_ox; p.OH = Ho * out_mul; p.OW = Wo * out_mul;
      p.out = out; p.ldo = Cout; p.out_f32 = out_f32; p.out_nchw = 0;
      p.bias = bias; p.rowvec = rowvec; p.ld_rowvec = ld_rowvec;
      p.residual = residual; p.ld_res = Cout;
      p.act = act; p.alpha = 1.0f; p.debug = g_debug;
      p.chan_stats = chan_stats; p.out2 = (__half*)out2_f16;
      p.vec_ok = 1;
      CUtensorMap ta, ta2, tb;
      {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
        uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        uint32_t box[4] = {kBlockK, (uint32_t)(hbw + 2), (uint32_t)(hbh + 2), 1};
        int r = encode_tmap(&ta, X, 4, dims, str, box, nullptr);
        if (r) return r;
      }
      ta2 = ta;
      if (X2) {
        uint64_t dims[4] = {(uint64_t)C2, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)NB};
        uint64_t str[3] = {(uint64_t)C2 * 2, (uint64_t)Wo * C2 * 2, (uint64_t)Ho * Wo * C2 * 2};
        uint32_t box[4] = {kBlockK, (uint32_t)(hbw + 2), (uint32_t)(hbh + 2), 1};
        int r = encode_tmap(&ta2, X2, 4, dims, str, box, nullptr);
        if (r) return r;
      }
      {
        const long long Kt = (long long)num_taps * Cin + (X2 ? C2 : 0);
        uint64_t dims[3] = {(uint64_t)Kt, (uint64_t)Cout, 1};
        uint64_t str[2] = {(uint64_t)Kt * 2, (uint64_t)Kt * Cout * 2};
        uint32_t box[3] = {kBlockK, (uint32_t)kBlockM, 1};
        int r = encode_tmap(&tb, Wp, 3, dims, str, box, nullptr);
        if (r) return r;
      }
      cudaStream_t st = (cudaStream_t)stream;
      g_last_path = 1;
      return out_f32 ? launch_one<256, float, true, false, true, true>(ta, ta2, tb, p, st)
                     : launch_one<256, __half, true, false, true, true>(ta, ta2, tb, p, st);
    }
  }
  g_last_path = 0;
  bool swap = false;
  int pix = 128, bn_norm = 0;
  {
    double best = 1e30;
    int bw, bh;
    pick_patch(Ho, Wo, stride, 128, &bw, &bh);
    const long long mt = (long long)NB * ((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh);
    const int nc[5] = {256, 160, 128, 64, 32};
    for (int i = 0; i < 5; ++i) {
      if (g_force_bn && nc[i] != g_force_bn) continue;
      double c = tiles_cost(mt * ((Cout + nc[i] - 1) / nc[i]), nc[i]);
      if (c < best - 1e-9) { best = c; bn_norm = nc[i]; swap = false; }
    }
    if (can_swap) {
      const int pc[3] = {256, 128, 64};
      for (int i = 0; i < 3; ++i) {
        if (g_force_bn && pc[i] != g_force_bn) continue;
        pick_patch(Ho, Wo, stride, pc[i], &bw, &bh);
        long long tiles = (long long)NB * ((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh) * ((Cout + 127) / 128);
        double c = tiles_cost(tiles, pc[i]) * 0.85;   // swapped tiles: cheaper epilogue, fewer barrier round trips
        if (c < best - 1e-9) { best = c; pix = pc[i]; swap = true; }
      }
    }
    if (!swap) pix = 128;
    B200_CHECK_ARG(swap || bn_norm != 0, "b200_conv2d_nhwc: no tile shape (forced %d)", g_force_bn);
  }
  pick_patch(Ho, Wo, stride, pix, &p.bw, &p.bh);
  p.col_pitch = p.bw;
  p.tiles_w = (Wo + p.bw - 1) / p.bw;
  p.tiles_h = (Ho + p.bh - 1) / p.bh;
  p.m_tiles = NB * p.tiles_w * p.tiles_h;
  p.M = NB * Ho * Wo;
  p.cin_blocks = Cin / 64;
  p.num_taps = num_taps;
  p.in_stride = stride;
  for (int i = 0; i < num_taps; ++i) { p.tap_dy[i] = tap_dy[i]; p.tap_dx[i] = tap_dx[i]; }
  p.k2_blocks = X2 ? C2 / 64 : 0;
  p.num_k_blocks = num_taps * p.cin_blocks + p.k2_blocks;
  p.out_mul = out_mul; p.out_oy = out_oy; p.out_ox = out_ox;
  p.OH = Ho * out_mul; p.OW = Wo * out_mul;
  int bn;
  if (swap) {
    bn = pix;
    p.n_tiles = (Cout + 127) / 128;
  } else {
    bn = bn_norm;
    p.n_tiles = (Cout + bn - 1) / bn;
  }
  p.out = out; p.ldo = Cout; p.out_f32 = out_f32; p.out_nchw = out_nchw;
  p.bias = bias; p.rowvec = rowvec; p.ld_rowvec = ld_rowvec;
  p.residual = residual; p.ld_res = Cout;
  p.act = act; p.alpha = 1.0f; p.debug = g_debug;
  p.chan_stats = out_nchw ? nullptr : chan_stats;
  p.out2 = out_nchw ? nullptr : (__half*)out2_f16;
  p.vec_ok = swap && !(g_debug & 64) && (Cout % 4 == 0) && (!residual || ((uintptr_t)residual & 15) == 0) &&
             (!out2_f16 || ((uintptr_t)out2_f16 & 7) == 0);

  CUtensorMap ta, ta2, tb;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
    uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
    uint32_t box[4] = {kBlockK, (uint32_t)(p.bw * stride), (uint32_t)(p.bh * stride), 1};
    uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
    int r = encode_tmap(&ta, X, 4, dims, str, box, es);
    if (r) return r;
  }
  ta2 = ta;
  if (X2) {
    uint64_t dims[4] = {(uint64_t)C2, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)NB};
    uint64_t str[3] = {(uint64_t)C2 * 2, (uint64_t)Wo * C2 * 2, (uint64_t)Ho * Wo * C2 * 2};
    uint32_t box[4] = {kBlockK, (uint32_t)p.bw, (uint32_t)p.bh, 1};
    int r = encode_tmap(&ta2, X2, 4, dims, str, box, nullptr);
    if (r) return r;
  }
  {
    const long long Kt = (long long)num_taps * Cin + (X2 ? C2 : 0);
    uint64_t dims[3] = {(uint64_t)Kt, (uint64_t)Cout, 1};
    uint64_t str[2] = {(uint64_t)Kt * 2, (uint64_t)Kt * Cout * 2};
    uint32_t box[3] = {kBlockK, (uint32_t)(swap ? kBlockM : bn), 1};
    int r = encode_tmap(&tb, Wp, 3, dims, str, box, nullptr);
    if (r) return r;
  }
  cudaStream_t st = (cudaStream_t)stream;
  return out_f32 ? launch_bn<float>(bn, swap, ta, ta2, tb, p, st) : launch_bn<__half>(bn, swap, ta, ta2, tb, p, st);
}
