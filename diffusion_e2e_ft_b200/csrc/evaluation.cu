// Evaluation of depth and normal predictions on the device (DESIGN.md §3 "Evaluation"):
//   b200_eval_align_depth    Marigold/src/util/alignment.py:8-55 as called at Marigold/eval.py:173-203
//   b200_eval_depth_metrics  Marigold/eval.py:173-220 + Marigold/src/util/metric.py (the ten metrics)
//   b200_eval_normal_error   DSINE/utils/utils.py:150-159 + the accumulation of DSINE/projects/dsine/test.py:100-115
//   b200_eval_kth_smallest   np.median of DSINE/utils/utils.py:168 (radix select)
// All HBM-bound reductions.  Every sum is an fp64 partial per block (thread-sequential, then a fixed xor-butterfly
// over the warp, then the warps in index order), written to a workspace slot and combined by a one-thread finalize
// kernel in block order: no floating-point atomics, so two runs on the same inputs give the same bits.  The grids
// depend only on the problem size, never on the device.  Counts and indices are 64-bit.  Nothing syncs the host.
#include <math_constants.h>

#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

constexpr int kEvalThreads = 256;
constexpr int kEvalWarps = kEvalThreads / 32;

// blocks per sample for a pass over `elems` elements: about 4 elements per thread, at most B200_EVAL_MAX_BLOCKS
static int eval_blocks(long long elems) {
  long long g = (elems + 4LL * kEvalThreads - 1) / (4LL * kEvalThreads);
  if (g < 1) g = 1;
  if (g > B200_EVAL_MAX_BLOCKS) g = B200_EVAL_MAX_BLOCKS;
  return (int)g;
}

// Block-wide fixed-order sum of NF per-thread values; thread 0 writes them to dst[0..NF).
template <int NF>
__device__ __forceinline__ void block_sum_store(double (&v)[NF], double* __restrict__ dst) {
  __shared__ double s[kEvalWarps][NF];
#pragma unroll
  for (int f = 0; f < NF; ++f) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[f] += __shfl_xor_sync(0xffffffffu, v[f], o);
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int f = 0; f < NF; ++f) s[warp][f] = v[f];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int f = 0; f < NF; ++f) {
      double t = 0.0;
      for (int w = 0; w < kEvalWarps; ++w) t += s[w][f];
      dst[f] = t;
    }
  }
}

// ------------------------------------------------------------------------------------ least-squares alignment
// Sampled grid: every row, columns j < OW read source column min(floor(float(j) * col_scale), W - 1) -- what
// torch.nn.Upsample(scale_factor=s, mode="nearest") samples from the [1, H, W] tensor alignment.py:26 hands it (a 3-D
// input, so a 1-D interpolation along W with the fp32 source step col_scale = float(1 / s)).
// Per-block partials: n, sum p, sum g, sum p^2, sum p g, min p, max p (the last two detect a rank-deficient system).
constexpr int kAlignFields = 7;

__global__ void eval_align_moments_kernel(const float* __restrict__ gt, const float* __restrict__ pred,
                                          const unsigned char* __restrict__ mask, int H, int W, int OW, float col_scale,
                                          int disparity, double* __restrict__ ws) {
  const int b = blockIdx.y;
  const long long HW = (long long)H * W, total = (long long)H * OW;
  const float* g_ = gt + b * HW;
  const float* p_ = pred + b * HW;
  const unsigned char* m_ = mask + b * HW;
  double v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  float lo = CUDART_INF_F, hi = -CUDART_INF_F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long src = i;
    if (OW != W) {
      const long long r = i / OW, j = i - r * OW;
      long long c = (long long)floorf(__fmul_rn((float)j, col_scale));
      if (c > W - 1) c = W - 1;
      src = r * W + c;
    }
    if (!m_[src]) continue;
    const float p = p_[src];
    float g = g_[src];
    if (disparity) {                                   // eval.py:184-189: target 1/gt, mask & gt > 0 & pred > 0
      if (!(g > 0.f) || !(p > 0.f)) continue;
      g = __fdiv_rn(1.0f, g);
    }
    const double pd = p, gd = g;
    v[0] += 1.0;
    v[1] += pd;
    v[2] += gd;
    v[3] += pd * pd;
    v[4] += pd * gd;
    lo = fminf(lo, p);
    hi = fmaxf(hi, p);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  __shared__ float s_lo[kEvalWarps], s_hi[kEvalWarps];
  if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; }
  double* dst = ws + ((long long)b * gridDim.x + blockIdx.x) * kAlignFields;
  block_sum_store<5>(v, dst);                          // its __syncthreads also publishes s_lo / s_hi
  if (threadIdx.x == 0) {
    for (int w = 0; w < kEvalWarps; ++w) { lo = fminf(lo, s_lo[w]); hi = fmaxf(hi, s_hi[w]); }
    dst[5] = lo;
    dst[6] = hi;
  }
}

// One thread per sample: combine the block partials in block order, then numpy's lstsq on the 2x2 normal equations
// in fp64.  Rank deficient (every sampled p equal): lstsq's minimum-norm solution [p, 1] * mean(g) / (p^2 + 1).
// Empty: 0, 0 (lstsq of a 0 x 2 system).
__global__ void eval_align_solve_kernel(const double* __restrict__ ws, int B, int nblk, float* __restrict__ scale_shift) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  double lo = CUDART_INF, hi = -CUDART_INF;
  for (int k = 0; k < nblk; ++k) {
    const double* p = ws + ((long long)b * nblk + k) * kAlignFields;
#pragma unroll
    for (int f = 0; f < 5; ++f) s[f] += p[f];
    lo = fmin(lo, p[5]);
    hi = fmax(hi, p[6]);
  }
  const double n = s[0];
  double scale = 0.0, shift = 0.0;
  if (n > 0.0) {
    if (lo == hi) {
      const double gm = s[2] / n, den = lo * lo + 1.0;
      scale = lo * gm / den;
      shift = gm / den;
    } else {
      const double det = n * s[3] - s[1] * s[1];
      scale = (n * s[4] - s[1] * s[2]) / det;
      shift = (s[3] * s[2] - s[1] * s[4]) / det;
    }
  }
  scale_shift[2 * b] = (float)scale;
  scale_shift[2 * b + 1] = (float)shift;
}

// ------------------------------------------------------------------------------------ depth metrics
// Per-sample partials: n, sum |d|/g, sum d^2/g, sum d^2, sum dl^2, sum |log10 p - log10 g|, sum dl, delta1..3
// counts, sum (1/p - 1/g)^2, with d = p - g and dl = log p - log g, each per-pixel term in fp32 as metric.py
// computes it.
constexpr int kMetricFields = 11;

__device__ __forceinline__ float clip_lo_hi(float x, float lo, float hi) {    // np.clip: NaN stays NaN
  x = x < lo ? lo : x;
  return x > hi ? hi : x;
}

__global__ void eval_depth_metrics_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                          const unsigned char* __restrict__ mask, long long HW,
                                          const float* __restrict__ scale_shift, int disparity, int clip,
                                          float min_depth, float max_depth, float* __restrict__ aligned,
                                          double* __restrict__ ws) {
  const int b = blockIdx.y;
  float s = 1.f, t = 0.f;
  if (scale_shift) { s = scale_shift[2 * b]; t = scale_shift[2 * b + 1]; }
  double v[kMetricFields];
#pragma unroll
  for (int f = 0; f < kMetricFields; ++f) v[f] = 0.0;
  const long long base = (long long)b * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    float p = pred[base + i];
    if (scale_shift) p = __fadd_rn(__fmul_rn(p, s), t);            // numpy float32 `pred * scale + shift`
    if (disparity) {                                                  // eval.py:199-202
      p = p < 1e-3f ? 1e-3f : p;
      p = p > 0.f ? __fdiv_rn(1.0f, p) : 0.f;
    }
    if (clip) {                                                       // eval.py:205-210
      p = clip_lo_hi(p, min_depth, max_depth);
      p = p < 1e-6f ? 1e-6f : p;
    }
    if (aligned) aligned[base + i] = p;
    if (!ws || (mask && !mask[base + i])) continue;
    const float g = gt[base + i];
    const float d = __fsub_rn(p, g), ad = fabsf(d);
    const float dl = __fsub_rn(logf(p), logf(g));
    const float l10 = fabsf(__fsub_rn(log10f(p), log10f(g)));
    const float r1 = __fdiv_rn(p, g), r2 = __fdiv_rn(g, p);
    const float di = __fsub_rn(__fdiv_rn(1.0f, p), __fdiv_rn(1.0f, g));
    v[0] += 1.0;
    v[1] += (double)__fdiv_rn(ad, g);
    v[2] += (double)__fdiv_rn(__fmul_rn(ad, ad), g);
    v[3] += (double)__fmul_rn(d, d);
    v[4] += (double)__fmul_rn(dl, dl);
    v[5] += (double)l10;
    v[6] += (double)dl;
    v[7] += (r1 < 1.25f && r2 < 1.25f) ? 1.0 : 0.0;                  // max(p/g, g/p) < 1.25^k, NaN counts as false
    v[8] += (r1 < 1.5625f && r2 < 1.5625f) ? 1.0 : 0.0;
    v[9] += (r1 < 1.953125f && r2 < 1.953125f) ? 1.0 : 0.0;
    v[10] += (double)__fmul_rn(di, di);
  }
  if (ws) block_sum_store<kMetricFields>(v, ws + ((long long)b * gridDim.x + blockIdx.x) * kMetricFields);
}

// One thread: per-sample sums in block order, then metric.py's batch semantics -- per-sample means averaged over B,
// log10 pooled over the batch's pixels (:90-98), silog with the batch mean inside the sqrt (:145-160).
__global__ void eval_depth_metrics_finalize_kernel(const double* __restrict__ ws, int B, int nblk,
                                                   float* __restrict__ out) {
  double m[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double l10_sum = 0.0, l10_n = 0.0;
  for (int b = 0; b < B; ++b) {
    double s[kMetricFields];
    for (int f = 0; f < kMetricFields; ++f) s[f] = 0.0;
    for (int k = 0; k < nblk; ++k) {
      const double* p = ws + ((long long)b * nblk + k) * kMetricFields;
      for (int f = 0; f < kMetricFields; ++f) s[f] += p[f];
    }
    const double n = s[0];
    m[0] += s[1] / n;
    m[1] += s[2] / n;
    m[2] += sqrt(s[3] / n);
    m[3] += sqrt(s[4] / n);
    l10_sum += s[5];
    l10_n += n;
    m[5] += s[7] / n;
    m[6] += s[8] / n;
    m[7] += s[9] / n;
    m[8] += sqrt(s[10] / n);
    m[9] += s[4] / n - (s[6] * s[6]) / (n * n);
  }
  for (int f = 0; f < 10; ++f) m[f] /= (double)B;
  m[4] = l10_sum / l10_n;
  m[9] = sqrt(m[9]) * 100.0;
  for (int f = 0; f < 10; ++f) out[f] = (float)m[f];
}

// ------------------------------------------------------------------------------------ normal angular error
// angle = acos(clamp(x.y / (max(|x|, 1e-8) max(|y|, 1e-8)), -1, 1)) * 180 / pi: torch.cosine_similarity then
// utils.py:155-157.  The cosine is evaluated in fp64 and rounded once to fp32, so pred == gt gives exactly 1 (0
// degrees, as torch gives): next to 0 degrees one fp32 ulp of the cosine moves the angle by 0.02 degrees, so a
// cosine rounded several times in fp32 would not stay within a few hundredths of a degree of torch's.  The rest is fp32.
constexpr int kNormalFields = 8;     // sum e, sum e^2, n, then the counts below 5, 7.5, 11.25, 22.5, 30 degrees

__device__ __forceinline__ float angle_deg(float x0, float x1, float x2, float y0, float y1, float y2) {
  const double nx = fmax(sqrt((double)x0 * x0 + (double)x1 * x1 + (double)x2 * x2), 1e-8);
  const double ny = fmax(sqrt((double)y0 * y0 + (double)y1 * y1 + (double)y2 * y2), 1e-8);
  const double dot = (double)x0 * y0 + (double)x1 * y1 + (double)x2 * y2;
  float c = (float)(dot / (nx * ny));
  c = fminf(fmaxf(c, -1.0f), 1.0f);
  return __fdiv_rn(__fmul_rn(acosf(c), 180.0f), (float)CUDART_PI);
}

__global__ void eval_normal_error_kernel(const float* __restrict__ pred, long long ps_b, long long ps_c,
                                         long long ps_h, long long ps_w, const float* __restrict__ gt, long long gs_b,
                                         long long gs_c, long long gs_h, long long gs_w,
                                         const unsigned char* __restrict__ mask, int H, int W,
                                         float* __restrict__ err_map, float* __restrict__ buf, long long buf_capacity,
                                         unsigned long long* __restrict__ buf_len, double* __restrict__ ws) {
  const int b = blockIdx.y;
  const long long HW = (long long)H * W;
  double v[kNormalFields];
#pragma unroll
  for (int f = 0; f < kNormalFields; ++f) v[f] = 0.0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  // every lane of a warp runs the same number of iterations, so the ballot below sees the whole warp
  const long long start = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long iters = (HW + stride - 1) / stride;
  for (long long it = 0; it < iters; ++it) {
    const long long i = start + it * stride;
    bool valid = false;
    float e = 0.f;
    if (i < HW) {
      const long long h = i / W, w = i - h * W;
      const float* p = pred + b * ps_b + h * ps_h + w * ps_w;
      const float* q = gt + b * gs_b + h * gs_h + w * gs_w;
      e = angle_deg(p[0], p[ps_c], p[2 * ps_c], q[0], q[gs_c], q[2 * gs_c]);
      if (err_map) err_map[b * HW + i] = e;
      valid = mask == nullptr || mask[b * HW + i] != 0;
    }
    if (buf) {                                        // compaction: one 64-bit counter atomic per warp
      const unsigned ballot = __ballot_sync(0xffffffffu, valid);
      unsigned long long base = 0;
      const int lane = threadIdx.x & 31;
      if (lane == 0 && ballot) base = atomicAdd(buf_len, (unsigned long long)__popc(ballot));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (valid) {
        const unsigned long long pos = base + __popc(ballot & ((1u << lane) - 1u));
        if (pos < (unsigned long long)buf_capacity) buf[pos] = e;
      }
    }
    if (valid) {
      v[0] += (double)e;
      v[1] += (double)e * (double)e;
      v[2] += 1.0;
      v[3] += e < 5.0f ? 1.0 : 0.0;
      v[4] += e < 7.5f ? 1.0 : 0.0;
      v[5] += e < 11.25f ? 1.0 : 0.0;
      v[6] += e < 22.5f ? 1.0 : 0.0;
      v[7] += e < 30.0f ? 1.0 : 0.0;
    }
  }
  block_sum_store<kNormalFields>(v, ws + ((long long)b * gridDim.x + blockIdx.x) * kNormalFields);
}

// One thread: add this launch's partials, sample by sample and block by block, to the caller's running totals.
__global__ void eval_normal_accumulate_kernel(const double* __restrict__ ws, int B, int nblk, double* __restrict__ sums,
                                              long long* __restrict__ counts) {
  for (int b = 0; b < B; ++b) {
    double s[kNormalFields];
    for (int f = 0; f < kNormalFields; ++f) s[f] = 0.0;
    for (int k = 0; k < nblk; ++k) {
      const double* p = ws + ((long long)b * nblk + k) * kNormalFields;
      for (int f = 0; f < kNormalFields; ++f) s[f] += p[f];
    }
    sums[0] += s[0];
    sums[1] += s[1];
    for (int f = 0; f < 6; ++f) counts[f] += (long long)s[2 + f];
  }
}

// ------------------------------------------------------------------------------------ k-th smallest (radix select)
// Keys are the fp32 bit patterns, which order non-negative floats as their values (-0 is folded onto +0).  Four
// passes of 8 bits each: a histogram of the keys that share the digits chosen so far (shared-memory counts, then one
// 64-bit integer atomic per bin and block), then one thread picks the bin holding the rank.  The (k+1)-th value is
// the k-th again when the k-th value occurs past rank k, else the smallest key above it (one more pass).
// ws layout (unsigned long long): [0, 256) histogram, then state.
enum { kKsHist = 0, kKsN = 256, kKsRank, kKsPrefix, kKsEqualEnd, kKsNextKey, kKsWords };

__device__ __forceinline__ unsigned int ks_key(float x) {
  const unsigned int u = __float_as_uint(x);
  return u == 0x80000000u ? 0u : u;
}

__global__ void eval_ks_init_kernel(const unsigned long long* __restrict__ n_dev, long long k,
                                    unsigned long long* __restrict__ ws) {
  const int t = threadIdx.x;
  if (t < 256) ws[kKsHist + t] = 0ull;
  if (t == 0) {
    const unsigned long long n = *n_dev;
    ws[kKsN] = n;
    ws[kKsRank] = k >= 0 ? (unsigned long long)k : (n > 0 ? (n - 1) / 2 : 0ull);
    ws[kKsPrefix] = 0ull;
    ws[kKsEqualEnd] = 0ull;
    ws[kKsNextKey] = 0xFFFFFFFFull;
  }
}

__global__ void eval_ks_hist_kernel(const float* __restrict__ x, int shift, unsigned long long* __restrict__ ws) {
  __shared__ unsigned int h[256];
  for (int t = threadIdx.x; t < 256; t += blockDim.x) h[t] = 0u;
  __syncthreads();
  const unsigned long long n = ws[kKsN];
  const unsigned int prefix = (unsigned int)ws[kKsPrefix];
  const int hi_shift = shift + 8;                     // the digits above this pass must equal the prefix
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned int key = ks_key(x[i]);
    if (hi_shift < 32 && ((key ^ prefix) >> hi_shift) != 0u) continue;
    atomicAdd(&h[(key >> shift) & 255u], 1u);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 256; t += blockDim.x)
    if (h[t]) atomicAdd(&ws[kKsHist + t], (unsigned long long)h[t]);
}

__global__ void eval_ks_select_kernel(int shift, unsigned long long* __restrict__ ws) {
  if (threadIdx.x != 0) return;
  unsigned long long rank = ws[kKsRank], below = 0ull;
  int d = 255;
  for (int t = 0; t < 256; ++t) {
    const unsigned long long c = ws[kKsHist + t];
    if (rank < below + c) { d = t; break; }
    below += c;
  }
  const unsigned long long equal = ws[kKsHist + d];
  ws[kKsRank] = rank - below;
  ws[kKsPrefix] |= (unsigned long long)d << shift;
  if (shift == 0) ws[kKsEqualEnd] = equal;           // copies of the k-th value at ranks >= k: rank - below .. equal - 1
  for (int t = 0; t < 256; ++t) ws[kKsHist + t] = 0ull;
}

__global__ void eval_ks_next_kernel(const float* __restrict__ x, long long k, unsigned long long* __restrict__ ws) {
  const unsigned long long n = ws[kKsN];
  if (ws[kKsRank] + 1 < ws[kKsEqualEnd]) return;     // the (k+1)-th value is the k-th again
  const unsigned int key_k = (unsigned int)ws[kKsPrefix];
  unsigned int best = 0xFFFFFFFFu;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned int key = ks_key(x[i]);
    if (key > key_k && key < best) best = key;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0xFFFFFFFFu) atomicMin(&ws[kKsNextKey], (unsigned long long)best);
}

// out[0] = k-th, out[1] = (k+1)-th (the k-th when k is the last rank), out[2] = out[0] for an explicit k or an odd
// median count, else (out[0] + out[1]) / 2 in fp32 (np.median of a float32 array); NaN for an empty input.
__global__ void eval_ks_finish_kernel(long long k, const unsigned long long* __restrict__ ws, float* __restrict__ out) {
  const unsigned long long n = ws[kKsN];
  if (n == 0ull || (k >= 0 && (unsigned long long)k >= n)) {
    out[0] = out[1] = out[2] = CUDART_NAN_F;
    return;
  }
  const float a = __uint_as_float((unsigned int)ws[kKsPrefix]);
  const unsigned long long kk = k >= 0 ? (unsigned long long)k : (n - 1) / 2;
  float b = a;
  if (kk + 1 < n && ws[kKsRank] + 1 >= ws[kKsEqualEnd]) b = __uint_as_float((unsigned int)ws[kKsNextKey]);
  out[0] = a;
  out[1] = b;
  out[2] = (k < 0 && (n % 2ull) == 0ull) ? __fdiv_rn(__fadd_rn(a, b), 2.0f) : a;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_eval_align_depth(const float* gt, const float* pred, const unsigned char* mask, int B, int H, int W,
                                     int OW, float col_scale, int disparity, double* ws, float* scale_shift,
                                     void* stream) {
  B200_CHECK_ARG(gt && pred && mask && ws && scale_shift, "b200_eval_align_depth: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && OW >= 1 && OW <= W,
                 "b200_eval_align_depth: bad shape B=%d H=%d W=%d OW=%d", B, H, W, OW);
  B200_CHECK_ARG(OW == W || col_scale > 0.f, "b200_eval_align_depth: col_scale must be > 0");
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = eval_blocks((long long)H * OW);
  eval_align_moments_kernel<<<dim3(nblk, B), kEvalThreads, 0, st>>>(gt, pred, mask, H, W, OW, col_scale, disparity, ws);
  B200_CHECK_LAUNCH("eval_align_moments_kernel");
  eval_align_solve_kernel<<<(B + 127) / 128, 128, 0, st>>>(ws, B, nblk, scale_shift);
  B200_CHECK_LAUNCH("eval_align_solve_kernel");
  return 0;
}

extern "C" int b200_eval_depth_metrics(const float* pred, const float* gt, const unsigned char* mask, int B,
                                       long long HW, const float* scale_shift, int disparity, int clip,
                                       float min_depth, float max_depth, float* aligned, double* ws, float* out,
                                       void* stream) {
  B200_CHECK_ARG(pred, "b200_eval_depth_metrics: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && HW >= 1, "b200_eval_depth_metrics: bad shape B=%d HW=%lld", B, HW);
  B200_CHECK_ARG(out == nullptr || (gt && ws), "b200_eval_depth_metrics: metrics need gt and ws");
  B200_CHECK_ARG(out || aligned, "b200_eval_depth_metrics: nothing to write");
  B200_CHECK_ARG(!disparity || scale_shift, "b200_eval_depth_metrics: disparity mode needs scale_shift");
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = eval_blocks(HW);
  eval_depth_metrics_kernel<<<dim3(nblk, B), kEvalThreads, 0, st>>>(pred, gt, mask, HW, scale_shift, disparity, clip,
                                                                    min_depth, max_depth, aligned, out ? ws : nullptr);
  B200_CHECK_LAUNCH("eval_depth_metrics_kernel");
  if (out) {
    eval_depth_metrics_finalize_kernel<<<1, 1, 0, st>>>(ws, B, nblk, out);
    B200_CHECK_LAUNCH("eval_depth_metrics_finalize_kernel");
  }
  return 0;
}

extern "C" int b200_eval_normal_error(const float* pred, const long long* pred_strides, const float* gt,
                                      const long long* gt_strides, const unsigned char* mask, int B, int H, int W,
                                      float* err_map, float* buf, long long buf_capacity, unsigned long long* buf_len,
                                      double* ws, double* sums, long long* counts, void* stream) {
  B200_CHECK_ARG(pred && gt && pred_strides && gt_strides && ws, "b200_eval_normal_error: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && H >= 1 && W >= 1, "b200_eval_normal_error: bad shape B=%d H=%d W=%d", B, H, W);
  B200_CHECK_ARG(!buf || (buf_len && buf_capacity >= 0), "b200_eval_normal_error: buf needs buf_len");
  B200_CHECK_ARG((sums == nullptr) == (counts == nullptr), "b200_eval_normal_error: sums and counts go together");
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = eval_blocks((long long)H * W);
  eval_normal_error_kernel<<<dim3(nblk, B), kEvalThreads, 0, st>>>(
      pred, pred_strides[0], pred_strides[1], pred_strides[2], pred_strides[3], gt, gt_strides[0], gt_strides[1],
      gt_strides[2], gt_strides[3], mask, H, W, err_map, buf, buf_capacity, buf_len, ws);
  B200_CHECK_LAUNCH("eval_normal_error_kernel");
  if (sums) {
    eval_normal_accumulate_kernel<<<1, 1, 0, st>>>(ws, B, nblk, sums, counts);
    B200_CHECK_LAUNCH("eval_normal_accumulate_kernel");
  }
  return 0;
}

extern "C" int b200_eval_kth_smallest(const float* x, const unsigned long long* n, long long n_max, long long k,
                                      unsigned long long* ws, float* out, void* stream) {
  B200_CHECK_ARG(x && n && ws && out, "b200_eval_kth_smallest: null pointer");
  B200_CHECK_ARG(n_max >= 0, "b200_eval_kth_smallest: n_max < 0");
  cudaStream_t st = (cudaStream_t)stream;
  long long g = (n_max + 8LL * kEvalThreads - 1) / (8LL * kEvalThreads);
  const long long cap = 4LL * B200_EVAL_MAX_BLOCKS;
  const unsigned grid = (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
  eval_ks_init_kernel<<<1, 256, 0, st>>>(n, k, ws);
  B200_CHECK_LAUNCH("eval_ks_init_kernel");
  for (int shift = 24; shift >= 0; shift -= 8) {
    eval_ks_hist_kernel<<<grid, kEvalThreads, 0, st>>>(x, shift, ws);
    B200_CHECK_LAUNCH("eval_ks_hist_kernel");
    eval_ks_select_kernel<<<1, 32, 0, st>>>(shift, ws);
    B200_CHECK_LAUNCH("eval_ks_select_kernel");
  }
  eval_ks_next_kernel<<<grid, kEvalThreads, 0, st>>>(x, k, ws);
  B200_CHECK_LAUNCH("eval_ks_next_kernel");
  eval_ks_finish_kernel<<<1, 1, 0, st>>>(k, ws, out);
  B200_CHECK_LAUNCH("eval_ks_finish_kernel");
  return 0;
}
