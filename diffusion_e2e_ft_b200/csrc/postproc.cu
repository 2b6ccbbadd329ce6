// Host-pipeline post-processing on the device (SURVEY.md §8 a11 / f2): test-time ensembling of normals (argmin index
// selection) and of affine-invariant depth maps (objective of the scipy-BFGS alignment + median / MAD reduction),
// row min/max for the [0,1] normalisation, uint8 -> [-1,1] conversion and the antialiased bilinear resize of the
// pipeline's input / output.  All HBM-bound streaming kernels; fp64 accumulators for the global sums.
//   Marigold/marigold/marigold_pipeline.py:59-71,237-247,300-321   GeoWizard/geowizard/utils/normal_ensemble.py:6-22
//   Marigold/marigold/util/ensemble.py:40-132
#include <math_constants.h>

#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

constexpr int kMaxEnsemble = 32;

__device__ __forceinline__ double pp_warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float pp_warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float pp_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// order-preserving float <-> uint32 map, so atomicMin / atomicMax work on floats of either sign
__device__ __forceinline__ unsigned int f2ord(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned int u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u);
}

// ------------------------------------------------------------------------------------------ normals ensembling
// preds [E][3][HW] fp32.  err[e] += sum over pixels of acos(clip(cos(mean_normal, n_e), -0.999, 0.999)), where
// n_e = p_e / (|p_e| + 1e-5) and the mean normal is rebuilt from the mean azimuth / polar angles (:62-68).
__device__ __forceinline__ void unit_normal(const float* __restrict__ p, long long HW, long long i, float& x, float& y,
                                            float& z) {
  const float a = p[i], b = p[HW + i], c = p[2 * HW + i];
  const float inv = 1.0f / (sqrtf(a * a + b * b + c * c) + 1e-5f);
  x = a * inv; y = b * inv; z = c * inv;
}

__global__ void ens_normals_err_kernel(const float* __restrict__ preds, int E, long long HW, double* __restrict__ err) {
  __shared__ double s_err[kMaxEnsemble];
  if (threadIdx.x < kMaxEnsemble) s_err[threadIdx.x] = 0.0;
  __syncthreads();
  double acc[kMaxEnsemble];
#pragma unroll
  for (int e = 0; e < kMaxEnsemble; ++e) acc[e] = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    float phi = 0.f, theta = 0.f;
    for (int e = 0; e < E; ++e) {
      float x, y, z;
      unit_normal(preds + (long long)e * 3 * HW, HW, i, x, y, z);
      phi += atan2f(y, x);
      theta += atan2f(sqrtf(x * x + y * y), z);
    }
    phi /= (float)E;
    theta /= (float)E;
    const float mx = sinf(theta) * cosf(phi), my = sinf(theta) * sinf(phi), mz = cosf(theta);
    const float mn = fmaxf(sqrtf(mx * mx + my * my + mz * mz), 1e-8f);
#pragma unroll
    for (int e = 0; e < kMaxEnsemble; ++e) {
      if (e < E) {
        float x, y, z;
        unit_normal(preds + (long long)e * 3 * HW, HW, i, x, y, z);
        const float nn = fmaxf(sqrtf(x * x + y * y + z * z), 1e-8f);
        float cs = (mx / mn) * (x / nn) + (my / mn) * (y / nn) + (mz / mn) * (z / nn);
        cs = fminf(fmaxf(cs, -0.999f), 0.999f);
        acc[e] += (double)acosf(cs);
      }
    }
  }
#pragma unroll
  for (int e = 0; e < kMaxEnsemble; ++e) {
    if (e < E) {
      const double s = pp_warp_sum_d(acc[e]);
      if ((threadIdx.x & 31) == 0) atomicAdd(&s_err[e], s);
    }
  }
  __syncthreads();
  if (threadIdx.x < E) atomicAdd(&err[threadIdx.x], s_err[threadIdx.x]);
}

// index = argmin_e err[e] (first minimum, like torch.argmin); out[3][HW] = normalised preds[index]
__global__ void ens_normals_pick_kernel(const float* __restrict__ preds, int E, long long HW,
                                        const double* __restrict__ err, float* __restrict__ out, int* __restrict__ index) {
  int best = 0;
  double bv = err[0];
  for (int e = 1; e < E; ++e)
    if (err[e] < bv) { bv = err[e]; best = e; }
  if (blockIdx.x == 0 && threadIdx.x == 0) *index = best;
  const float* p = preds + (long long)best * 3 * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    float x, y, z;
    unit_normal(p, HW, i, x, y, z);
    out[i] = x; out[HW + i] = y; out[2 * HW + i] = z;
  }
}

// ------------------------------------------------------------------------------------------ depth ensembling
// v_e = img_e * s_e + t_e (two roundings, as torch evaluates `input * s + t`).  reduction 0 = median (torch.median:
// the lower of the two middle values for an even count), 1 = mean.
__device__ __forceinline__ float lower_median(float* v, int E) {
  for (int a = 1; a < E; ++a) {            // insertion sort, E <= 32
    const float key = v[a];
    int b = a - 1;
    while (b >= 0 && v[b] > key) { v[b + 1] = v[b]; --b; }
    v[b + 1] = key;
  }
  return v[(E - 1) / 2];
}

// acc[0] += sum over pixels and pairs i<j of (v_i - v_j)^2;  mm[0] = min(pred), mm[1] = max(pred) (ordered-uint encoded)
__global__ void ens_depths_objective_kernel(const float* __restrict__ imgs, const float* __restrict__ s,
                                            const float* __restrict__ t, int E, long long HW, int reduction,
                                            double* __restrict__ acc, unsigned int* __restrict__ mm) {
  float sc[kMaxEnsemble], sh[kMaxEnsemble];
  for (int e = 0; e < E; ++e) { sc[e] = s[e]; sh[e] = t[e]; }
  double sum = 0.0;
  float lo = CUDART_INF_F, hi = -CUDART_INF_F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    float v[kMaxEnsemble];
    float mean = 0.f;
    for (int e = 0; e < E; ++e) {
      v[e] = __fadd_rn(__fmul_rn(imgs[(long long)e * HW + i], sc[e]), sh[e]);
      mean += v[e];
    }
    float d2 = 0.f;
    for (int a = 0; a < E; ++a)
      for (int b = a + 1; b < E; ++b) { const float d = v[a] - v[b]; d2 = fmaf(d, d, d2); }
    sum += (double)d2;
    const float pred = reduction == 1 ? mean / (float)E : lower_median(v, E);
    lo = fminf(lo, pred);
    hi = fmaxf(hi, pred);
  }
  sum = pp_warp_sum_d(sum);
  lo = pp_warp_min(lo);
  hi = pp_warp_max(hi);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(acc, sum);
    atomicMin(&mm[0], f2ord(lo));
    atomicMax(&mm[1], f2ord(hi));
  }
}

// aligned[HW] = median / mean of the transformed maps, unc[HW] = MAD / std (unbiased); mm = min / max of aligned
__global__ void ens_depths_reduce_kernel(const float* __restrict__ imgs, const float* __restrict__ s,
                                         const float* __restrict__ t, int E, long long HW, int reduction,
                                         float* __restrict__ aligned, float* __restrict__ unc,
                                         unsigned int* __restrict__ mm) {
  float sc[kMaxEnsemble], sh[kMaxEnsemble];
  for (int e = 0; e < E; ++e) { sc[e] = s[e]; sh[e] = t[e]; }
  float lo = CUDART_INF_F, hi = -CUDART_INF_F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    float v[kMaxEnsemble], w[kMaxEnsemble];
    float mean = 0.f;
    for (int e = 0; e < E; ++e) {
      v[e] = __fadd_rn(__fmul_rn(imgs[(long long)e * HW + i], sc[e]), sh[e]);
      w[e] = v[e];
      mean += v[e];
    }
    float a, u;
    if (reduction == 1) {
      a = mean / (float)E;
      float q = 0.f;
      for (int e = 0; e < E; ++e) { const float d = v[e] - a; q = fmaf(d, d, q); }
      u = sqrtf(q / (float)(E > 1 ? E - 1 : 1));
    } else {
      a = lower_median(w, E);
      for (int e = 0; e < E; ++e) w[e] = fabsf(v[e] - a);
      u = lower_median(w, E);
    }
    aligned[i] = a;
    unc[i] = u;
    lo = fminf(lo, a);
    hi = fmaxf(hi, a);
  }
  lo = pp_warp_min(lo);
  hi = pp_warp_max(hi);
  if ((threadIdx.x & 31) == 0) {
    atomicMin(&mm[0], f2ord(lo));
    atomicMax(&mm[1], f2ord(hi));
  }
}

// x = (x - min) / (max - min), u /= (max - min)    (ensemble.py:126-130; also marigold_pipeline.py:307-312 with u = null)
__global__ void minmax_normalise_kernel(float* __restrict__ x, float* __restrict__ u, long long n,
                                        const unsigned int* __restrict__ mm, float* __restrict__ mm_out) {
  const float lo = ord2f(mm[0]), hi = ord2f(mm[1]);
  const float range = hi - lo;
  if (mm_out && blockIdx.x == 0 && threadIdx.x == 0) { mm_out[0] = lo; mm_out[1] = hi; }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    x[i] = (x[i] - lo) / range;
    if (u) u[i] = u[i] / range;
  }
}

// per-row (min, max) of a [rows][cols] fp32 matrix -> out[rows][2]; one CTA per (row, chunk), ordered-uint atomics
__global__ void minmax_rows_kernel(const float* __restrict__ x, long long cols, unsigned int* __restrict__ mm) {
  const int r = blockIdx.y;
  const float* xr = x + (long long)r * cols;
  float lo = CUDART_INF_F, hi = -CUDART_INF_F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cols; i += (long long)gridDim.x * blockDim.x) {
    const float v = xr[i];
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  lo = pp_warp_min(lo);
  hi = pp_warp_max(hi);
  if ((threadIdx.x & 31) == 0) {
    atomicMin(&mm[2 * r], f2ord(lo));
    atomicMax(&mm[2 * r + 1], f2ord(hi));
  }
}
__global__ void minmax_decode_kernel(const unsigned int* __restrict__ mm, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ord2f(mm[i]);
}
__global__ void minmax_init_kernel(unsigned int* __restrict__ mm, int pairs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < pairs) { mm[2 * i] = 0xFFFFFFFFu; mm[2 * i + 1] = 0u; }
}

// ------------------------------------------------------------------------------------------ pre-processing
// uint8 / fp32 image in [0,255] -> fp32 in [-1,1]:  x / 255 * 2 - 1   (marigold_pipeline.py:245-247)
// round_u8: first round-half-even to an integer (torchvision's resize of a uint8 tensor rounds its float result back
// to uint8 before the pipeline normalises it: Marigold/marigold/util/image_util.py:107).
template <typename T>
__global__ void rgb_normalise_kernel(const T* __restrict__ x, long long n, int round_u8, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = (float)x[i];
    if (round_u8) v = fminf(fmaxf(rintf(v), 0.f), 255.f);
    out[i] = v / 255.0f * 2.0f - 1.0f;
  }
}

// Separable antialiased resize along one axis with torch's weights (aten upsample_{bilinear,bicubic}2d_aa, align_corners =
// False): for output index o, centre c = scale * (o + 0.5), support = (interp_size / 2) * max(scale, 1) with interp_size 2
// (triangle filter) or 4 (Keys cubic, a = -0.5), taps x in [floor(c - support + 0.5), floor(c + support + 0.5)) clipped to
// the input, weight filter((x - c + 0.5) / max(scale, 1)), normalised to sum 1.
// x: [planes][in_len][inner] -> out [planes][out_len][inner]  (inner = 1 for the width pass, = width for the height pass)
template <bool CUBIC>
__device__ __forceinline__ float aa_filter(float x) {
  x = fabsf(x);
  if constexpr (!CUBIC) {
    return x < 1.0f ? 1.0f - x : 0.f;
  } else {
    const float a = -0.5f;
    if (x < 1.0f) return ((a + 2.0f) * x - (a + 3.0f)) * x * x + 1.0f;
    if (x < 2.0f) return (((x - 5.0f) * x + 8.0f) * x - 4.0f) * a;
    return 0.f;
  }
}

template <bool CUBIC>
__global__ void resize_aa_axis_kernel(const float* __restrict__ x, long long planes, int in_len, int out_len,
                                      long long inner, float scale, float* __restrict__ out) {
  const long long total = planes * out_len * inner;
  const float half_size = CUBIC ? 2.0f : 1.0f;
  const float support = scale >= 1.0f ? half_size * scale : half_size;
  const float invscale = scale >= 1.0f ? 1.0f / scale : 1.0f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long in_i = idx % inner;
    const int o = (int)((idx / inner) % out_len);
    const long long pl = idx / (inner * out_len);
    const float center = scale * ((float)o + 0.5f);
    int xmin = (int)(center - support + 0.5f);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5f);
    if (xmax > in_len) xmax = in_len;
    float total_w = 0.f;
    for (int j = xmin; j < xmax; ++j) total_w += aa_filter<CUBIC>(((float)j - center + 0.5f) * invscale);
    const float* src = x + pl * in_len * inner + in_i;
    float acc = 0.f;
    for (int j = xmin; j < xmax; ++j)
      acc += (aa_filter<CUBIC>(((float)j - center + 0.5f) * invscale) / total_w) * src[(long long)j * inner];
    out[idx] = acc;
  }
}

// nearest resize of a [planes][H][W] fp32 tensor (geowizard_pipeline.py:206-209 normals at the input resolution):
// src = min(floor(dst * in / out), in - 1)
__global__ void resize_nearest_kernel(const float* __restrict__ x, long long planes, int H, int W, int OH, int OW,
                                      float* __restrict__ out) {
  const long long total = planes * OH * OW;
  const float sh = (float)H / (float)OH, sw = (float)W / (float)OW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int ow = (int)(idx % OW);
    const int oh = (int)((idx / OW) % OH);
    const long long pl = idx / ((long long)OW * OH);
    const int ih = min((int)floorf((float)oh * sh), H - 1);
    const int iw = min((int)floorf((float)ow * sw), W - 1);
    out[idx] = x[(pl * H + ih) * W + iw];
  }
}

// torch's `nearest-exact` resize of a [planes][H][W] fp32 tensor (the reference's resample_method="nearest",
// Marigold/marigold/util/image_util.py:115 NEAREST_EXACT): src = min(floor((dst + 0.5) * scale), in - 1) with the fp32
// scale in / out of aten's CUDA kernel (compute_scales_value), each operation rounded on its own.
// blockIdx.y strides over the planes * OH output rows (the source row is resolved once per row), x over the columns.
__global__ void resize_nearest_exact_kernel(const float* __restrict__ x, long long rows, int H, int W, int OH, int OW,
                                            float sh, float sw, float* __restrict__ out) {
  for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
    const int oh = (int)(r % OH);
    const long long pl = r / OH;
    const int ih = min((int)floorf(__fmul_rn(__fadd_rn((float)oh, 0.5f), sh)), H - 1);
    const float* __restrict__ src = x + (pl * H + ih) * W;
    float* __restrict__ dst = out + r * OW;
    for (int ow = blockIdx.x * blockDim.x + threadIdx.x; ow < OW; ow += gridDim.x * blockDim.x) {
      const int iw = min((int)floorf(__fmul_rn(__fadd_rn((float)ow, 0.5f), sw)), W - 1);
      dst[ow] = src[iw];
    }
  }
}

// ------------------------------------------------------------------------------------------ colouring
// Both colour kernels write uint8 HWC.  A thread owns a group of 4 pixels, so its 12 output bytes go out as three
// aligned 32-bit stores (the output base is 4-byte aligned); the n % 4 tail is written byte by byte.
__device__ __forceinline__ void store_rgb4(unsigned char* __restrict__ out, long long g, const unsigned char (&c)[12]) {
  unsigned int* o = reinterpret_cast<unsigned int*>(out + 12 * g);
#pragma unroll
  for (int w = 0; w < 3; ++w)
    o[w] = (unsigned)c[4 * w] | ((unsigned)c[4 * w + 1] << 8) | ((unsigned)c[4 * w + 2] << 16) |
           ((unsigned)c[4 * w + 3] << 24);
}

// matplotlib Colormap.__call__(clip(x, 0, 1)) on a float32 array: xa = x * N (one fp32 multiply), xa == N -> N - 1,
// int truncation, NaN -> the "bad" colour (0, 0, 0).  table [n][3] uint8 already holds (lut * 255).astype(uint8).
__device__ __forceinline__ int cmap_index(float v, int n, float fn) {
  v = fminf(fmaxf(v, 0.f), 1.f);
  const int k = (int)__fmul_rn(v, fn);
  return k >= n ? n - 1 : k;
}

__global__ void colorize_depth_kernel(const float* __restrict__ x, long long n, const unsigned char* __restrict__ table,
                                      int ncol, unsigned char* __restrict__ out) {
  extern __shared__ unsigned char s_tab[];
  for (int i = threadIdx.x; i < 3 * ncol; i += blockDim.x) s_tab[i] = table[i];
  __syncthreads();
  const float fn = (float)ncol;
  const long long groups = n / 4;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    unsigned char c[12];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const float v = x[4 * g + p];
      const int k = cmap_index(v, ncol, fn);
      const bool bad = isnan(v);
      c[3 * p] = bad ? 0 : s_tab[3 * k];
      c[3 * p + 1] = bad ? 0 : s_tab[3 * k + 1];
      c[3 * p + 2] = bad ? 0 : s_tab[3 * k + 2];
    }
    store_rgb4(out, g, c);
  }
  for (long long i = 4 * groups + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float v = x[i];
    const int k = cmap_index(v, ncol, fn);
    const bool bad = isnan(v);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) out[3 * i + ch] = bad ? 0 : s_tab[3 * k + ch];
  }
}

// numpy's ((clip(x, -1, 1) + 1) / 2 * 255).astype(uint8) on float32 (marigold_pipeline.py:340-343,
// geowizard_pipeline.py:219): every operation rounded separately (no FMA contraction), truncated; NaN -> 0.
__device__ __forceinline__ unsigned char normal_u8(float v) {
  if (isnan(v)) return 0;
  v = fminf(fmaxf(v, -1.f), 1.f);
  return (unsigned char)__float2uint_rz(__fmul_rn(__fdiv_rn(__fadd_rn(v, 1.f), 2.f), 255.f));
}

// x [3][HW] planar -> out [HW][3]
__global__ void colorize_normals_kernel(const float* __restrict__ x, long long HW, unsigned char* __restrict__ out) {
  const long long groups = HW / 4;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    unsigned char c[12];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) c[3 * p + ch] = normal_u8(x[ch * HW + 4 * g + p]);
    store_rgb4(out, g, c);
  }
  for (long long i = 4 * groups + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += stride) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) out[3 * i + ch] = normal_u8(x[ch * HW + i]);
  }
}

static unsigned pp_grid(long long n, int per_thread = 4) {
  long long g = (n + 256LL * per_thread - 1) / (256LL * per_thread);
  const long long cap = (long long)sm_count() * 8;
  if (g > cap) g = cap;
  return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_ensemble_normals(const float* preds, int E, long long HW, double* err_ws, float* out, int* index,
                                     void* stream) {
  B200_CHECK_ARG(preds && err_ws && out && index && HW > 0, "b200_ensemble_normals: bad arguments");
  B200_CHECK_ARG(E >= 1 && E <= kMaxEnsemble, "b200_ensemble_normals: ensemble size %d not in [1, %d]", E, kMaxEnsemble);
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(err_ws, 0, sizeof(double) * E, st);
  ens_normals_err_kernel<<<pp_grid(HW, 1), 256, 0, st>>>(preds, E, HW, err_ws);
  ens_normals_pick_kernel<<<pp_grid(HW), 256, 0, st>>>(preds, E, HW, err_ws, out, index);
  B200_CHECK_LAUNCH("ensemble_normals kernels");
  return 0;
}

extern "C" int b200_ensemble_depths_objective(const float* imgs, const float* s, const float* t, int E, long long HW,
                                              int reduction, double* ws, float* out3, void* stream) {
  B200_CHECK_ARG(imgs && s && t && ws && out3 && HW > 0, "b200_ensemble_depths_objective: bad arguments");
  B200_CHECK_ARG(E >= 1 && E <= kMaxEnsemble && (reduction == 0 || reduction == 1),
                 "b200_ensemble_depths_objective: E=%d (max %d) reduction=%d", E, kMaxEnsemble, reduction);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int* mm = reinterpret_cast<unsigned int*>(ws + 1);
  cudaMemsetAsync(ws, 0, sizeof(double), st);
  minmax_init_kernel<<<1, 32, 0, st>>>(mm, 1);
  ens_depths_objective_kernel<<<pp_grid(HW, 1), 256, 0, st>>>(imgs, s, t, E, HW, reduction, ws, mm);
  minmax_decode_kernel<<<1, 32, 0, st>>>(mm, 2, out3 + 1);
  // out3[0] = sqrt(mean over pairs and pixels of d^2) is finished on the host from ws[0] (double)
  B200_CHECK_LAUNCH("ensemble_depths_objective kernels");
  return 0;
}

extern "C" int b200_ensemble_depths_reduce(const float* imgs, const float* s, const float* t, int E, long long HW,
                                           int reduction, double* ws, float* aligned, float* uncertainty,
                                           void* stream) {
  B200_CHECK_ARG(imgs && s && t && ws && aligned && uncertainty && HW > 0, "b200_ensemble_depths_reduce: bad arguments");
  B200_CHECK_ARG(E >= 1 && E <= kMaxEnsemble && (reduction == 0 || reduction == 1),
                 "b200_ensemble_depths_reduce: E=%d (max %d) reduction=%d", E, kMaxEnsemble, reduction);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int* mm = reinterpret_cast<unsigned int*>(ws);
  minmax_init_kernel<<<1, 32, 0, st>>>(mm, 1);
  ens_depths_reduce_kernel<<<pp_grid(HW, 1), 256, 0, st>>>(imgs, s, t, E, HW, reduction, aligned, uncertainty, mm);
  minmax_normalise_kernel<<<pp_grid(HW), 256, 0, st>>>(aligned, uncertainty, HW, mm, nullptr);
  B200_CHECK_LAUNCH("ensemble_depths_reduce kernels");
  return 0;
}

extern "C" int b200_minmax_rows(const float* x, int rows, long long cols, unsigned int* ws, float* out, void* stream) {
  B200_CHECK_ARG(x && ws && out && rows > 0 && cols > 0, "b200_minmax_rows: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  minmax_init_kernel<<<(rows + 127) / 128, 128, 0, st>>>(ws, rows);
  long long g = (cols + 1023) / 1024;
  const long long cap = (long long)sm_count() * 8 / rows + 1;
  if (g > cap) g = cap;
  minmax_rows_kernel<<<dim3((unsigned)g, rows), 256, 0, st>>>(x, cols, ws);
  minmax_decode_kernel<<<(2 * rows + 127) / 128, 128, 0, st>>>(ws, 2 * rows, out);
  B200_CHECK_LAUNCH("minmax_rows kernels");
  return 0;
}

extern "C" int b200_minmax_normalise(float* x, long long n, unsigned int* ws, float* minmax_out, void* stream) {
  B200_CHECK_ARG(x && ws && n > 0, "b200_minmax_normalise: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  minmax_init_kernel<<<1, 32, 0, st>>>(ws, 1);
  long long g = (n + 1023) / 1024;
  const long long cap = (long long)sm_count() * 8;
  if (g > cap) g = cap;
  minmax_rows_kernel<<<dim3((unsigned)g, 1), 256, 0, st>>>(x, n, ws);
  minmax_normalise_kernel<<<pp_grid(n), 256, 0, st>>>(x, nullptr, n, ws, minmax_out);
  B200_CHECK_LAUNCH("minmax_normalise kernels");
  return 0;
}

extern "C" int b200_rgb_normalise(const void* x, int in_u8, long long n, int round_u8, float* out, void* stream) {
  B200_CHECK_ARG(x && out && n > 0, "b200_rgb_normalise: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (in_u8)
    rgb_normalise_kernel<unsigned char><<<pp_grid(n), 256, 0, st>>>((const unsigned char*)x, n, round_u8, out);
  else
    rgb_normalise_kernel<float><<<pp_grid(n), 256, 0, st>>>((const float*)x, n, round_u8, out);
  B200_CHECK_LAUNCH("rgb_normalise_kernel");
  return 0;
}

extern "C" int b200_resize_bilinear_aa(const float* x, long long planes, int H, int W, int OH, int OW, float* tmp,
                                       float* out, void* stream) {
  B200_CHECK_ARG(x && tmp && out && planes > 0 && H > 0 && W > 0 && OH > 0 && OW > 0,
                 "b200_resize_bilinear_aa: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  // width pass [planes*H][W] -> tmp [planes*H][OW], then height pass [planes][H][OW] -> out [planes][OH][OW]
  resize_aa_axis_kernel<false><<<pp_grid(planes * H * OW, 1), 256, 0, st>>>(x, planes * H, W, OW, 1, (float)W / (float)OW, tmp);
  resize_aa_axis_kernel<false><<<pp_grid(planes * OH * OW, 1), 256, 0, st>>>(tmp, planes, H, OH, OW, (float)H / (float)OH, out);
  B200_CHECK_LAUNCH("resize_aa_axis_kernel");
  return 0;
}

extern "C" int b200_resize_bicubic_aa(const float* x, long long planes, int H, int W, int OH, int OW, float* tmp,
                                      float* out, void* stream) {
  B200_CHECK_ARG(x && tmp && out && planes > 0 && H > 0 && W > 0 && OH > 0 && OW > 0,
                 "b200_resize_bicubic_aa: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  resize_aa_axis_kernel<true><<<pp_grid(planes * H * OW, 1), 256, 0, st>>>(x, planes * H, W, OW, 1, (float)W / (float)OW, tmp);
  resize_aa_axis_kernel<true><<<pp_grid(planes * OH * OW, 1), 256, 0, st>>>(tmp, planes, H, OH, OW, (float)H / (float)OH, out);
  B200_CHECK_LAUNCH("resize_aa_axis_kernel<cubic>");
  return 0;
}

extern "C" int b200_resize_nearest(const float* x, long long planes, int H, int W, int OH, int OW, float* out,
                                   void* stream) {
  B200_CHECK_ARG(x && out && planes > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "b200_resize_nearest: bad arguments");
  resize_nearest_kernel<<<pp_grid(planes * OH * OW, 1), 256, 0, (cudaStream_t)stream>>>(x, planes, H, W, OH, OW, out);
  B200_CHECK_LAUNCH("resize_nearest_kernel");
  return 0;
}

extern "C" int b200_resize_nearest_exact(const float* x, long long planes, int H, int W, int OH, int OW, float* out,
                                         void* stream) {
  B200_CHECK_ARG(x && out && planes > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "b200_resize_nearest_exact: bad arguments");
  const float sh = (float)H / (float)OH, sw = (float)W / (float)OW;
  const long long rows = planes * OH;
  const dim3 grid((unsigned)((OW + 255) / 256), (unsigned)(rows < 65535 ? rows : 65535));
  resize_nearest_exact_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, rows, H, W, OH, OW, sh, sw, out);
  B200_CHECK_LAUNCH("resize_nearest_exact_kernel");
  return 0;
}

extern "C" int b200_colorize_depth(const float* x, long long n, const unsigned char* table, int ncol,
                                   unsigned char* out, void* stream) {
  B200_CHECK_ARG(x && table && out && n > 0 && ncol > 0 && ncol <= 4096, "b200_colorize_depth: bad arguments");
  B200_CHECK_ARG(((uintptr_t)out & 3) == 0, "b200_colorize_depth: out must be 4-byte aligned");
  colorize_depth_kernel<<<pp_grid(n), 256, 3 * ncol, (cudaStream_t)stream>>>(x, n, table, ncol, out);
  B200_CHECK_LAUNCH("colorize_depth_kernel");
  return 0;
}

extern "C" int b200_colorize_normals(const float* x, long long HW, unsigned char* out, void* stream) {
  B200_CHECK_ARG(x && out && HW > 0, "b200_colorize_normals: bad arguments");
  B200_CHECK_ARG(((uintptr_t)out & 3) == 0, "b200_colorize_normals: out must be 4-byte aligned");
  colorize_normals_kernel<<<pp_grid(HW), 256, 0, (cudaStream_t)stream>>>(x, HW, out);
  B200_CHECK_LAUNCH("colorize_normals_kernel");
  return 0;
}
