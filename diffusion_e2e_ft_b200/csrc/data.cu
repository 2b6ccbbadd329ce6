// Training-batch preparation on the device (DESIGN.md §3 "Training inputs"): the per-sample transforms of
// training/dataloaders/load.py applied to decoded uint8 / uint16 images.
//   b200_data_hypersim_source  depth mm -> m and the normal orientation fix (load.py:217-238), flip correction of x
//   b200_data_resize_u8        Pillow's two-pass fixed-point BILINEAR resize (transforms.Resize on a PIL image)
//   b200_data_depth_gather     Pillow's NEAREST resize of the depth, or the KITTI benchmark crop; the flip folded in
//   b200_data_depth_range      torch.quantile(valid, 0.02 / 0.98) per image (segmented radix select)
//   b200_data_finalise         load.py:248-281 / :343-376 per output pixel
//   b200_data_vkitti_normals   the D2NT v3 normals of depth-to-normal-translator/python/gen_vkitti_normals.py
// All HBM-bound but the last, which is most likely fp64-bound.  Per-pixel arithmetic the reference does in fp32 / fp64 is written
// with explicitly rounded intrinsics so nvcc cannot contract it into FMAs: the outputs are bitwise those of the
// reference.  Nothing syncs the host.
#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

constexpr int kDataThreads = 256;
constexpr int kRangeThreads = 1024;

static unsigned data_grid(long long n) {
  long long g = (n + kDataThreads - 1) / kDataThreads;
  if (g > (1LL << 20)) g = 1LL << 20;
  return (unsigned)(g < 1 ? 1 : g);
}

// ToTensor of a uint8 channel (x / 255 in fp32) followed by `* 2.0 - 1.0`, each a separate torch op
__device__ __forceinline__ float u8_to_signed(unsigned char u) {
  return __fsub_rn(__fmul_rn(__fdiv_rn((float)u, 255.0f), 2.0f), 1.0f);
}

// ------------------------------------------------------------------------------------ Hypersim source pass
// load.py:222-238 in fp64 as numpy does it: depth = float32(mm / 1000); n = (b / 255) * 2 - 1 with y, z negated;
// p = (invK . (x, y, 1)) * depth (np.matmul, then the product); n is flipped where (n0 p0 + n1 p1) + n2 p2 > 0, then
// negated, and written back as uint8((n + 1) / 2 * 255) (truncated).  Then 255 - x for flipped samples (:81-84).
struct InvK { double m[9]; };

__global__ void data_hypersim_source_kernel(const unsigned short* __restrict__ depth_mm,
                                            const unsigned char* __restrict__ normal,
                                            const unsigned char* __restrict__ flip, int H, int W, InvK k,
                                            float* __restrict__ depth_m, unsigned char* __restrict__ normal_out) {
  const int b = blockIdx.y;
  const long long HW = (long long)H * W;
  const bool fl = flip && flip[b];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    const long long g = (long long)b * HW + i;
    const float d = (float)__ddiv_rn((double)depth_mm[g], 1000.0);
    depth_m[g] = d;
    const double x = (double)(i % W), y = (double)(i / W), dd = (double)d;
    double n[3], p[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      n[c] = __dadd_rn(__dmul_rn(__ddiv_rn((double)normal[3 * g + c], 255.0), 2.0), -1.0);
      p[c] = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(k.m[3 * c], x), __dmul_rn(k.m[3 * c + 1], y)), k.m[3 * c + 2]), dd);
    }
    n[1] = -n[1];
    n[2] = -n[2];
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(n[0], p[0]), __dmul_rn(n[1], p[1])), __dmul_rn(n[2], p[2]));
    const bool keep = !(dot > 0.0);             // orient_mask flips, then the whole map is negated
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double v = keep ? -n[c] : n[c];
      unsigned char u = (unsigned char)(int)__dmul_rn(__dmul_rn(__dadd_rn(v, 1.0), 0.5), 255.0);
      if (c == 0 && fl) u = (unsigned char)(255 - u);
      normal_out[3 * g + c] = u;
    }
  }
}

// ------------------------------------------------------------------------------------ Pillow BILINEAR (uint8)
// ImagingResample: the horizontal pass first, into a uint8 intermediate, then the vertical pass.  Output o of an axis
// reads source taps min[o] .. min[o] + ks - 1 with 22-bit integer weights kk[o * ks ..] (zero past the support);
// value = clamp((2^21 + sum w * src) >> 22, 0, 255).  A flipped sample reads the mirrored source column, which is
// what resizing the flipped image does.
__device__ __forceinline__ unsigned char clip8(int acc) {
  acc >>= 22;
  return (unsigned char)(acc < 0 ? 0 : (acc > 255 ? 255 : acc));
}

__global__ void data_resize_h_kernel(const unsigned char* __restrict__ src, int H, int W, int C, int OW,
                                     const int* __restrict__ xmin, const int* __restrict__ kk, int ks,
                                     const unsigned char* __restrict__ flip, unsigned char* __restrict__ dst) {
  const int b = blockIdx.y;
  const long long n = (long long)H * OW * C;
  const bool fl = flip && flip[b];
  const unsigned char* s = src + (long long)b * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long t = i / C;
    const int o = (int)(t % OW), y = (int)(t / OW);
    const unsigned char* row = s + (long long)y * W * C + c;
    int acc = 1 << 21;
    for (int j = 0; j < ks; ++j) {
      const int w = kk[o * ks + j];
      if (w == 0) continue;
      const int x = xmin[o] + j;
      acc += w * (int)row[(long long)(fl ? W - 1 - x : x) * C];
    }
    dst[(long long)b * n + i] = clip8(acc);
  }
}

__global__ void data_resize_v_kernel(const unsigned char* __restrict__ src, int H, int OW, int C, int OH,
                                     const int* __restrict__ ymin, const int* __restrict__ kk, int ks,
                                     unsigned char* __restrict__ dst) {
  const int b = blockIdx.y;
  const long long rowlen = (long long)OW * C, n = (long long)OH * rowlen;
  const unsigned char* s = src + (long long)b * H * rowlen;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i / rowlen);
    const long long r = i - (long long)o * rowlen;
    int acc = 1 << 21;
    for (int j = 0; j < ks; ++j) {
      const int w = kk[o * ks + j];
      if (w == 0) continue;
      acc += w * (int)s[(long long)(ymin[o] + j) * rowlen + r];
    }
    dst[(long long)b * n + i] = clip8(acc);
  }
}

// ------------------------------------------------------------------------------------ depth gather
// dst[b][i][j] = src[b][rows[i]][c] with c = cols[j], or W - 1 - cols[j] for a flipped sample.  The source is fp32
// metres, or uint16 centimetres converted as numpy's float32(cm) / 100.0 (load.py:330).
__global__ void data_depth_gather_kernel(const float* __restrict__ src_m, const unsigned short* __restrict__ src_cm,
                                         int H, int W, int OH, int OW, const int* __restrict__ rows,
                                         const int* __restrict__ cols, const unsigned char* __restrict__ flip,
                                         float* __restrict__ dst) {
  const int b = blockIdx.y;
  const long long n = (long long)OH * OW;
  const bool fl = flip && flip[b];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = rows[i / OW], c0 = cols[i % OW];
    const long long s = ((long long)b * H + r) * W + (fl ? W - 1 - c0 : c0);
    dst[(long long)b * n + i] = src_m ? src_m[s] : __fdiv_rn((float)src_cm[s], 100.0f);
  }
}

// ------------------------------------------------------------------------------------ per-image depth range
// One block per image.  n = #(near < d < far); for q in (0.02, 0.98) torch.quantile takes rank r = float32(q) *
// float32(n - 1) in fp32, the order statistics at floor(r) and ceil(r), and torch's CPU lerp, which is fused:
// small weight (< 0.5) fma(w, hi - lo, lo), else fma(w - 1, hi - lo, hi).  The four order statistics are found
// together by a radix select on the fp32 bit patterns (valid depths are positive, so the patterns order as the
// values): four passes of 8 bits, each a shared-memory histogram per wanted rank of the keys that share the digits
// chosen so far.  flag[b]: 0 = no valid pixel, 1 = min == max, 2 = a proper range in range[b] = (min, max).
__global__ void __launch_bounds__(kRangeThreads)
data_depth_range_kernel(const float* __restrict__ depth, long long HW, float near_plane, float far_plane,
                        float* __restrict__ range, int* __restrict__ flag) {
  __shared__ unsigned int hist[4][256];
  __shared__ unsigned int prefix[4], rank[4];
  __shared__ unsigned long long s_count[kRangeThreads / 32];
  const int b = blockIdx.x;
  const float* d = depth + (long long)b * HW;
  unsigned long long cnt = 0;
  for (long long i = threadIdx.x; i < HW; i += blockDim.x) cnt += (d[i] > near_plane && d[i] < far_plane) ? 1ull : 0ull;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) s_count[threadIdx.x >> 5] = cnt;
  __syncthreads();
  unsigned long long n = 0;
  for (int w = 0; w < kRangeThreads / 32; ++w) n += s_count[w];
  if (n == 0) {
    if (threadIdx.x == 0) { range[2 * b] = range[2 * b + 1] = 0.f; flag[b] = 0; }
    return;
  }
  const float q[2] = {0.02f, 0.98f};
  float r[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) r[k] = __fmul_rn(q[k], (float)(long long)(n - 1));
  if (threadIdx.x < 4) {
    const float rk = r[threadIdx.x >> 1];
    rank[threadIdx.x] = (threadIdx.x & 1) ? (unsigned int)ceilf(rk) : (unsigned int)rk;
    prefix[threadIdx.x] = 0u;
  }
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int t = threadIdx.x; t < 4 * 256; t += blockDim.x) hist[t >> 8][t & 255] = 0u;
    __syncthreads();
    const int hi_shift = shift + 8;
    unsigned int pre[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) pre[t] = prefix[t];
    for (long long i = threadIdx.x; i < HW; i += blockDim.x) {
      const float v = d[i];
      if (!(v > near_plane && v < far_plane)) continue;
      const unsigned int key = __float_as_uint(v);
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (hi_shift == 32 || ((key ^ pre[t]) >> hi_shift) == 0u) atomicAdd(&hist[t][(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      const int t = threadIdx.x;
      unsigned int below = 0, want = rank[t];
      int dig = 255;
      for (int j = 0; j < 256; ++j) {
        const unsigned int c = hist[t][j];
        if (want < below + c) { dig = j; break; }
        below += c;
      }
      rank[t] = want - below;
      prefix[t] |= (unsigned int)dig << shift;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float out[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const float lo = __uint_as_float(prefix[2 * k]), hi = __uint_as_float(prefix[2 * k + 1]);
      const float w = __fsub_rn(r[k], (float)(long long)r[k]);
      const float diff = __fsub_rn(hi, lo);
      out[k] = fabsf(w) < 0.5f ? __fmaf_rn(w, diff, lo) : __fmaf_rn(__fsub_rn(w, 1.0f), diff, hi);
    }
    range[2 * b] = out[0];
    range[2 * b + 1] = out[1];
    flag[b] = out[0] == out[1] ? 1 : 2;
  }
}

// ------------------------------------------------------------------------------------ finalise
// One thread per output pixel (b, i, j) of load.py:248-281.  rgb / normal are uint8 [B][H][W][3] read at row top + i
// and column left + j (mirrored, with 255 - x on the normal, for a flipped sample); depth is [B][OH][OW] fp32.
__global__ void data_finalise_kernel(const unsigned char* __restrict__ rgb, const unsigned char* __restrict__ normal,
                                     int H, int W, int top, int left, const unsigned char* __restrict__ flip,
                                     const float* __restrict__ depth, int OH, int OW, float near_plane,
                                     float far_plane, const float* __restrict__ range, const int* __restrict__ flag,
                                     float* __restrict__ rgb_out, float* __restrict__ depth_out,
                                     float* __restrict__ metric_out, float* __restrict__ normal_out,
                                     unsigned char* __restrict__ mask_out) {
  const int b = blockIdx.y;
  const long long n = (long long)OH * OW;
  const bool fl = flip && flip[b];
  const int f = flag[b];
  const float mn = range[2 * b], mx = range[2 * b + 1];
  const float span = __fsub_rn(mx, mn);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int oi = (int)(i / OW), oj = (int)(i % OW);
    const int c = left + oj;
    const long long s = (((long long)b * H + top + oi) * W + (fl ? W - 1 - c : c)) * 3;
    const long long o = (long long)b * 3 * n + i;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) rgb_out[o + ch * n] = u8_to_signed(rgb[s + ch]);

    const float d = depth[(long long)b * n + i];
    bool valid = d > near_plane && d < far_plane;
    float dn = 0.f, metric = 0.f;
    if (f == 1) {
      valid = false;
    } else if (f == 2) {
      metric = valid ? fminf(fmaxf(d, mn), mx) : mx;
      dn = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(metric, mn), span), 2.0f), 1.0f);
      dn = fminf(fmaxf(dn, -1.0f), 1.0f);
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) depth_out[o + ch * n] = dn;
    metric_out[(long long)b * n + i] = metric;
    mask_out[(long long)b * n + i] = valid ? 1 : 0;

    // F.normalize: fp32 squares summed in order, a correctly rounded sqrt, clamp_min(1e-12), one division each
    float v[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      unsigned char u = normal[s + ch];
      if (ch == 0 && fl) u = (unsigned char)(255 - u);
      v[ch] = u8_to_signed(u);
    }
    const float ss = __fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2]));
    const float nrm = fmaxf(__fsqrt_rn(ss), 1e-12f);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) normal_out[o + ch * n] = valid ? __fdiv_rn(v[ch], nrm) : 0.f;
  }
}

// ------------------------------------------------------------------------------------ Virtual KITTI 2 normals
// D2NT "v3" of depth-to-normal-translator/python/gen_vkitti_normals.py:97-136 (DAG-filtered gradients, the
// depth-to-normal translation, the DLF-alpha MRF refinement) per pixel, in the script's precisions (DESIGN.md §3.11).
// A CTA owns a kNrmTW x kNrmTH output tile and holds the fp32 depth of the tile plus a 3-pixel halo in shared memory
// (BORDER_REFLECT_101 applied at load).  Each thread picks its MRF candidate first and then computes the D2NT normal
// of that one pixel only: the refinement copies a neighbour's normal, so no other normal is needed.
constexpr int kNrmTW = 32, kNrmTH = 8, kNrmHalo = 3;
constexpr int kNrmSW = kNrmTW + 2 * kNrmHalo, kNrmSH = kNrmTH + 2 * kNrmHalo;
constexpr double kLnE32Hi = 0x1.fffffefb245eap-1;     // ln(float32(e)) = kLnE32Hi + kLnE32Lo (double-double)
constexpr double kLnE32Lo = 0x1.a2d208d1c4e82p-56;
constexpr double kLn2Hi = 0.6931471805599453, kLn2Lo = 2.3190468138462996e-17;

struct DD { double hi, lo; };

__device__ __forceinline__ DD quick_two_sum(double a, double b) {
  const double s = __dadd_rn(a, b);
  return {s, __dsub_rn(b, __dsub_rn(s, a))};
}
__device__ __forceinline__ DD two_sum(double a, double b) {
  const double s = __dadd_rn(a, b), bb = __dsub_rn(s, a);
  return {s, __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb))};
}
__device__ __forceinline__ DD dd_add(DD a, DD b) {
  DD s = two_sum(a.hi, b.hi);
  const DD t = two_sum(a.lo, b.lo);
  s = quick_two_sum(s.hi, __dadd_rn(s.lo, t.hi));
  return quick_two_sum(s.hi, __dadd_rn(s.lo, t.lo));
}
__device__ __forceinline__ DD dd_mul(DD a, DD b) {
  const double p = __dmul_rn(a.hi, b.hi);
  double e = __fma_rn(a.hi, b.hi, -p);
  e = __dadd_rn(e, __dadd_rn(__dmul_rn(a.hi, b.lo), __dmul_rn(a.lo, b.hi)));
  return quick_two_sum(p, e);
}
__device__ __forceinline__ DD dd_mul_d(DD a, double b) {
  const double p = __dmul_rn(a.hi, b);
  return quick_two_sum(p, __fma_rn(a.lo, b, __fma_rn(a.hi, b, -p)));
}
__device__ __forceinline__ DD dd_div_d(DD a, double b) {
  const double q1 = __ddiv_rn(a.hi, b);
  const double p = __dmul_rn(q1, b), pe = __fma_rn(q1, b, -p);
  const double r = __dadd_rn(__dsub_rn(__dsub_rn(a.hi, p), pe), a.lo);
  return quick_two_sum(q1, __ddiv_rn(r, b));
}

// exp(t) for a double-double t in about [-745, 709], to ~2^-95 relative: t = k ln2 + r, exp(r) = exp(r / 512)^512 with a
// degree-12 Taylor polynomial of exp(r / 512).
__device__ __forceinline__ DD dd_exp(DD t) {
  const double k = rint(__dmul_rn(t.hi, 1.4426950408889634));
  const DD r = dd_add(t, dd_mul_d(DD{-kLn2Hi, -kLn2Lo}, k));
  const DD s{r.hi * 0x1p-9, r.lo * 0x1p-9};
  DD acc{1.0, 0.0};
  for (int n = 12; n >= 1; --n) acc = dd_add(DD{1.0, 0.0}, dd_div_d(dd_mul(s, acc), (double)n));
  for (int i = 0; i < 9; ++i) acc = dd_mul(acc, acc);
  return {scalbn(acc.hi, (int)k), scalbn(acc.lo, (int)k)};
}

// float32(e) ** -x correctly rounded to fp32 (x >= 0 finite), returned widened to double.  soft_min's np.power runs
// in fp32 and is not correctly rounded on every CPU; this is the value its correctly rounded counterpart gives.  The
// fast path is exp() of the double-double argument -x ln(float32(e)), good to < 2^-51 relative; when that is within
// 2^-46 of an fp32 rounding boundary the double-double exp decides.  Subnormal results are kept.  force_slow takes the
// double-double path for every x and *slow reports whether it was taken (both only for b200_debug_pow_e32_neg).
__device__ __forceinline__ double pow_e32_neg(float x, bool force_slow = false, bool* slow = nullptr) {
  const double nx = -(double)x;
  const double th = __dmul_rn(nx, kLnE32Hi);
  const double tl = __fma_rn(nx, kLnE32Lo, __fma_rn(nx, kLnE32Hi, -th));
  const double e = exp(th);
  const double y = __fma_rn(e, tl, e);
  const float a = __double2float_rn(__dmul_rn(y, 1.0 - 0x1p-46)), b = __double2float_rn(__dmul_rn(y, 1.0 + 0x1p-46));
  if (a == b && !force_slow) return (double)a;
  if (slow) *slow = true;
  const DD v = dd_exp(DD{th, tl});
  const float lo = __double2float_rd(v.hi), hi = __double2float_ru(v.hi);
  if (lo == hi) return (double)lo;
  const double d = __dadd_rn(__dsub_rn(v.hi, __dmul_rn(__dadd_rn((double)lo, (double)hi), 0.5)), v.lo);
  if (d != 0.0) return (double)(d > 0.0 ? hi : lo);
  return (double)((__float_as_uint(lo) & 1u) ? hi : lo);
}

// soft_min's weights of one direction followed by get_DAG_filter's four in-place threshold updates (myApis.py:48-70,
// :112-120), in fp64; pa / pb are the powers of the laplacian one pixel before / after (0 off the image).
__device__ __forceinline__ void dag_weights(double pa, double pb, double& wa, double& wb) {
  const double eps = 1e-8, E = 2.718281828459045;
  const double den = __dadd_rn(__dadd_rn(eps, pa), pb);
  wa = __ddiv_rn(__dadd_rn(pa, eps * 0.5), den);
  wb = __ddiv_rn(__dadd_rn(pb, eps * 0.5), den);
  if (__ddiv_rn(wa, __dadd_rn(wb, eps)) > E) wa = 1.0;
  if (__ddiv_rn(wa, __dadd_rn(wb, eps)) > E) wb = 0.0;
  if (__ddiv_rn(wb, __dadd_rn(wa, eps)) > E) wa = 0.0;
  if (__ddiv_rn(wb, __dadd_rn(wa, eps)) > E) wb = 1.0;
}

__global__ void __launch_bounds__(kNrmTW * kNrmTH)
data_vkitti_normals_kernel(const unsigned short* __restrict__ depth_cm, int H, int W, float fx, float fy, float u0,
                           float v0, unsigned short* __restrict__ out) {
  __shared__ float z[kNrmSH][kNrmSW];
  const int b = blockIdx.z, x0 = blockIdx.x * kNrmTW, y0 = blockIdx.y * kNrmTH;
  const unsigned short* src = depth_cm + (long long)b * H * W;
  for (int t = threadIdx.y * kNrmTW + threadIdx.x; t < kNrmSH * kNrmSW; t += kNrmTW * kNrmTH) {
    int gy = y0 - kNrmHalo + t / kNrmSW, gx = x0 - kNrmHalo + t % kNrmSW;
    gy = gy < 0 ? -gy : (gy >= H ? 2 * H - 2 - gy : gy);   // BORDER_REFLECT_101; only distance 1 is ever read
    gx = gx < 0 ? -gx : (gx >= W ? 2 * W - 2 - gx : gx);
    gy = min(max(gy, 0), H - 1);
    gx = min(max(gx, 0), W - 1);
    // cv2.imread -> float32 / 100 (gen_vkitti_normals.py:63) -> ToTensor -> * 100 (:100)
    z[t / kNrmSW][t % kNrmSW] = __fmul_rn(__fdiv_rn((float)src[(long long)gy * W + gx], 100.0f), 100.0f);
  }
  __syncthreads();
  const int py = y0 + threadIdx.y, px = x0 + threadIdx.x;
  if (py >= H || px >= W) return;
  const int ty = threadIdx.y + kNrmHalo, tx = threadIdx.x + kNrmHalo;

  // MRF_optim (DLF-alpha): |cv2.filter2D(depth, lap_ker_alpha)| summed as cv2 does, of [left, right, up, down,
  // self]; off-image candidates are +inf and argmin keeps the first minimum
  auto lap_alpha = [&](int cy, int cx) {
    const float s = __fsub_rn(__fsub_rn(__fadd_rn(__fsub_rn(__fsub_rn(0.0f, z[cy - 1][cx]), z[cy][cx - 1]),
                                                  __fmul_rn(4.0f, z[cy][cx])), z[cy][cx + 1]), z[cy + 1][cx]);
    return fabsf(s);
  };
  const float inf = __int_as_float(0x7f800000);
  const float cand[5] = {px > 0 ? lap_alpha(ty, tx - 1) : inf, px < W - 1 ? lap_alpha(ty, tx + 1) : inf,
                         py > 0 ? lap_alpha(ty - 1, tx) : inf, py < H - 1 ? lap_alpha(ty + 1, tx) : inf,
                         lap_alpha(ty, tx)};
  int best = 0;
  float least = cand[0];
#pragma unroll
  for (int k = 1; k < 5; ++k)
    if (cand[k] < least) {
      least = cand[k];
      best = k;
    }
  const int qy = ty + (best == 2 ? -1 : best == 3 ? 1 : 0), qx = tx + (best == 0 ? -1 : best == 1 ? 1 : 0);
  const int gy = py + (qy - ty), gx = px + (qx - tx);

  // get_DAG_filter (1D-DLF) at q: one-sided fp32 gradients, their fp32 laplacians one pixel either side
  auto grad_l = [&](int cy, int cx) { return __fsub_rn(z[cy][cx], z[cy][cx - 1]); };
  auto grad_u = [&](int cy, int cx) { return __fsub_rn(z[cy][cx], z[cy - 1][cx]); };
  auto lap_hor = [&](int cy, int cx) { return fabsf(__fsub_rn(grad_l(cy, cx), grad_l(cy, cx + 1))); };
  auto lap_ver = [&](int cy, int cx) { return fabsf(__fsub_rn(grad_u(cy, cx), grad_u(cy + 1, cx))); };
  double l1, l2, l3, l4;
  dag_weights(gx > 0 ? pow_e32_neg(lap_hor(qy, qx - 1)) : 0.0, gx < W - 1 ? pow_e32_neg(lap_hor(qy, qx + 1)) : 0.0,
              l1, l2);
  dag_weights(gy > 0 ? pow_e32_neg(lap_ver(qy - 1, qx)) : 0.0, gy < H - 1 ? pow_e32_neg(lap_ver(qy + 1, qx)) : 0.0,
              l3, l4);
  const double Gu = __dadd_rn(__dmul_rn(l1, (double)grad_l(qy, qx)), __dmul_rn(l2, (double)grad_l(qy, qx + 1)));
  const double Gv = __dadd_rn(__dmul_rn(l3, (double)grad_u(qy, qx)), __dmul_rn(l4, (double)grad_u(qy + 1, qx)));

  // translation (:116-118) and vector_normalization (apis.py:38-41), fp64
  const double um = __dsub_rn((double)(gx + 1), (double)u0), vm = __dsub_rn((double)(gy + 1), (double)v0);
  const double n[3] = {__dmul_rn(Gu, (double)fx), __dmul_rn(Gv, (double)fy),
                       -__dadd_rn(__dadd_rn((double)z[qy][qx], __dmul_rn(vm, Gv)), __dmul_rn(um, Gu))};
  const double mag = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(n[0], n[0]), __dmul_rn(n[1], n[1])),
                                          __dmul_rn(n[2], n[2])));
  const double den = __dadd_rn(mag, 1e-8);
  // uint16((-n + 1) * 32767.5), truncated, stored in cvtColor(RGB2BGR) order: z, y, x
  unsigned short* o = out + (((long long)b * H + py) * W + px) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    o[2 - c] = (unsigned short)__double2uint_rz(__dmul_rn(__dadd_rn(-__ddiv_rn(n[c], den), 1.0), 32767.5));
}

// out[i] = pow_e32_neg(x[i]); counts in *slow_count (nullable) how many took the double-double path
__global__ void debug_pow_e32_neg_kernel(const float* __restrict__ x, long long n, int force_slow,
                                         float* __restrict__ out, unsigned int* __restrict__ slow_count) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    bool slow = false;
    out[i] = (float)pow_e32_neg(x[i], force_slow != 0, &slow);
    if (slow && slow_count) atomicAdd(slow_count, 1u);
  }
}

// ------------------------------------------------------------------------------------ Hypersim preprocessing
// Marigold's preprocess_hypersim.py / hypersim_util.py per frame (DESIGN.md §3.12), in the script's precisions:
//   brightness = (0.3 r + 0.59 g) + 0.11 b in fp64 over the valid pixels (entity id != -1);
//   p90 = np.percentile(brightness_valid, 90) (method 'linear'): the two order statistics by an exact radix select
//         on fp64 keys (8 passes of 8 bits over a per-pixel key buffer), then NumPy's virtual index, gamma and _lerp;
//   scale = 1 (no valid pixel), 0 (p90 < 1e-4), else pow(0.8, 2.2) / p90 (a NaN p90 gives a NaN scale);
//   rgb   = uint8(clip(pow(max(scale x, 0), 1 / 2.2), 0, 1) * 255) with the power correctly rounded, stored B, G, R;
//   depth = uint16(distance / ||(x, y, f)||_fp32 * f * 1000), 0 where invalid.
// NumPy's float64 -> uint8 / uint16 casts truncate through int32 on x86 and keep the low bits: NaN and anything
// outside the int32 range give 0, -3.7 gives 65533 (trunc_wrap).
constexpr int kHsPasses = 8;                           // 8-bit digits of a 64-bit key
constexpr int kHsHistThreads = 1024, kHsHistCtas = 64;  // per frame
constexpr unsigned long long kHsNoKey = ~0ull;         // invalid or NaN brightness: never a key of a non-NaN double
constexpr double kHsGamma = 1.0 / 2.2;                 // the script's gamma, 0.45454545454545453

__device__ __forceinline__ unsigned long long hs_key(double v) {   // orders as the values (-0 before +0)
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double hs_value(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}
__device__ __forceinline__ unsigned int trunc_wrap(double v) {
  return (v > -2147483649.0 && v < 2147483648.0) ? (unsigned int)(int)v : 0u;
}
template <typename T> __device__ __forceinline__ double hs_load(const T* p, long long i);
template <> __device__ __forceinline__ double hs_load<float>(const float* p, long long i) { return (double)p[i]; }
template <> __device__ __forceinline__ double hs_load<__half>(const __half* p, long long i) {
  return (double)__half2float(p[i]);
}

// The uint8 level of a tone-mapped value p = pow(m, gamma): uint8(clip(p, 0, 1) * 255), NaN -> 0.
__device__ __forceinline__ unsigned char hs_level(double p) {
  if (isnan(p)) return 0;
  return (unsigned char)trunc_wrap(__dmul_rn(fmin(fmax(p, 0.0), 1.0), 255.0));
}

// pow(m, gamma) for m > 0 finite in double-double: log(m) = e ln2 + log(f), m = f 2^e, f in [1, 2), with log(f) from
// one Newton step y0 + (f exp(-y0) - 1) on the fp64 log; then dd_exp of gamma log(m).  Good to ~2^-94 relative.
__device__ __forceinline__ double hs_pow_gamma_dd(double m) {
  int e;
  double f = frexp(m, &e);                             // [0.5, 1)
  f = __dmul_rn(f, 2.0);
  e -= 1;
  const double y0 = log(f);
  const DD ef = dd_mul_d(dd_exp(DD{-y0, 0.0}), f);
  const DD lf = dd_add(DD{y0, 0.0}, dd_add(ef, DD{-1.0, 0.0}));
  const DD lm = dd_add(dd_mul_d(DD{kLn2Hi, kLn2Lo}, (double)e), lf);
  const DD p = dd_exp(dd_mul_d(lm, kHsGamma));
  return __dadd_rn(p.hi, p.lo);
}

// The uint8 level of pow(m, gamma) with the power correctly rounded, for m = np.maximum(scale x, 0) (NaN kept).
// The fast fp64 pow is within a few ulp; when the level differs anywhere in +-2^-48 (relative) of it, the
// double-double power decides.  *p_out gets the power used; force_slow / *slow are for b200_debug_hypersim_pow.
__device__ __forceinline__ unsigned char hs_tone(double m, bool force_slow = false, bool* slow = nullptr,
                                                 double* p_out = nullptr) {
  double p;
  if (isnan(m) || m == 0.0 || isinf(m)) {
    p = isnan(m) ? m : (m == 0.0 ? 0.0 : m);
  } else {
    p = pow(m, kHsGamma);
    const unsigned char lo = hs_level(__dmul_rn(p, 1.0 - 0x1p-48)), hi = hs_level(__dmul_rn(p, 1.0 + 0x1p-48));
    if (lo != hi || force_slow) {
      if (slow) *slow = true;
      p = hs_pow_gamma_dd(m);
    }
  }
  if (p_out) *p_out = p;
  return hs_level(p);
}

// Pass 0: one fp64 brightness key per pixel (kHsNoKey where invalid or NaN), the per-frame counts of valid and of
// NaN-valued valid pixels, and the entity_id == 0 flag the script asserts on.
template <typename TR>
__global__ void hs_keys_kernel(const TR* __restrict__ rgb, const int* __restrict__ eid, long long HW,
                               unsigned long long* __restrict__ keys, unsigned long long* __restrict__ counts,
                               int* __restrict__ err) {
  const int b = blockIdx.y;
  unsigned long long n_valid = 0, n_nan = 0;
  bool zero = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    const long long g = (long long)b * HW + i;
    const int e = eid[g];
    zero |= e == 0;
    unsigned long long k = kHsNoKey;
    if (e != -1) {
      const double br = __dadd_rn(__dadd_rn(__dmul_rn(0.3, hs_load(rgb, 3 * g)), __dmul_rn(0.59, hs_load(rgb, 3 * g + 1))),
                                  __dmul_rn(0.11, hs_load(rgb, 3 * g + 2)));
      ++n_valid;
      if (isnan(br)) ++n_nan;
      else k = hs_key(br);
    }
    keys[g] = k;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    n_valid += __shfl_xor_sync(0xffffffffu, n_valid, o);
    n_nan += __shfl_xor_sync(0xffffffffu, n_nan, o);
  }
  if (__any_sync(0xffffffffu, zero) && (threadIdx.x & 31) == 0) atomicOr(err + b, 1);
  if ((threadIdx.x & 31) == 0 && n_valid) {
    atomicAdd(counts + 2 * b, n_valid);
    if (n_nan) atomicAdd(counts + 2 * b + 1, n_nan);
  }
}

// One radix pass: per frame and wanted rank (0: floor of the virtual index, 1: the next), the histogram of digit
// `pass` over the keys that share the digits chosen so far.  Warp-aggregated shared-memory counts, then one global
// atomic per non-empty bin per CTA.  Frames with no valid pixel or a NaN skip the select.
__global__ void __launch_bounds__(kHsHistThreads)
hs_hist_kernel(const unsigned long long* __restrict__ keys, long long HW, int pass,
               const unsigned long long* __restrict__ counts, const unsigned long long* __restrict__ sel,
               unsigned int* __restrict__ hist) {
  __shared__ unsigned int h[2 * 256];
  const int b = blockIdx.y;
  if (counts[2 * b] == 0 || counts[2 * b + 1] != 0) return;
  for (int t = threadIdx.x; t < 512; t += blockDim.x) h[t] = 0u;
  __syncthreads();
  const int shift = 56 - 8 * pass, hi_shift = shift + 8;
  const unsigned long long pre[2] = {sel[4 * b], sel[4 * b + 1]};
  const unsigned long long* k = keys + (long long)b * HW;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long end = (HW + 31) / 32 * 32;           // whole warps iterate together for __match_any_sync
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
    const unsigned long long key = i < HW ? k[i] : kHsNoKey;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const bool in = key != kHsNoKey && (pass == 0 || ((key ^ pre[r]) >> hi_shift) == 0ull);
      const unsigned int bin = in ? (unsigned int)(r * 256 + ((key >> shift) & 255ull)) : 512u;
      const unsigned int peers = __match_any_sync(0xffffffffu, bin);
      if (in && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&h[bin], (unsigned)__popc(peers));
    }
  }
  __syncthreads();
  unsigned int* g = hist + ((long long)pass * gridDim.y + b) * 512;
  for (int t = threadIdx.x; t < 512; t += blockDim.x)
    if (h[t]) atomicAdd(g + t, h[t]);
}

// After pass `pass`: each frame's two wanted ranks choose their digit.  After the last pass the order statistics
// are known and thread 0 writes stats[b] = (p90, scale): p90 by NumPy's _quantile / _lerp, operation for operation
// (NaN when the frame has no valid pixel, where the script computes none), then the script's scale.
__global__ void hs_pick_kernel(int pass, int B, const unsigned long long* __restrict__ counts,
                               const unsigned int* __restrict__ hist, unsigned long long* __restrict__ sel,
                               double scale_num, double* __restrict__ stats) {
  const int b = blockIdx.x, r = threadIdx.x;
  const unsigned long long n = counts[2 * b], n_nan = counts[2 * b + 1];
  // (n - 1) * 0.9 in fp64; previous = floor, or -1 (the last element) when at or past n - 1 (n == 1)
  const double v = __dmul_rn((double)(long long)(n - 1), 0.9);
  const bool above = v >= (double)(long long)(n - 1);
  const double prev = above ? -1.0 : floor(v);
  if (n != 0 && n_nan == 0) {
    if (pass == 0) {
      sel[4 * b + r] = 0ull;
      sel[4 * b + 2 + r] = above ? n - 1 : (unsigned long long)prev + r;
    }
    const unsigned int* h = hist + ((long long)pass * B + b) * 512 + r * 256;
    unsigned long long below = 0, want = sel[4 * b + 2 + r];
    int dig = 255;
    for (int j = 0; j < 256; ++j) {
      if (want < below + h[j]) { dig = j; break; }
      below += h[j];
    }
    sel[4 * b + 2 + r] = want - below;
    sel[4 * b + r] |= (unsigned long long)dig << (56 - 8 * pass);
  }
  __syncthreads();
  if (pass != kHsPasses - 1 || r != 0) return;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  double s, p90 = nan;
  if (n == 0) {
    s = 1.0;
  } else {
    if (n_nan == 0) {
      const double a = hs_value(sel[4 * b]), c = hs_value(sel[4 * b + 1]);
      const double gamma = __dsub_rn(v, prev);
      const double diff = __dsub_rn(c, a);
      p90 = __dadd_rn(a, __dmul_rn(diff, gamma));
      if (gamma >= 0.5) p90 = __dsub_rn(c, __dmul_rn(diff, __dsub_rn(1.0, gamma)));
    }
    s = p90 < 1e-4 ? 0.0 : __ddiv_rn(scale_num, p90);
  }
  stats[2 * b] = p90;
  stats[2 * b + 1] = s;
}

// Per pixel: the tone-mapped B, G, R bytes and the uint16 plane depth in millimetres.
template <typename TR, typename TD>
__global__ void hs_frame_kernel(const TR* __restrict__ rgb, const TD* __restrict__ dist, const int* __restrict__ eid,
                                int H, int W, double focal, const double* __restrict__ stats,
                                unsigned char* __restrict__ bgr, unsigned short* __restrict__ depth) {
  const int b = blockIdx.y;
  const long long HW = (long long)H * W;
  const double s = stats[2 * b + 1];
  const float ff = __double2float_rn(focal), fz = __fmul_rn(ff, ff);
  const double x0 = __dadd_rn(-0.5 * W, 0.5), y0 = __dadd_rn(-0.5 * H, 0.5);   // np.linspace's start
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    const long long g = (long long)b * HW + i;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double t = __dmul_rn(s, hs_load(rgb, 3 * g + c));
      bgr[3 * g + 2 - c] = hs_tone(isnan(t) ? t : (t > 0.0 ? t : 0.0));
    }
    // dist_2_depth: the float32 image-plane point (x, y, f), its fp32 norm, then fp64 distance / norm * f
    const float px = (float)__dadd_rn((double)(i % W), x0), py = (float)__dadd_rn((double)(i / W), y0);
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), fz));
    const double d = eid[g] != -1 ? __dmul_rn(__ddiv_rn(hs_load(dist, g), (double)nrm), focal) : 0.0;
    depth[g] = (unsigned short)trunc_wrap(__dmul_rn(d, 1000.0));
  }
}

// p_out[i] = the power hs_tone uses for m = x[i] and level_out[i] its uint8 level
__global__ void debug_hypersim_pow_kernel(const double* __restrict__ x, long long n, int force_slow,
                                          double* __restrict__ p_out, unsigned char* __restrict__ level_out,
                                          unsigned int* __restrict__ slow_count) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    bool slow = false;
    double p;
    level_out[i] = hs_tone(x[i], force_slow != 0, &slow, &p);
    p_out[i] = p;
    if (slow && slow_count) atomicAdd(slow_count, 1u);
  }
}

// workspace: keys [B][HW] | counts [B][2] | sel [B][4] | stats [B][2] (p90, scale) | hist [passes][B][2][256]
static long long hs_workspace_bytes(int B, long long HW) {
  return (long long)B * (HW * 8 + 2 * 8 + 4 * 8 + 2 * 8 + kHsPasses * 512 * 4);
}

template <typename TR, typename TD>
static int hs_launch(const void* rgb, const void* dist, const int* eid, int B, int H, int W, double focal,
                     double scale_num, unsigned char* bgr, unsigned short* depth, int* err, double* stats_out,
                     void* ws, cudaStream_t st) {
  const long long HW = (long long)H * W;
  unsigned long long* keys = (unsigned long long*)ws;
  unsigned long long* counts = keys + (long long)B * HW;
  unsigned long long* sel = counts + 2 * B;
  double* stats = (double*)(sel + 4 * B);
  unsigned int* hist = (unsigned int*)(stats + 2 * B);
  cudaError_t e = cudaMemsetAsync(counts, 0, (size_t)B * 2 * 8, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(hist, 0, (size_t)B * kHsPasses * 512 * 4, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(err, 0, (size_t)B * sizeof(int), st);
  if (e != cudaSuccess) {
    set_last_error("b200_data_hypersim_frames: memset: %s", cudaGetErrorString(e));
    return (int)e;
  }
  hs_keys_kernel<TR><<<dim3(data_grid(HW), B), kDataThreads, 0, st>>>((const TR*)rgb, eid, HW, keys, counts, err);
  B200_CHECK_LAUNCH("hs_keys_kernel");
  const long long ctas = (HW + kHsHistThreads * 16 - 1) / (kHsHistThreads * 16);
  const unsigned hist_grid = (unsigned)(ctas < 1 ? 1 : (ctas > kHsHistCtas ? kHsHistCtas : ctas));
  for (int pass = 0; pass < kHsPasses; ++pass) {
    hs_hist_kernel<<<dim3(hist_grid, B), kHsHistThreads, 0, st>>>(keys, HW, pass, counts, sel, hist);
    B200_CHECK_LAUNCH("hs_hist_kernel");
    hs_pick_kernel<<<B, 2, 0, st>>>(pass, B, counts, hist, sel, scale_num, stats);
    B200_CHECK_LAUNCH("hs_pick_kernel");
  }
  hs_frame_kernel<TR, TD><<<dim3(data_grid(HW), B), kDataThreads, 0, st>>>((const TR*)rgb, (const TD*)dist, eid, H, W,
                                                                          focal, stats, bgr, depth);
  B200_CHECK_LAUNCH("hs_frame_kernel");
  if (stats_out) {
    e = cudaMemcpyAsync(stats_out, stats, (size_t)B * 2 * sizeof(double), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) {
      set_last_error("b200_data_hypersim_frames: stats copy: %s", cudaGetErrorString(e));
      return (int)e;
    }
  }
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_debug_pow_e32_neg(const float* x, long long n, int force_slow, float* out,
                                      unsigned int* slow_count, void* stream) {
  B200_CHECK_ARG(x && out, "b200_debug_pow_e32_neg: null pointer");
  B200_CHECK_ARG(n >= 1, "b200_debug_pow_e32_neg: n=%lld", n);
  debug_pow_e32_neg_kernel<<<data_grid(n), kDataThreads, 0, (cudaStream_t)stream>>>(x, n, force_slow, out, slow_count);
  B200_CHECK_LAUNCH("debug_pow_e32_neg_kernel");
  return 0;
}

extern "C" long long b200_data_hypersim_workspace_bytes(int B, int H, int W) {
  return (B >= 1 && H >= 1 && W >= 1) ? hs_workspace_bytes(B, (long long)H * W) : -1;
}

extern "C" int b200_data_hypersim_frames(const void* rgb, int rgb_half, const void* dist, int dist_half,
                                         const int* entity_id, int B, int H, int W, double focal, double scale_num,
                                         unsigned char* bgr, unsigned short* depth_mm, int* error_flag,
                                         double* stats_out, void* workspace, long long workspace_bytes,
                                         void* stream) {
  B200_CHECK_ARG(rgb && dist && entity_id && bgr && depth_mm && error_flag && workspace,
                 "b200_data_hypersim_frames: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && H < (1 << 23) && W < (1 << 23) &&
                     (long long)H * W < (1LL << 40),
                 "b200_data_hypersim_frames: bad shape B=%d H=%d W=%d", B, H, W);
  B200_CHECK_ARG(isfinite(focal) && isfinite((float)focal), "b200_data_hypersim_frames: non-finite focal length");
  B200_CHECK_ARG(workspace_bytes >= hs_workspace_bytes(B, (long long)H * W),
                 "b200_data_hypersim_frames: workspace of %lld bytes, need %lld", workspace_bytes,
                 hs_workspace_bytes(B, (long long)H * W));
  B200_CHECK_ARG(((uintptr_t)workspace & 7) == 0, "b200_data_hypersim_frames: workspace not 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (rgb_half && dist_half)
    return hs_launch<__half, __half>(rgb, dist, entity_id, B, H, W, focal, scale_num, bgr, depth_mm, error_flag,
                                     stats_out, workspace, st);
  if (rgb_half)
    return hs_launch<__half, float>(rgb, dist, entity_id, B, H, W, focal, scale_num, bgr, depth_mm, error_flag,
                                    stats_out, workspace, st);
  if (dist_half)
    return hs_launch<float, __half>(rgb, dist, entity_id, B, H, W, focal, scale_num, bgr, depth_mm, error_flag,
                                    stats_out, workspace, st);
  return hs_launch<float, float>(rgb, dist, entity_id, B, H, W, focal, scale_num, bgr, depth_mm, error_flag, stats_out,
                                 workspace, st);
}

extern "C" int b200_debug_hypersim_pow(const double* x, long long n, int force_slow, double* p_out,
                                       unsigned char* level_out, unsigned int* slow_count, void* stream) {
  B200_CHECK_ARG(x && p_out && level_out, "b200_debug_hypersim_pow: null pointer");
  B200_CHECK_ARG(n >= 1, "b200_debug_hypersim_pow: n=%lld", n);
  debug_hypersim_pow_kernel<<<data_grid(n), kDataThreads, 0, (cudaStream_t)stream>>>(x, n, force_slow, p_out, level_out,
                                                                                   slow_count);
  B200_CHECK_LAUNCH("debug_hypersim_pow_kernel");
  return 0;
}

extern "C" int b200_data_vkitti_normals(const unsigned short* depth_cm, int B, int H, int W, float fx, float fy,
                                        float u0, float v0, unsigned short* out, void* stream) {
  B200_CHECK_ARG(depth_cm && out, "b200_data_vkitti_normals: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && H >= 3 && W >= 3 && (long long)H * W < (1LL << 40),
                 "b200_data_vkitti_normals: bad shape B=%d H=%d W=%d (H, W >= 3)", B, H, W);
  B200_CHECK_ARG(isfinite(fx) && isfinite(fy) && isfinite(u0) && isfinite(v0),
                 "b200_data_vkitti_normals: non-finite intrinsics");
  const dim3 grid((W + kNrmTW - 1) / kNrmTW, (H + kNrmTH - 1) / kNrmTH, B);
  B200_CHECK_ARG(grid.y <= 65535, "b200_data_vkitti_normals: H=%d too large", H);
  data_vkitti_normals_kernel<<<grid, dim3(kNrmTW, kNrmTH), 0, (cudaStream_t)stream>>>(depth_cm, H, W, fx, fy, u0, v0,
                                                                                      out);
  B200_CHECK_LAUNCH("data_vkitti_normals_kernel");
  return 0;
}

extern "C" int b200_data_hypersim_source(const unsigned short* depth_mm, const unsigned char* normal,
                                         const unsigned char* flip, int B, int H, int W, const double* inv_k,
                                         float* depth_m, unsigned char* normal_out, void* stream) {
  B200_CHECK_ARG(depth_mm && normal && inv_k && depth_m && normal_out, "b200_data_hypersim_source: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && H >= 1 && W >= 1, "b200_data_hypersim_source: bad shape B=%d H=%d W=%d", B, H,
                 W);
  InvK k;
  for (int i = 0; i < 9; ++i) k.m[i] = inv_k[i];
  data_hypersim_source_kernel<<<dim3(data_grid((long long)H * W), B), kDataThreads, 0, (cudaStream_t)stream>>>(
      depth_mm, normal, flip, H, W, k, depth_m, normal_out);
  B200_CHECK_LAUNCH("data_hypersim_source_kernel");
  return 0;
}

extern "C" int b200_data_resize_u8(const unsigned char* src, int B, int H, int W, int C, int OH, int OW,
                                   const int* xmin, const int* xk, int xks, const int* ymin, const int* yk, int yks,
                                   const unsigned char* flip, unsigned char* tmp, unsigned char* dst, void* stream) {
  B200_CHECK_ARG(src && xmin && xk && ymin && yk && tmp && dst, "b200_data_resize_u8: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && C >= 1 && OH >= 1 && OW >= 1 && xks >= 1 && yks >= 1,
                 "b200_data_resize_u8: bad shape B=%d H=%d W=%d C=%d OH=%d OW=%d", B, H, W, C, OH, OW);
  cudaStream_t st = (cudaStream_t)stream;
  data_resize_h_kernel<<<dim3(data_grid((long long)H * OW * C), B), kDataThreads, 0, st>>>(src, H, W, C, OW, xmin, xk,
                                                                                           xks, flip, tmp);
  B200_CHECK_LAUNCH("data_resize_h_kernel");
  data_resize_v_kernel<<<dim3(data_grid((long long)OH * OW * C), B), kDataThreads, 0, st>>>(tmp, H, OW, C, OH, ymin, yk,
                                                                                            yks, dst);
  B200_CHECK_LAUNCH("data_resize_v_kernel");
  return 0;
}

extern "C" int b200_data_depth_gather(const float* src_m, const unsigned short* src_cm, int B, int H, int W, int OH,
                                      int OW, const int* rows, const int* cols, const unsigned char* flip, float* dst,
                                      void* stream) {
  B200_CHECK_ARG((src_m == nullptr) != (src_cm == nullptr), "b200_data_depth_gather: exactly one of src_m / src_cm");
  B200_CHECK_ARG(rows && cols && dst, "b200_data_depth_gather: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && OH >= 1 && OW >= 1,
                 "b200_data_depth_gather: bad shape B=%d H=%d W=%d OH=%d OW=%d", B, H, W, OH, OW);
  data_depth_gather_kernel<<<dim3(data_grid((long long)OH * OW), B), kDataThreads, 0, (cudaStream_t)stream>>>(
      src_m, src_cm, H, W, OH, OW, rows, cols, flip, dst);
  B200_CHECK_LAUNCH("data_depth_gather_kernel");
  return 0;
}

extern "C" int b200_data_depth_range(const float* depth, int B, long long HW, float near_plane, float far_plane,
                                     float* range, int* flag, void* stream) {
  B200_CHECK_ARG(depth && range && flag, "b200_data_depth_range: null pointer");
  B200_CHECK_ARG(B >= 1 && HW >= 1 && HW < (1LL << 32), "b200_data_depth_range: bad shape B=%d HW=%lld", B, HW);
  B200_CHECK_ARG(near_plane >= 0.f, "b200_data_depth_range: near_plane must be >= 0");
  data_depth_range_kernel<<<B, kRangeThreads, 0, (cudaStream_t)stream>>>(depth, HW, near_plane, far_plane, range, flag);
  B200_CHECK_LAUNCH("data_depth_range_kernel");
  return 0;
}

extern "C" int b200_data_finalise(const unsigned char* rgb, const unsigned char* normal, int B, int H, int W, int top,
                                  int left, const unsigned char* flip, const float* depth, int OH, int OW,
                                  float near_plane, float far_plane, const float* range, const int* flag,
                                  float* rgb_out, float* depth_out, float* metric_out, float* normal_out,
                                  unsigned char* mask_out, void* stream) {
  B200_CHECK_ARG(rgb && normal && depth && range && flag && rgb_out && depth_out && metric_out && normal_out && mask_out,
                 "b200_data_finalise: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && OH >= 1 && OW >= 1 && top >= 0 && left >= 0 && top + OH <= H &&
                     left + OW <= W,
                 "b200_data_finalise: bad shape B=%d H=%d W=%d top=%d left=%d OH=%d OW=%d", B, H, W, top, left, OH, OW);
  data_finalise_kernel<<<dim3(data_grid((long long)OH * OW), B), kDataThreads, 0, (cudaStream_t)stream>>>(
      rgb, normal, H, W, top, left, flip, depth, OH, OW, near_plane, far_plane, range, flag, rgb_out, depth_out,
      metric_out, normal_out, mask_out);
  B200_CHECK_LAUNCH("data_finalise_kernel");
  return 0;
}
