// Training-batch preparation on the device (DESIGN.md §3 "Training inputs"): the per-sample transforms of
// training/dataloaders/load.py applied to decoded uint8 / uint16 images.
//   b200_data_hypersim_source  depth mm -> m and the normal orientation fix (load.py:217-238), flip correction of x
//   b200_data_resize_u8        Pillow's two-pass fixed-point BILINEAR resize (transforms.Resize on a PIL image)
//   b200_data_depth_gather     Pillow's NEAREST resize of the depth, or the KITTI benchmark crop; the flip folded in
//   b200_data_depth_range      torch.quantile(valid, 0.02 / 0.98) per image (segmented radix select)
//   b200_data_finalise         load.py:248-281 / :343-376 per output pixel
// All HBM-bound.  Per-pixel arithmetic the reference does in fp32 / fp64 is written with explicitly rounded intrinsics
// so nvcc cannot contract it into FMAs: the outputs are bitwise those of the reference.  Nothing syncs the host.
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

}  // namespace b200

using namespace b200;

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
