// Backward-pass kernels of the fine-tuning step (SURVEY.md §8 row a10; reference: training/train.py:545-566,
// `accelerator.backward(loss)` through the UNet and the frozen VAE decoder).  Everything here is HBM-bound
// streaming / reduction work; the GEMM-shaped halves of the backward pass (conv dgrad, conv/linear wgrad,
// attention S/dP/dQ/dK/dV products) run on the wgmma kernels in gemm_conv.cu with re-packed or transposed
// operands (backward_packing.py / backward.py).
//
//   gather_planar       NHWC -> [C][pixels] transpose with an optional tap shift / stride / nearest-2x source map:
//                       produces the K-major operands of the weight-gradient GEMMs (K = pixels)
//   col_sum             bias gradients (and the split-K sums of the weight gradients)
//   gn_mean_rstd        group statistics from the forward's fp64 group sums or per-channel sums
//   gn_bwd_sums/apply   GroupNorm(+SiLU) backward, two streaming passes
//   layer_norm_bwd      one warp per row, d_gamma/d_beta through per-warp shared-memory rows
//   softmax_bwd_rows    dS = scale * P o (dP - rowsum(dP o P))
//   act_bwd / geglu_bwd SiLU / exact-GELU / GEGLU derivatives
//
// Reductions across pixels or rows (col_sum, gn_bwd_sums, layer_norm_bwd's d_gamma / d_beta, the loss moments) give
// one output slot to one thread-block cluster (cluster_reduce.cuh): each CTA reduces a fixed share in a fixed order
// (thread-sequential, then a fixed xor butterfly or a fixed row order in shared memory, then warps in index order) and
// rank 0 adds the CTAs' partials in rank order with one plain read-modify-write.  No floating-point atomics; grids and
// cluster sizes depend only on the problem size, never on the SM count, so a backward pass repeats bit for bit.
#include "cluster_reduce.cuh"
#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

// ----------------------------------------------------------------------------------------------- helpers
__device__ __forceinline__ void bw_load8(const __half* p, float* v) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __half22float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void bw_load8(const float* p, float* v) {
  float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void bw_store8(__half* p, const float* v) {
  __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
  __half2 h2 = __floats2half2_rn(v[4], v[5]), h3 = __floats2half2_rn(v[6], v[7]);
  uint4 u;
  u.x = *reinterpret_cast<uint32_t*>(&h0);
  u.y = *reinterpret_cast<uint32_t*>(&h1);
  u.z = *reinterpret_cast<uint32_t*>(&h2);
  u.w = *reinterpret_cast<uint32_t*>(&h3);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void bw_store8(float* p, const float* v) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ float bw_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(float v) { return v; }

__device__ __forceinline__ float silu_grad(float z) {
  const float s = 1.0f / (1.0f + __expf(-z));
  return s * (1.0f + z * (1.0f - s));
}
__device__ __forceinline__ float gelu_fwd(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// ------------------------------------------------------------------------------------------ gather_planar
// out[c][q] (row stride ldo, q = (n*Ho + o)*Wo + p) = x[n][(stride*o + oy) / up][(stride*p + ox) / up][c] (pixel stride ldx),
// zero when the source row/column is outside [0, up*H) x [0, up*W) or q >= P (q runs to Ppad).
// grid (ceil(Ppad/32), ceil(C/32)), block (32, 8); 32x32 tile through shared memory, coalesced both sides.
template <typename T>
__global__ void gather_planar_kernel(const T* __restrict__ x, long long ldx, int H, int W, int C, int Ho, int Wo, int stride,
                                     int up, int oy, int ox, long long P, long long Ppad,
                                     __half* __restrict__ out, long long ldo) {
  __shared__ float tile[32][33];
  const long long q0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += 8) {
    const long long q = q0 + i;
    const int c = c0 + tx;
    float v = 0.f;
    if (q < P && c < C) {
      const int p = (int)(q % Wo);
      const long long t = q / Wo;
      const int o = (int)(t % Ho);
      const long long n = t / Ho;
      const int yy = stride * o + oy, xx = stride * p + ox;
      if (yy >= 0 && yy < up * H && xx >= 0 && xx < up * W) {
        const int sy = yy / up, sx = xx / up;
        v = to_f(x[((n * H + sy) * W + sx) * ldx + c]);
      }
    }
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i;
    const long long q = q0 + tx;
    if (c < C && q < Ppad) out[(long long)c * ldo + q] = __float2half_rn(tile[tx][i]);
  }
}

// ------------------------------------------------------------------------------------------------ rowdot
// delta[b][h][t] = sum_{d < D} a[b][t][h*D + d] * c[b][t][h*D + d]   (fp16 in, fp32 accumulate / out).
// One warp per (t, h): lane l reads the __half2 at d = 64 j + 2 l of each 64-column chunk j that reaches it.
template <int D>
__global__ void rowdot_heads_kernel(const __half* __restrict__ a, long long a_bs, long long a_ls,
                                    const __half* __restrict__ c, long long c_bs, long long c_ls, int L, int heads,
                                    float* __restrict__ out) {
  const int b = blockIdx.z, h = blockIdx.y;
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= L) return;
  const int lane = threadIdx.x & 31;
  const __half* ar = a + (long long)b * a_bs + (long long)t * a_ls + h * D;
  const __half* cr = c + (long long)b * c_bs + (long long)t * c_ls + h * D;
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < (D + 63) / 64; ++j) {
    const int d = 64 * j + 2 * lane;
    if (d < D) {
      const float2 xf = __half22float2(*reinterpret_cast<const __half2*>(ar + d));
      const float2 yf = __half22float2(*reinterpret_cast<const __half2*>(cr + d));
      const float v = fmaf(xf.x, yf.x, xf.y * yf.y);
      s = j == 0 ? v : s + v;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[((long long)b * heads + h) * L + t] = s;
}

// ------------------------------------------------------------------------------------------------ col_sum
// out[c] += sum over rows of x[row][c];  grid (ceil(C/32), R), block (32, Y), cluster (1, R): one cluster per 32-column
// slice.  CTA y of the cluster sums a fixed contiguous share of the rows: thread (c, j) every Y-th row from j, the Y
// row-threads in order, then rank 0 adds the R CTAs in rank order.  Y = 8, or 32 when the rows span a cluster.
template <typename T>
__global__ void col_sum_kernel(const T* __restrict__ x, long long rows, int C, long long ld, float* __restrict__ out) {
  __shared__ float red[32][33];
  const int Y = blockDim.y;
  const int c0 = blockIdx.x * 32;
  const int c = c0 + threadIdx.x;
  long long r0, r1;
  cluster_share(rows, gridDim.y, blockIdx.y, r0, r1);
  // one CTA per slot (few rows, e.g. the split-K partials of a weight gradient): the CTA is short, so the old value
  // of its output is fetched before the loads instead of after the sum
  const bool alone = gridDim.y == 1;
  const float old = alone && threadIdx.y == 0 && c < C ? out[c] : 0.f;
  float acc = 0.f;
  if (c < C) {
#pragma unroll 4
    for (long long r = r0 + threadIdx.y; r < r1; r += Y) acc += to_f(x[r * ld + c]);
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0) {
    float s = red[0][threadIdx.x];
    for (int i = 1; i < Y; ++i) s += red[i][threadIdx.x];
    if (alone) {
      if (c < C) out[c] = old + s;
      return;
    }
    red[0][threadIdx.x] = s;
  }
  if (alone) return;
  cluster_add_partials(&red[0][0], min(32, C - c0), [&](int k) { return out + c0 + k; });
}

// ------------------------------------------------------------------------------------------ GroupNorm bwd
// mr[n][g] = (mean, rstd) from the forward's statistics: fp64 group sums, or per-channel fp32 sums of the one
// or two (channel-concatenated) inputs written by the producing kernels' epilogues.
__global__ void gn_mean_rstd_kernel(const double* __restrict__ sums, const double* __restrict__ cs1, int C1,
                                    const double* __restrict__ cs2, int C2, int NB, int HW, int groups, float eps,
                                    float* __restrict__ mr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NB * groups) return;
  const int n = i / groups, g = i % groups;
  const int C = C1 + C2, cg = C / groups;
  double su = 0.0, sq = 0.0;
  if (sums) {
    su = sums[2 * (long long)i];
    sq = sums[2 * (long long)i + 1];
  } else {
    for (int c = g * cg; c < (g + 1) * cg; ++c) {
      const double* src = c < C1 ? cs1 + ((long long)n * C1 + c) * 2 : cs2 + ((long long)n * C2 + (c - C1)) * 2;
      su += (double)src[0];
      sq += (double)src[1];
    }
  }
  const double cnt = (double)HW * cg;
  const double mean = su / cnt;
  double var = sq / cnt - mean * mean;
  if (var < 0) var = 0;
  mr[2 * (long long)i] = (float)mean;
  mr[2 * (long long)i + 1] = (float)(1.0 / sqrt(var + (double)eps));
}

// Pass 1: S[n][c_off + c] += (sum dz, sum dz * xhat) over the pixels, dz = dy * silu'(gamma*xhat + beta).
// x: [NB][HW][Cx] (one of the concatenated inputs, channels c_off.. of the normalised tensor); dy: fp16 [NB][HW][Ctot].
// grid (R, ceil(Cx/16), NB), cluster (R): one cluster per (image, 16-channel slice); block kGnSumsThreads, thread t
// owns the 8-channel vector t % 2 of the slice and every (kGnSumsThreads/2)-th pixel of its CTA's contiguous share.
// Per-thread sums -> xor butterfly over the lanes of the same vector -> warps in order -> ranks in order.
constexpr int kGnSumsThreads = 512;
template <typename T>
__global__ void __launch_bounds__(kGnSumsThreads) gn_bwd_sums_kernel(const T* __restrict__ x, int Cx, int c_off,
                                                                    int Ctot, const __half* __restrict__ dy, int HW,
                                                                    int groups, const float* __restrict__ mr,
                                                                    const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta, int silu,
                                                                    float* __restrict__ S) {
  constexpr int VS = 2, kWarps = kGnSumsThreads / 32, rpb = kGnSumsThreads / VS;
  __shared__ float red[kWarps][VS * 16];
  __shared__ float part[VS * 16];
  const int n = blockIdx.z;
  const int V = Cx / 8;
  const int vl = threadIdx.x % VS, r = threadIdx.x / VS;
  const int vg = blockIdx.y * VS + vl;                        // vector index within x's channels
  const int cpg = Ctot / groups;
  float s1[8], s2[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s1[e] = s2[e] = 0.f;
  if (vg < V) {
    const int c0 = vg * 8;
    float a[8], b[8], rs[8], ms[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = c_off + c0 + e;
      const int g = c / cpg;
      const float mean = mr[((long long)n * groups + g) * 2], rstd = mr[((long long)n * groups + g) * 2 + 1];
      rs[e] = rstd;
      ms[e] = -mean * rstd;
      a[e] = rstd * gamma[c];
      b[e] = beta[c] - mean * a[e];
    }
    const T* xb = x + (long long)n * HW * Cx + c0;
    const __half* db = dy + (long long)n * HW * Ctot + c_off + c0;
    long long p0, p1;
    cluster_share(HW, gridDim.x, blockIdx.x, p0, p1);
#pragma unroll 2
    for (long long p = p0 + r; p < p1; p += rpb) {
      float f[8], d[8];
      bw_load8(xb + p * Cx, f);
      bw_load8(db + p * Ctot, d);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float dz = silu ? d[e] * silu_grad(f[e] * a[e] + b[e]) : d[e];
        s1[e] += dz;
        s2[e] += dz * (f[e] * rs[e] + ms[e]);
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e)
#pragma unroll
    for (int o = 16; o >= VS; o >>= 1) {
      s1[e] += __shfl_xor_sync(0xffffffffu, s1[e], o);
      s2[e] += __shfl_xor_sync(0xffffffffu, s2[e], o);
    }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane < VS) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {                              // channel j = 8 lane + e of the slice at [2 j + {0, 1}]
      red[warp][(8 * lane + e) * 2 + 0] = s1[e];
      red[warp][(8 * lane + e) * 2 + 1] = s2[e];
    }
  }
  __syncthreads();
  if (threadIdx.x < VS * 16) {
    float t = red[0][threadIdx.x];
    for (int w = 1; w < kWarps; ++w) t += red[w][threadIdx.x];
    part[threadIdx.x] = t;
  }
  const int cs0 = blockIdx.y * VS * 8;                         // first channel of the slice within x
  cluster_add_partials(part, 2 * min(VS * 8, Cx - cs0),
                       [&](int k) { return S + ((long long)n * Ctot + c_off + cs0) * 2 + k; });
}

// Pass 2: dx = rstd * (dz*gamma - A_g - xhat * B_g) (+ add), A_g = mean_g(gamma * dz), B_g = mean_g(gamma * dz * xhat)
// from the complete S of pass 1 (all concatenated inputs accumulated).
template <typename T, typename TO>
__global__ void gn_bwd_apply_kernel(const T* __restrict__ x, int Cx, int c_off, int Ctot,
                                    const __half* __restrict__ dy, int HW, int groups, int pix_per_cta,
                                    const float* __restrict__ mr, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, int silu, const float* __restrict__ S,
                                    const TO* add, TO* dx) {
  extern __shared__ float sm[];   // gA[groups], gB[groups]
  const int V = Cx / 8;
  const int n = blockIdx.y;
  const int cpg = Ctot / groups;
  const float inv_m = 1.0f / ((float)HW * (float)cpg);
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float A = 0.f, B = 0.f;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      A += gamma[c] * S[((long long)n * Ctot + c) * 2 + 0];
      B += gamma[c] * S[((long long)n * Ctot + c) * 2 + 1];
    }
    sm[g] = A * inv_m;
    sm[groups + g] = B * inv_m;
  }
  __syncthreads();
  const int rpb = blockDim.x / V;
  const int v = threadIdx.x % V;
  const int r = threadIdx.x / V;
  if (r >= rpb) return;
  const int c0 = v * 8;
  float a[8], b[8], rs[8], ms[8], k0[8], k1[8], k2[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = c_off + c0 + e;
    const int g = c / cpg;
    const float mean = mr[((long long)n * groups + g) * 2], rstd = mr[((long long)n * groups + g) * 2 + 1];
    rs[e] = rstd;
    ms[e] = -mean * rstd;
    a[e] = rstd * gamma[c];
    b[e] = beta[c] - mean * a[e];
    k0[e] = rstd * gamma[c];
    k1[e] = rstd * sm[g];
    k2[e] = rstd * sm[groups + g];
  }
  const T* xb = x + (long long)n * HW * Cx + c0;
  const __half* db = dy + (long long)n * HW * Ctot + c_off + c0;
  TO* ob = dx + (long long)n * HW * Cx + c0;
  const TO* ab = add ? add + (long long)n * HW * Cx + c0 : nullptr;
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  for (int p = p0 + r; p < p1; p += rpb) {
    float f[8], d[8], o[8];
    bw_load8(xb + (long long)p * Cx, f);
    bw_load8(db + (long long)p * Ctot, d);
    if (ab) bw_load8(ab + (long long)p * Cx, o);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float dz = silu ? d[e] * silu_grad(f[e] * a[e] + b[e]) : d[e];
      const float g = dz * k0[e] - k1[e] - (f[e] * rs[e] + ms[e]) * k2[e];
      o[e] = ab ? o[e] + g : g;
    }
    bw_store8(ob + (long long)p * Cx, o);
  }
}

// ------------------------------------------------------------------------------------------ LayerNorm bwd
// one warp per row; C <= 2048, C % 8 == 0.  grid (R), cluster (R): ONE cluster owns d_gamma / d_beta.  CTA rank k
// takes a fixed contiguous share of the rows, its warp w every wpb-th row of that share from w; lane l owns the
// columns of vectors l + 32 i and adds their d_gamma / d_beta terms to the warp's own shared-memory row in row order.
// The warps' rows are then summed in warp order and the CTAs' in rank order.
template <typename T, typename TO, int kMaxV>
__global__ void __launch_bounds__(kMaxV <= 2 ? 1024 : 512) layer_norm_bwd_kernel(const T* __restrict__ x, long long rows, int C,
                                      const float* __restrict__ gamma, const __half* __restrict__ dy, float eps,
                                      const TO* add, TO* dx,
                                      float* __restrict__ dgamma, float* __restrict__ dbeta) {
  extern __shared__ float sm[];   // [wpb][2C] per-warp (dgamma, dbeta) rows, then the CTA's [2C] partial
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int V = C / 8;                                       // <= 32 kMaxV vectors of 8 per row
  for (int i = threadIdx.x; i < wpb * 2 * C; i += blockDim.x) sm[i] = 0.f;
  __syncthreads();
  float* wacc = sm + (threadIdx.x >> 5) * 2 * C;
  long long r0, r1;
  cluster_share(rows, gridDim.x, blockIdx.x, r0, r1);
  for (long long row = r0 + (threadIdx.x >> 5); row < r1; row += wpb) {
    float f[kMaxV][8];
    float s = 0.f;
    const T* xr = x + row * C;
    const __half* dr = dy + row * C;
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int v = lane + 32 * i;
      if (v < V) {
        bw_load8(xr + v * 8, f[i]);
#pragma unroll
        for (int e = 0; e < 8; ++e) s += f[i][e];
      }
    }
    const float mean = bw_warp_sum(s) / C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int v = lane + 32 * i;
      if (v < V) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float d = f[i][e] - mean; q += d * d; }
      }
    }
    const float rstd = rsqrtf(bw_warp_sum(q) / C + eps);
    // xhat in place; m1 = mean(dy*gamma), m2 = mean(dy*gamma*xhat)
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int v = lane + 32 * i;
      if (v < V) {
        float d[8], g[8];
        bw_load8(dr + v * 8, d);
        bw_load8(gamma + v * 8, g);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          f[i][e] = (f[i][e] - mean) * rstd;
          const float t = d[e] * g[e];
          m1 += t;
          m2 += t * f[i][e];
        }
      }
    }
    m1 = bw_warp_sum(m1) / C;
    m2 = bw_warp_sum(m2) / C;
#pragma unroll
    for (int i = 0; i < kMaxV; ++i) {
      const int v = lane + 32 * i;
      if (v < V) {
        float d[8], g[8], o[8];
        bw_load8(dr + v * 8, d);
        bw_load8(gamma + v * 8, g);
        if (add) bw_load8(add + row * C + v * 8, o);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float gx = rstd * (d[e] * g[e] - m1 - f[i][e] * m2);
          o[e] = add ? o[e] + gx : gx;
          wacc[v * 8 + e] += d[e] * f[i][e];
          wacc[C + v * 8 + e] += d[e];
        }
        bw_store8(dx + row * C + v * 8, o);
      }
    }
  }
  __syncthreads();
  float* part = sm + wpb * 2 * C;
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    float t = sm[i];
    for (int w = 1; w < wpb; ++w) t += sm[w * 2 * C + i];
    part[i] = t;
  }
  cluster_add_partials(part, 2 * C, [&](int k) { return k < C ? dgamma + k : dbeta + (k - C); });
}

// ------------------------------------------------------------------------------------------- softmax bwd
// one CTA per row: dS[j] = scale * P[j] * (dP[j] - sum_k dP[k] P[k]);  P, dS fp16 (row stride ldp), dP fp32 (ldd).
__global__ void softmax_bwd_rows_kernel(const __half* __restrict__ P, long long ldp, const float* __restrict__ dP,
                                        long long ldd, __half* __restrict__ dS, int cols, float scale) {
  __shared__ float red[32];
  const __half* p = P + (long long)blockIdx.x * ldp;
  const float* d = dP + (long long)blockIdx.x * ldd;
  __half* o = dS + (long long)blockIdx.x * ldp;
  const int tid = threadIdx.x, nw = blockDim.x >> 5;
  float dot = 0.f;
  for (int c = tid; c < cols; c += blockDim.x) dot += __half2float(p[c]) * d[c];
  dot = bw_warp_sum(dot);
  if ((tid & 31) == 0) red[tid >> 5] = dot;
  __syncthreads();
  dot = 0.f;
  for (int i = 0; i < nw; ++i) dot += red[i];
  for (int c = tid; c < cols; c += blockDim.x) o[c] = __float2half_rn(scale * __half2float(p[c]) * (d[c] - dot));
}

// -------------------------------------------------------------------------------------------- activations
// mode 1 SiLU, 3 exact GELU: dx = dy * act'(x)
__global__ void act_bwd_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, long long n, int mode,
                               __half* __restrict__ dx) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float xv = __half2float(x[i]), d = __half2float(dy[i]);
    dx[i] = __float2half_rn(d * (mode == 1 ? silu_grad(xv) : gelu_grad(xv)));
  }
}
// GEGLU y = h * gelu(g): dh = dy * gelu(g), dg = dy * h * gelu'(g); h/g/dh/dg rows may be strided (two halves of
// one [rows][2*inner] projection), dy is [rows][inner] contiguous.
__global__ void geglu_bwd_kernel(const __half* __restrict__ h, const __half* __restrict__ g, long long ldhg,
                                 const __half* __restrict__ dy, long long rows, int inner,
                                 __half* __restrict__ dh, __half* __restrict__ dg, long long ldd) {
  const long long n = rows * inner;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / inner;
    const int c = (int)(i % inner);
    const float hv = __half2float(h[r * ldhg + c]), gv = __half2float(g[r * ldhg + c]), d = __half2float(dy[i]);
    dh[r * ldd + c] = __float2half_rn(d * gelu_fwd(gv));
    dg[r * ldd + c] = __float2half_rn(d * hv * gelu_grad(gv));
  }
}


// ------------------------------------------------------------------------------------------- loss backward
// Scale-and-shift-invariant L1 (training/util/loss.py:13-47) differentiated THROUGH the per-image least-squares
// (s, t), as torch.autograd does in the reference.  ws (zeroed double [7*B]): [5b..5b+4] = moments
// (sum m p p, sum m p, sum m, sum m p y, sum m y), [5B+2b..] = (sum m sgn(r), sum m sgn(r) p), r = s p + t - y.
__device__ __forceinline__ double bw_warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ void ssi_fit(const double* ws, int b, double& s, double& t, double& det) {
  const double a00 = ws[b * 5 + 0], a01 = ws[b * 5 + 1], a11 = ws[b * 5 + 2], b0 = ws[b * 5 + 3], b1 = ws[b * 5 + 4];
  det = a00 * a11 - a01 * a01;
  s = 0.0; t = 0.0;
  if (det > 0) { s = (a11 * b0 - a01 * b1) / det; t = (-a01 * b0 + a00 * b1) / det; }
}
constexpr int kLossBwdThreads = 512;
// grid (R, B), cluster (R): one cluster per image b (fixed-order sums, cluster_reduce.cuh)
__global__ void __launch_bounds__(kLossBwdThreads) ssi_bwd_moments_kernel(const float* __restrict__ pred,
                                                                          const float* __restrict__ tgt,
                                                                          const uint8_t* __restrict__ mask,
                                                                          long long HW, double* __restrict__ ws) {
  __shared__ double part[5];
  const int b = blockIdx.y;
  const float* p = pred + (long long)b * HW;
  const float* y = tgt + (long long)b * HW;
  const uint8_t* m = mask + (long long)b * HW;
  double v[5] = {0, 0, 0, 0, 0};
  long long lo, hi;
  cluster_share(HW, gridDim.x, blockIdx.x, lo, hi);
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    if (m[i]) {
      const double pv = p[i], yv = y[i];
      v[0] += pv * pv; v[1] += pv; v[2] += 1.0; v[3] += pv * yv; v[4] += yv;
    }
  }
  block_sum_fixed(v, part);
  cluster_add_partials(part, 5, [&](int k) { return ws + b * 5 + k; });
}
__global__ void __launch_bounds__(kLossBwdThreads) ssi_bwd_sign_sums_kernel(const float* __restrict__ pred,
                                                                            const float* __restrict__ tgt,
                                                                            const uint8_t* __restrict__ mask,
                                                                            long long HW, int B,
                                                                            double* __restrict__ ws) {
  __shared__ double part[2];
  const int b = blockIdx.y;
  double s, t, det;
  ssi_fit(ws, b, s, t, det);
  const float sf = (float)s, tf = (float)t;                   // the forward evaluates the residual in fp32
  const float* p = pred + (long long)b * HW;
  const float* y = tgt + (long long)b * HW;
  const uint8_t* m = mask + (long long)b * HW;
  double v[2] = {0, 0};
  long long lo, hi;
  cluster_share(HW, gridDim.x, blockIdx.x, lo, hi);
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x)
    if (m[i]) {
      const float r = sf * p[i] + tf - y[i];
      const double sg = (r > 0.f) - (r < 0.f);
      v[0] += sg; v[1] += sg * (double)p[i];
    }
  block_sum_fixed(v, part);
  cluster_add_partials(part, 2, [&](int k) { return ws + 5 * B + 2 * b + k; });
}
__global__ void ssi_bwd_grad_kernel(const float* __restrict__ pred, const float* __restrict__ tgt,
                                    const uint8_t* __restrict__ mask, long long HW, int B, const double* __restrict__ ws,
                                    const float* __restrict__ gscale, float* __restrict__ dpred) {
  const int b = blockIdx.y;
  double s, t, det;
  ssi_fit(ws, b, s, t, det);
  double N = 0;
  for (int i = 0; i < B; ++i) N += ws[i * 5 + 2];
  const double a01 = ws[b * 5 + 1], a11 = ws[b * 5 + 2], b0 = ws[b * 5 + 3], b1 = ws[b * 5 + 4];
  const double G0 = ws[5 * B + 2 * b] / N, G1 = ws[5 * B + 2 * b + 1] / N;
  const double up = (double)gscale[0];
  const float sf = (float)s, tf = (float)t;
  const float* p = pred + (long long)b * HW;
  const float* y = tgt + (long long)b * HW;
  const uint8_t* m = mask + (long long)b * HW;
  float* o = dpred + (long long)b * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    double g = 0.0;
    if (m[i] && N > 0) {
      const double pv = p[i], yv = y[i];
      const float r = sf * p[i] + tf - y[i];
      g = ((r > 0.f) - (r < 0.f)) * s / N;
      if (det > 0) {
        const double ddet = 2.0 * pv * a11 - 2.0 * a01;
        const double dns = a11 * yv - b1;
        const double dnt = -b0 - a01 * yv + 2.0 * pv * b1;
        g += (G1 * (dns - s * ddet) + G0 * (dnt - t * ddet)) / det;
      }
    }
    o[i] = (float)(up * g);
  }
}

// AngularLoss (loss.py:51-67): mean over the mask of acos(clamp(<p, y>, -1, 1)); ws (zeroed double [1]) = count.
// grid (R), cluster (R): one cluster counts the whole mask.
__global__ void __launch_bounds__(kLossBwdThreads) mask_count_kernel(const uint8_t* __restrict__ mask, long long n,
                                                                     double* __restrict__ ws) {
  __shared__ double part[1];
  double c[1] = {0};
  long long lo, hi;
  cluster_share(n, gridDim.x, blockIdx.x, lo, hi);
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) c[0] += mask[i] ? 1.0 : 0.0;
  block_sum_fixed(c, part);
  cluster_add_partials(part, 1, [&](int) { return ws; });
}
__global__ void angular_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ tgt,
                                   const uint8_t* __restrict__ mask, long long HW, const double* __restrict__ ws,
                                   const float* __restrict__ gscale, float* __restrict__ dpred) {
  const int b = blockIdx.y;
  const float* p = pred + (long long)b * 3 * HW;
  const float* y = tgt + (long long)b * 3 * HW;
  const uint8_t* m = mask + (long long)b * HW;
  float* o = dpred + (long long)b * 3 * HW;
  const float k = (float)((double)gscale[0] / ws[0]);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
    float g = 0.f;
    if (m[i]) {
      const float d = p[i] * y[i] + p[HW + i] * y[HW + i] + p[2 * HW + i] * y[2 * HW + i];
      if (d > -1.0f && d < 1.0f) g = -k * rsqrtf(1.0f - d * d);
    }
    o[i] = g * y[i];
    o[HW + i] = g * y[HW + i];
    o[2 * HW + i] = g * y[2 * HW + i];
  }
}

// decode_post training modes (train.py:532-540) backward.  mode 2: est = clamp(mean_c x, -1, 1);
// mode 3: est_c = clamp(x_c / (|x| + 1e-5), -1, 1).
__global__ void decode_post_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dout, long long HW,
                                       int mode, float* __restrict__ dx) {
  const int n = blockIdx.y;
  const float* xb = x + (long long)n * 3 * HW;
  float* ob = dx + (long long)n * 3 * HW;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    const float a = xb[p], b = xb[HW + p], c = xb[2 * HW + p];
    if (mode == 2) {
      const float m = (a + b + c) / 3.0f;
      const float g = (m >= -1.0f && m <= 1.0f) ? dout[(long long)n * HW + p] / 3.0f : 0.f;
      ob[p] = g; ob[HW + p] = g; ob[2 * HW + p] = g;
    } else {
      const float* db = dout + (long long)n * 3 * HW;
      const float nrm = sqrtf(a * a + b * b + c * c);
      const float inv = 1.0f / (nrm + 1e-5f);
      const float u0 = a * inv, u1 = b * inv, u2 = c * inv;
      const float g0 = (u0 >= -1.f && u0 <= 1.f) ? db[p] : 0.f;
      const float g1 = (u1 >= -1.f && u1 <= 1.f) ? db[HW + p] : 0.f;
      const float g2 = (u2 >= -1.f && u2 <= 1.f) ? db[2 * HW + p] : 0.f;
      // u = x / (|x| + eps):  du_c/dx_k = delta_ck * inv - x_c x_k * inv^2 / |x|
      const float dot = g0 * a + g1 * b + g2 * c;
      const float k = nrm > 0.f ? dot * inv * inv / nrm : 0.f;
      ob[p] = g0 * inv - a * k;
      ob[HW + p] = g1 * inv - b * k;
      ob[2 * HW + p] = g2 * inv - c * k;
    }
  }
}

// ------------------------------------------------------------------------------------ nearest-upsample backward
// dx[n,h,w,:] (+ add) = sum of dy[n,oh,ow,:] over the output pixels whose torch-nearest source
// (floor(o * in / out), the map of upsample_nearest_kernel) is (h, w).  fp32 NHWC, C % 4 == 0.
__global__ void upsample_nearest_bwd_kernel(const float* __restrict__ dy, int NB, int H, int W, int C, int OH, int OW,
                                            const float* add, float* dx) {
  const int V = C / 4;
  const long long total = (long long)NB * H * W * V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    const long long pix = i / V;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const int n = (int)(pix / ((long long)W * H));
    const int oh0 = (int)(((long long)h * OH + H - 1) / H), ow0 = (int)(((long long)w * OW + W - 1) / W);
    float4 acc = add ? reinterpret_cast<const float4*>(add + pix * C)[v] : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int oh = oh0; oh < OH && (int)(((long long)oh * H) / OH) == h; ++oh)
      for (int ow = ow0; ow < OW && (int)(((long long)ow * W) / OW) == w; ++ow) {
        const float4 d = reinterpret_cast<const float4*>(dy + (((long long)n * OH + oh) * OW + ow) * C)[v];
        acc.x += d.x; acc.y += d.y; acc.z += d.z; acc.w += d.w;
      }
    reinterpret_cast<float4*>(dx + pix * C)[v] = acc;
  }
}

}  // namespace b200

using namespace b200;

static int bw_gn_block(int C) {
  const int V = C / 8;
  if (V > 1024) return -1;
  int rpb = 256 / V;
  if (rpb < 1) rpb = 1;
  return V * rpb;
}
static int bw_gn_ppc(int NB, int HW, int rows_per_pass) {
  int target = (sm_count() * 8 + NB - 1) / NB;
  int ppc = (HW + target - 1) / target;
  if (ppc < rows_per_pass * 4) ppc = rows_per_pass * 4;
  return ppc;
}
static unsigned bw_grid1d(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = (long long)sm_count() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (unsigned)g;
}

extern "C" int b200_gather_planar(const void* x, int in_f32, long long ldx, int NB, int H, int W, int C, int Ho, int Wo,
                                  int stride, int up, int oy, int ox, void* out, long long ldo, void* stream) {
  B200_CHECK_ARG(x && out && NB > 0 && H > 0 && W > 0 && C > 0 && Ho > 0 && Wo > 0, "b200_gather_planar: bad arguments");
  B200_CHECK_ARG(stride >= 1 && (up == 1 || up == 2) && ldx >= C, "b200_gather_planar: stride=%d up=%d ldx=%lld", stride, up, ldx);
  const long long P = (long long)NB * Ho * Wo;
  B200_CHECK_ARG(ldo >= P, "b200_gather_planar: ldo=%lld < pixels=%lld", ldo, P);
  const long long Ppad = ldo;   // the whole row is written (zeros past P)
  dim3 grid((unsigned)((Ppad + 31) / 32), (unsigned)((C + 31) / 32));
  B200_CHECK_ARG(grid.y <= 65535, "b200_gather_planar: C=%d too large", C);
  dim3 block(32, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    gather_planar_kernel<float><<<grid, block, 0, st>>>((const float*)x, ldx, H, W, C, Ho, Wo, stride, up, oy, ox, P, Ppad,
                                                        (__half*)out, ldo);
  else
    gather_planar_kernel<__half><<<grid, block, 0, st>>>((const __half*)x, ldx, H, W, C, Ho, Wo, stride, up, oy, ox, P, Ppad,
                                                         (__half*)out, ldo);
  B200_CHECK_LAUNCH("gather_planar_kernel");
  return 0;
}

extern "C" int b200_rowdot_heads_d(const void* a, long long a_bs, long long a_ls, const void* c, long long c_bs,
                                   long long c_ls, int B, int L, int heads, int head_dim, float* out, void* stream) {
  B200_CHECK_ARG(head_dim == 40 || head_dim == 64 || head_dim == 80 || head_dim == 160,
                 "b200_rowdot_heads_d: head_dim=%d is not one of 40, 64, 80, 160", head_dim);
  B200_CHECK_ARG(a && c && out && B > 0 && L > 0 && heads > 0, "b200_rowdot_heads: bad arguments");
  B200_CHECK_ARG(a_ls % 2 == 0 && c_ls % 2 == 0 && a_bs % 2 == 0 && c_bs % 2 == 0 &&
                     (((uintptr_t)a | (uintptr_t)c) & 3) == 0, "b200_rowdot_heads: 4-byte alignment");
  dim3 grid((L + 7) / 8, heads, B);
  const cudaStream_t st = (cudaStream_t)stream;
  const __half *ah = (const __half*)a, *ch = (const __half*)c;
  switch (head_dim) {
    case 40: rowdot_heads_kernel<40><<<grid, 256, 0, st>>>(ah, a_bs, a_ls, ch, c_bs, c_ls, L, heads, out); break;
    case 64: rowdot_heads_kernel<64><<<grid, 256, 0, st>>>(ah, a_bs, a_ls, ch, c_bs, c_ls, L, heads, out); break;
    case 80: rowdot_heads_kernel<80><<<grid, 256, 0, st>>>(ah, a_bs, a_ls, ch, c_bs, c_ls, L, heads, out); break;
    default: rowdot_heads_kernel<160><<<grid, 256, 0, st>>>(ah, a_bs, a_ls, ch, c_bs, c_ls, L, heads, out); break;
  }
  B200_CHECK_LAUNCH("rowdot_heads_kernel");
  return 0;
}

extern "C" int b200_rowdot_heads(const void* a, long long a_bs, long long a_ls, const void* c, long long c_bs,
                                 long long c_ls, int B, int L, int heads, float* out, void* stream) {
  return b200_rowdot_heads_d(a, a_bs, a_ls, c, c_bs, c_ls, B, L, heads, 64, out, stream);
}

extern "C" int b200_col_sum(const void* x, int in_f32, long long rows, int C, long long ld, float* out, void* stream) {
  B200_CHECK_ARG(x && out && rows > 0 && C > 0 && ld >= C, "b200_col_sum: bad arguments");
  const int R = cluster_ctas(rows, 512);
  const dim3 grid((C + 31) / 32, R), block(32, R > 1 ? 32 : 8), cluster(1, R, 1);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    launch_clustered(col_sum_kernel<float>, grid, block, 0, st, cluster, (const float*)x, rows, C, ld, out);
  else
    launch_clustered(col_sum_kernel<__half>, grid, block, 0, st, cluster, (const __half*)x, rows, C, ld, out);
  B200_CHECK_LAUNCH("col_sum_kernel");
  return 0;
}

extern "C" int b200_group_norm_mean_rstd(const double* sums, const double* cs1, int C1, const double* cs2, int C2,
                                         int NB, int HW, int groups, float eps, float* mean_rstd, void* stream) {
  B200_CHECK_ARG(mean_rstd && NB > 0 && HW > 0 && groups > 0 && C1 > 0, "b200_group_norm_mean_rstd: bad arguments");
  B200_CHECK_ARG(sums || cs1, "b200_group_norm_mean_rstd: need group sums or per-channel sums");
  B200_CHECK_ARG((C2 == 0) || sums || cs2, "b200_group_norm_mean_rstd: cs2 missing");
  B200_CHECK_ARG((C1 + C2) % groups == 0, "b200_group_norm_mean_rstd: C=%d groups=%d", C1 + C2, groups);
  const int n = NB * groups;
  gn_mean_rstd_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sums, cs1, C1, cs2, C2, NB, HW, groups, eps,
                                                                         mean_rstd);
  B200_CHECK_LAUNCH("gn_mean_rstd_kernel");
  return 0;
}

static int gn_bwd_check(const char* fn, const void* x, int Cx, int c_off, int Ctot, const void* dy, int NB, int HW,
                        int groups) {
  B200_CHECK_ARG(x && dy && NB > 0 && HW > 0 && Cx > 0, "%s: bad arguments", fn);
  B200_CHECK_ARG(Cx % 8 == 0 && c_off % 8 == 0 && Ctot % 8 == 0 && c_off + Cx <= Ctot,
                 "%s: Cx=%d c_off=%d Ctot=%d must be multiples of 8 with c_off+Cx <= Ctot", fn, Cx, c_off, Ctot);
  B200_CHECK_ARG(groups > 0 && Ctot % groups == 0, "%s: Ctot=%d groups=%d", fn, Ctot, groups);
  B200_CHECK_ARG(bw_gn_block(Cx) > 0 && bw_gn_block(Cx) <= 1024, "%s: Cx=%d unsupported", fn, Cx);
  return 0;
}

extern "C" int b200_group_norm_bwd_sums(const void* x, int in_f32, int Cx, int c_off, int Ctot, const void* dy,
                                        int NB, int HW, int groups, const float* mean_rstd, const float* gamma,
                                        const float* beta, int silu, float* S, void* stream) {
  int r = gn_bwd_check("b200_group_norm_bwd_sums", x, Cx, c_off, Ctot, dy, NB, HW, groups);
  if (r) return r;
  B200_CHECK_ARG(mean_rstd && gamma && beta && S, "b200_group_norm_bwd_sums: null pointer");
  const int R = cluster_ctas(HW, 4LL * kGnSumsThreads);
  const dim3 grid(R, (Cx + 15) / 16, NB), cluster(R, 1, 1);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    launch_clustered(gn_bwd_sums_kernel<float>, grid, dim3(kGnSumsThreads), 0, st, cluster, (const float*)x, Cx, c_off,
                     Ctot, (const __half*)dy, HW, groups, mean_rstd, gamma, beta, silu, S);
  else
    launch_clustered(gn_bwd_sums_kernel<__half>, grid, dim3(kGnSumsThreads), 0, st, cluster, (const __half*)x, Cx, c_off,
                     Ctot, (const __half*)dy, HW, groups, mean_rstd, gamma, beta, silu, S);
  B200_CHECK_LAUNCH("gn_bwd_sums_kernel");
  return 0;
}

extern "C" int b200_group_norm_bwd_apply(const void* x, int in_f32, int Cx, int c_off, int Ctot, const void* dy,
                                         int NB, int HW, int groups, const float* mean_rstd, const float* gamma,
                                         const float* beta, int silu, const float* S, const void* add, void* dx,
                                         int out_f32, void* stream) {
  int r = gn_bwd_check("b200_group_norm_bwd_apply", x, Cx, c_off, Ctot, dy, NB, HW, groups);
  if (r) return r;
  B200_CHECK_ARG(mean_rstd && gamma && beta && S && dx, "b200_group_norm_bwd_apply: null pointer");
  const int T = bw_gn_block(Cx);
  const int ppc = bw_gn_ppc(NB, HW, T / (Cx / 8));
  dim3 grid((HW + ppc - 1) / ppc, NB);
  const size_t smem = 2 * groups * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define B200_GN_BWD(T_, TO_)                                                                                          \
  gn_bwd_apply_kernel<T_, TO_><<<grid, T, smem, st>>>((const T_*)x, Cx, c_off, Ctot, (const __half*)dy, HW, groups,   \
                                                      ppc, mean_rstd, gamma, beta, silu, S, (const TO_*)add, (TO_*)dx)
  if (in_f32 && out_f32) B200_GN_BWD(float, float);
  else if (in_f32) B200_GN_BWD(float, __half);
  else if (out_f32) B200_GN_BWD(__half, float);
  else B200_GN_BWD(__half, __half);
#undef B200_GN_BWD
  B200_CHECK_LAUNCH("gn_bwd_apply_kernel");
  return 0;
}

extern "C" int b200_layer_norm_bwd(const void* x, int in_f32, long long rows, int C, const float* gamma,
                                   const void* dy, float eps, const void* add, void* dx, int out_f32,
                                   float* dgamma, float* dbeta, void* stream) {
  B200_CHECK_ARG(x && dy && dx && gamma && dgamma && dbeta && rows > 0, "b200_layer_norm_bwd: bad arguments");
  B200_CHECK_ARG(C % 8 == 0 && C <= 2048, "b200_layer_norm_bwd: C=%d must be a multiple of 8 and <= 2048", C);
  // vectors of 8 per lane (the row is held in registers), then warps per CTA: as many per-warp (d_gamma, d_beta) rows
  // as fit in 200 KB of shared memory, at most 32 (16 with more than 2 vectors per lane: registers)
  const int nv_need = (C / 8 + 31) / 32;
  const int nv = nv_need <= 2 ? nv_need : (nv_need <= 5 ? 5 : 8);
  int wpb = (int)((200 * 1024 / sizeof(float) - 2 * C) / (2 * C));
  const int wmax = nv <= 2 ? 32 : 16;
  wpb = wpb < 1 ? 1 : (wpb > wmax ? wmax : wpb);
  const int R = cluster_ctas(rows, 4LL * wpb, kMaxSingleSlotCtas);
  const size_t smem = (size_t)(wpb + 1) * 2 * C * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
#define B200_LN_BWD_NV(T_, TO_, NV_)                                                                                 \
  do {                                                                                                              \
    cudaFuncSetAttribute(layer_norm_bwd_kernel<T_, TO_, NV_>, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                         (int)smem);                                                                                \
    launch_clustered(layer_norm_bwd_kernel<T_, TO_, NV_>, dim3(R), dim3(wpb * 32), smem, st, dim3(R, 1, 1),         \
                     (const T_*)x, rows, C, gamma, (const __half*)dy, eps, (const TO_*)add, (TO_*)dx, dgamma, dbeta); \
  } while (0)
#define B200_LN_BWD(T_, TO_)                                                                                        \
  do {                                                                                                              \
    if (nv == 1) B200_LN_BWD_NV(T_, TO_, 1);                                                                        \
    else if (nv == 2) B200_LN_BWD_NV(T_, TO_, 2);                                                                   \
    else if (nv == 5) B200_LN_BWD_NV(T_, TO_, 5);                                                                   \
    else B200_LN_BWD_NV(T_, TO_, 8);                                                                                \
  } while (0)
  if (in_f32 && out_f32) B200_LN_BWD(float, float);
  else if (in_f32) B200_LN_BWD(float, __half);
  else if (out_f32) B200_LN_BWD(__half, float);
  else B200_LN_BWD(__half, __half);
#undef B200_LN_BWD
#undef B200_LN_BWD_NV
  B200_CHECK_LAUNCH("layer_norm_bwd_kernel");
  return 0;
}

extern "C" int b200_softmax_bwd_rows(const void* P, long long ldp, const float* dP, long long ldd, void* dS,
                                     long long rows, int cols, float scale, void* stream) {
  B200_CHECK_ARG(P && dP && dS && rows > 0 && cols > 0 && ldp >= cols && ldd >= cols, "b200_softmax_bwd_rows: bad arguments");
  B200_CHECK_ARG(rows <= 2147483647LL, "b200_softmax_bwd_rows: too many rows");
  softmax_bwd_rows_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const __half*)P, ldp, dP, ldd, (__half*)dS,
                                                                            cols, scale);
  B200_CHECK_LAUNCH("softmax_bwd_rows_kernel");
  return 0;
}

extern "C" int b200_act_bwd(const void* x, const void* dy, long long n, int act, void* dx, void* stream) {
  B200_CHECK_ARG(x && dy && dx && n > 0, "b200_act_bwd: bad arguments");
  B200_CHECK_ARG(act == B200_ACT_SILU || act == B200_ACT_GELU, "b200_act_bwd: act=%d (SiLU or GELU)", act);
  act_bwd_kernel<<<bw_grid1d(n, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, (const __half*)dy, n,
                                                                      act == B200_ACT_SILU ? 1 : 3, (__half*)dx);
  B200_CHECK_LAUNCH("act_bwd_kernel");
  return 0;
}

extern "C" int b200_geglu_bwd(const void* h, const void* g, long long ld_hg, const void* dy, long long rows, int inner,
                              void* dh, void* dg, long long ld_d, void* stream) {
  B200_CHECK_ARG(h && g && dy && dh && dg && rows > 0 && inner > 0 && ld_hg >= inner && ld_d >= inner,
                 "b200_geglu_bwd: bad arguments");
  geglu_bwd_kernel<<<bw_grid1d(rows * inner, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)h, (const __half*)g, ld_hg, (const __half*)dy, rows, inner, (__half*)dh, (__half*)dg, ld_d);
  B200_CHECK_LAUNCH("geglu_bwd_kernel");
  return 0;
}

static dim3 bw_loss_grid(long long HW, int B) {
  long long g = (HW + 256 * 8 - 1) / (256 * 8);
  long long cap = (long long)sm_count() * 4 / (B > 0 ? B : 1) + 1;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return dim3((unsigned)g, B);
}

extern "C" int b200_ssi_loss_bwd(const float* pred, const float* target, const unsigned char* mask, int B,
                                 long long HW, double* workspace, const float* grad_out, float* dpred, void* stream) {
  B200_CHECK_ARG(pred && target && mask && workspace && grad_out && dpred && B > 0 && HW > 0,
                 "b200_ssi_loss_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int R = cluster_ctas(HW, 8LL * kLossBwdThreads);
  launch_clustered(ssi_bwd_moments_kernel, dim3(R, B), dim3(kLossBwdThreads), 0, st, dim3(R, 1, 1), pred, target, mask,
                   HW, workspace);
  launch_clustered(ssi_bwd_sign_sums_kernel, dim3(R, B), dim3(kLossBwdThreads), 0, st, dim3(R, 1, 1), pred, target,
                   mask, HW, B, workspace);
  dim3 grid = bw_loss_grid(HW, B);
  ssi_bwd_grad_kernel<<<grid, 256, 0, st>>>(pred, target, mask, HW, B, workspace, grad_out, dpred);
  B200_CHECK_LAUNCH("ssi_loss_bwd kernels");
  return 0;
}

extern "C" int b200_angular_loss_bwd(const float* pred, const float* target, const unsigned char* mask, int B,
                                     long long HW, double* workspace, const float* grad_out, float* dpred,
                                     void* stream) {
  B200_CHECK_ARG(pred && target && mask && workspace && grad_out && dpred && B > 0 && HW > 0,
                 "b200_angular_loss_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int R = cluster_ctas((long long)B * HW, 8LL * kLossBwdThreads, kMaxSingleSlotCtas);
  launch_clustered(mask_count_kernel, dim3(R), dim3(kLossBwdThreads), 0, st, dim3(R, 1, 1), mask, (long long)B * HW,
                   workspace);
  angular_bwd_kernel<<<bw_loss_grid(HW, B), 256, 0, st>>>(pred, target, mask, HW, workspace, grad_out, dpred);
  B200_CHECK_LAUNCH("angular_loss_bwd kernels");
  return 0;
}

extern "C" int b200_decode_post_bwd(const float* x, const float* dout, int NB, long long HW, int mode, float* dx,
                                    void* stream) {
  B200_CHECK_ARG(x && dout && dx && NB > 0 && HW > 0 && (mode == 2 || mode == 3), "b200_decode_post_bwd: bad arguments");
  decode_post_bwd_kernel<<<bw_loss_grid(HW, NB), 256, 0, (cudaStream_t)stream>>>(x, dout, HW, mode, dx);
  B200_CHECK_LAUNCH("decode_post_bwd_kernel");
  return 0;
}

extern "C" int b200_upsample_nearest_bwd(const float* dy, int NB, int H, int W, int C, int OH, int OW, const float* add,
                                         float* dx, void* stream) {
  B200_CHECK_ARG(dy && dx && NB > 0 && H > 0 && W > 0 && OH >= H && OW >= W, "b200_upsample_nearest_bwd: bad arguments");
  B200_CHECK_ARG(C % 4 == 0, "b200_upsample_nearest_bwd: C=%d must be a multiple of 4", C);
  const long long total = (long long)NB * H * W * (C / 4);
  upsample_nearest_bwd_kernel<<<bw_grid1d(total, 256), 256, 0, (cudaStream_t)stream>>>(dy, NB, H, W, C, OH, OW, add, dx);
  B200_CHECK_LAUNCH("upsample_nearest_bwd_kernel");
  return 0;
}
