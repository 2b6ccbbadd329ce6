// HBM-bound normalisation kernels: GroupNorm (two-pass, NHWC, fused concat + SiLU), LayerNorm,
// row softmax.  16-byte vectorised coalesced loads, warp-shuffle reductions, fp32 statistics.
#include <type_traits>

#include "cluster_reduce.cuh"
#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

__device__ __forceinline__ void load8(const __half* p, float* v) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __half22float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const float* p, float* v) {
  float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8h(__half* p, const float* v) {
  __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
  __half2 h2 = __floats2half2_rn(v[4], v[5]), h3 = __floats2half2_rn(v[6], v[7]);
  uint4 u;
  u.x = *reinterpret_cast<uint32_t*>(&h0);
  u.y = *reinterpret_cast<uint32_t*>(&h1);
  u.z = *reinterpret_cast<uint32_t*>(&h2);
  u.w = *reinterpret_cast<uint32_t*>(&h3);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------ GroupNorm stats
// sums[n][g] += (sum x, sum x^2) in fp64.  grid (R, slices, NB), cluster (R): one cluster per (image, slice of gs whole
// groups, gs * C/groups a multiple of 8 channels).  Thread t owns the 8-channel vector t % VS of the slice and every
// rpb-th pixel of its CTA's contiguous share.  Per-thread sums (shifted, see below) -> a [rpb][2 CS] table in shared
// memory -> channels summed over the rows in row order -> groups over their channels in order -> the cluster's CTAs
// in rank order (cluster_reduce.cuh), added to `sums` by rank 0.  No atomics: the bits depend only on the inputs.
template <typename T>
__global__ void gn_stats_kernel(const T* __restrict__ x1, int C1, const T* __restrict__ x2, int C2,
                                int HW, int groups, int gs, double* __restrict__ sums) {
  extern __shared__ double smd[];   // [rpb][2 CS] per-thread sums, [2 CS] per-channel sums, [2 gs] group partials
  const int C = C1 + C2, cpg = C / groups, CS = gs * cpg, VS = CS / 8;
  const int n = blockIdx.z;
  const int g0 = blockIdx.y * gs, ng = min(gs, groups - g0);
  const int rpb = blockDim.x / VS;
  const int v = threadIdx.x % VS;
  const int r = threadIdx.x / VS;
  // per-thread sums of (x - shift), (x - shift)^2 with shift = the thread's first element of each channel:
  // no cancellation for |mean| >> std; converted to plain sums in fp64 before merging
  float s[8], q[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = q[e] = sh[e] = 0.f;
  int cnt = 0;
  long long lp0, lp1;
  cluster_share(HW, gridDim.x, blockIdx.x, lp0, lp1);
  const int p0 = (int)lp0, p1 = (int)lp1;
  const int c0 = g0 * cpg + v * 8;
  const bool second = c0 >= C1;
  const T* base = second ? x2 + (long long)n * HW * C2 + (c0 - C1) : x1 + (long long)n * HW * C1 + c0;
  const int ld = second ? C2 : C1;
  if (v * 8 < ng * cpg) {
    int p = p0 + r;
    if (p < p1) load8(base + (long long)p * ld, sh);
    for (; p + 3 * rpb < p1; p += 4 * rpb) {
      float f[4][8];
#pragma unroll
      for (int u = 0; u < 4; ++u) load8(base + (long long)(p + u * rpb) * ld, f[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float d = f[u][e] - sh[e]; s[e] += d; q[e] = fmaf(d, d, q[e]); }
      cnt += 4;
    }
    for (; p < p1; p += rpb) {
      float f[8];
      load8(base + (long long)p * ld, f);
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = f[e] - sh[e]; s[e] += d; q[e] = fmaf(d, d, q[e]); }
      cnt += 1;
    }
  }
  const double nn = (double)cnt;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const double shd = (double)sh[e], s1 = (double)s[e];
    smd[(long long)r * 2 * CS + (v * 8 + e) * 2 + 0] = s1 + nn * shd;
    smd[(long long)r * 2 * CS + (v * 8 + e) * 2 + 1] = (double)q[e] + 2.0 * shd * s1 + nn * shd * shd;
  }
  __syncthreads();
  double* ch = smd + (long long)rpb * 2 * CS;
  for (int k = threadIdx.x; k < 2 * CS; k += blockDim.x) {
    double t = smd[k];
    for (int rr = 1; rr < rpb; ++rr) t += smd[(long long)rr * 2 * CS + k];
    ch[k] = t;
  }
  __syncthreads();
  double* part = ch + 2 * CS;
  for (int k = threadIdx.x; k < 2 * ng; k += blockDim.x) {
    const int g = k >> 1, f = k & 1;
    double t = 0.0;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) t += ch[c * 2 + f];
    part[k] = t;
  }
  cluster_add_partials(part, 2 * ng, [&](int k) { return sums + ((long long)n * groups + g0) * 2 + k; });
}

// ------------------------------------------------------------------------------ GroupNorm apply
// grid (chunks, NB).  Per-(n,c) scale/shift precomputed into smem, then a pure streaming pass.
template <typename T>
__global__ void gn_apply_kernel(const T* __restrict__ x1, int C1, const T* __restrict__ x2, int C2,
                                int HW, int groups, int pix_per_cta, const double* __restrict__ sums,
                                const double* __restrict__ cs1, const double* __restrict__ cs2,
                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                float eps, int silu, __half* __restrict__ y, __half* __restrict__ raw) {
  extern __shared__ float sm[];   // scale[C], shift[C], then group (mean, rstd)[groups][2]
  const int C = C1 + C2;
  const int V = C / 8;
  const int n = blockIdx.y;
  const int cg = C / groups;
  const double cnt = (double)HW * cg;
  float* gstat = sm + 2 * C;
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    double su, sq;
    if (sums) {
      su = sums[((long long)n * groups + g) * 2 + 0];
      sq = sums[((long long)n * groups + g) * 2 + 1];
    } else {
      // per-channel sums written by the producing kernels' epilogues; a group may straddle the concat
      su = 0.0; sq = 0.0;
      for (int c = g * cg; c < (g + 1) * cg; ++c) {
        const double* src = c < C1 ? cs1 + ((long long)n * C1 + c) * 2 : cs2 + ((long long)n * C2 + (c - C1)) * 2;
        su += src[0];
        sq += src[1];
      }
    }
    const double mean = su / cnt;
    double var = sq / cnt - mean * mean;
    if (var < 0) var = 0;
    gstat[2 * g] = (float)mean;
    gstat[2 * g + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cg;
    const float a = gstat[2 * g + 1] * gamma[c];
    sm[c] = a;
    sm[C + c] = beta[c] - gstat[2 * g] * a;
  }
  __syncthreads();
  const int rpb = blockDim.x / V;
  const int v = threadIdx.x % V;
  const int r = threadIdx.x / V;
  if (r >= rpb) return;
  const int c0 = v * 8;
  const bool second = c0 >= C1;
  const T* base = second ? x2 + (long long)n * HW * C2 + (c0 - C1) : x1 + (long long)n * HW * C1 + c0;
  const int ld = second ? C2 : C1;
  float a[8], b[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { a[e] = sm[c0 + e]; b[e] = sm[C + c0 + e]; }
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  __half* yb = y + (long long)n * HW * C + c0;
  __half* rb = raw ? raw + (long long)n * HW * C + c0 : nullptr;
  // 8 pixels per iteration: eight independent 16/32-byte loads in flight per thread (latency-bound otherwise).  The
  // loaded vectors stay in their storage type until use (fp16 input: 4 registers per pixel instead of 8), which keeps
  // the fp16 instantiation under 85 registers = three 256-thread CTAs per SM instead of two.
  using Raw = typename std::conditional<sizeof(T) == 2, uint4, float4>::type;
  constexpr int kRawPerPix = sizeof(T) == 2 ? 1 : 2;
  auto unpack = [](const Raw* rv, float* f) {
    if constexpr (sizeof(T) == 2) {
      const __half2* h = reinterpret_cast<const __half2*>(rv);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
      }
    } else {
      f[0] = rv[0].x; f[1] = rv[0].y; f[2] = rv[0].z; f[3] = rv[0].w;
      f[4] = rv[1].x; f[5] = rv[1].y; f[6] = rv[1].z; f[7] = rv[1].w;
    }
  };
  int p = p0 + r;
  for (; p + 7 * rpb < p1; p += 8 * rpb) {
    Raw raw[8][kRawPerPix];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const Raw* src = reinterpret_cast<const Raw*>(base + (long long)(p + u * rpb) * ld);
#pragma unroll
      for (int k = 0; k < kRawPerPix; ++k) raw[u][k] = src[k];
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      float f[8], o[8];
      unpack(raw[u], f);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float t = f[e] * a[e] + b[e];
        o[e] = silu ? __fdividef(t, 1.0f + __expf(-t)) : t;
      }
      store8h(yb + (long long)(p + u * rpb) * C, o);
      if (rb) store8h(rb + (long long)(p + u * rpb) * C, f);
    }
  }
  for (; p < p1; p += rpb) {
    float f[8], o[8];
    load8(base + (long long)p * ld, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float t = f[e] * a[e] + b[e];
      o[e] = silu ? __fdividef(t, 1.0f + __expf(-t)) : t;
    }
    store8h(yb + (long long)p * C, o);
    if (rb) store8h(rb + (long long)p * C, f);
  }
}

static int gn_block(int C) {
  const int V = C / 8;
  if (V > 1024) return -1;
  int rpb = 256 / V;
  if (rpb < 1) rpb = 1;
  return V * rpb;
}

// ------------------------------------------------------------------------------ LayerNorm
// one warp per row; C <= 2048, C % 8 == 0.  Two-pass in registers (exact mean, then variance).
// NV = per-lane 8-element vectors actually needed (ceil(C / 256)) is a template parameter: with the fixed 8 (64 value
// registers, most of them dead for C = 320 / 640) the kernel runs 2 CTAs per SM and keeps too few bytes in flight to
// approach the HBM roofline.
template <typename T, int NV>
__global__ void layer_norm_kernel(const T* __restrict__ x, long long rows, int C,
                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                  float eps, __half* __restrict__ y) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int V = C / 8;
  float f[NV][8];
  float s = 0.f;
  const T* xr = x + row * C;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + 32 * i;
    if (v < V) {
      load8(xr + v * 8, f[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) s += f[i][e];
    }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + 32 * i;
    if (v < V) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = f[i][e] - mean; q += d * d; }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  __half* yr = y + row * C;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + 32 * i;
    if (v < V) {
      float g[8], b[8], o[8];
      load8(gamma + v * 8, g);
      load8(beta + v * 8, b);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = (f[i][e] - mean) * rstd * g[e] + b[e];
      store8h(yr + v * 8, o);
    }
  }
}

template <typename T>
static void launch_layer_norm(const T* x, long long rows, int C, const float* gamma, const float* beta, float eps,
                              __half* y, cudaStream_t st) {
  const int wpb = 8;
  const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
  switch ((C + 255) / 256) {
    case 1: layer_norm_kernel<T, 1><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
    case 2: layer_norm_kernel<T, 2><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
    case 3: layer_norm_kernel<T, 3><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
    case 4: layer_norm_kernel<T, 4><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
    case 5: layer_norm_kernel<T, 5><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
    case 6: layer_norm_kernel<T, 6><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
    case 7: layer_norm_kernel<T, 7><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
    default: layer_norm_kernel<T, 8><<<grid, wpb * 32, 0, st>>>(x, rows, C, gamma, beta, eps, y); break;
  }
}

// ------------------------------------------------------------------------------ row softmax
// one CTA (256 threads) per row: fp32 logits -> fp16 probabilities; three streaming passes
// (row re-reads hit L2: a 9216-float row is 36 KB).  VEC = 4 when cols and strides are %4.
template <int VEC>
__global__ void softmax_rows_kernel(const float* __restrict__ S, long long lds, __half* __restrict__ P,
                                    long long ldp, int cols, float scale) {
  __shared__ float red[32];
  const float* s = S + (long long)blockIdx.x * lds;
  __half* p = P + (long long)blockIdx.x * ldp;
  const int tid = threadIdx.x, nw = blockDim.x >> 5;
  float m = -INFINITY;
  for (int c = tid * VEC; c < cols; c += blockDim.x * VEC) {
    if constexpr (VEC == 4) {
      float4 v = *reinterpret_cast<const float4*>(s + c);
      m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    } else {
      m = fmaxf(m, s[c]);
    }
  }
  m = warp_max(m);
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int i = 1; i < nw; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  const float sl2 = scale * 1.4426950408889634f;
  const float ms = m * sl2;
  float sum = 0.f;
  for (int c = tid * VEC; c < cols; c += blockDim.x * VEC) {
    if constexpr (VEC == 4) {
      float4 v = *reinterpret_cast<const float4*>(s + c);
      sum += exp2f(v.x * sl2 - ms) + exp2f(v.y * sl2 - ms) + exp2f(v.z * sl2 - ms) + exp2f(v.w * sl2 - ms);
    } else {
      sum += exp2f(s[c] * sl2 - ms);
    }
  }
  sum = warp_sum(sum);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < nw; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int c = tid * VEC; c < cols; c += blockDim.x * VEC) {
    if constexpr (VEC == 4) {
      float4 v = *reinterpret_cast<const float4*>(s + c);
      __half2 a = __floats2half2_rn(exp2f(v.x * sl2 - ms) * inv, exp2f(v.y * sl2 - ms) * inv);
      __half2 b = __floats2half2_rn(exp2f(v.z * sl2 - ms) * inv, exp2f(v.w * sl2 - ms) * inv);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&a);
      u.y = *reinterpret_cast<uint32_t*>(&b);
      *reinterpret_cast<uint2*>(p + c) = u;
    } else {
      p[c] = __float2half_rn(exp2f(s[c] * sl2 - ms) * inv);
    }
  }
}

// Same result, one HBM read per row: the fp32 row is staged in shared memory (cols <= 16384) and the max / sum / write
// passes run out of it.  Persistent CTAs; the rows arrive by cp.async.bulk (one elected thread, no register staging)
// into a two-deep ring, so the next row is in flight while this one is reduced and written — with register-staged
// loads issued by the same threads that later do the exp / store passes the kernel keeps too few bytes in flight per SM
// to approach the HBM roofline.
__device__ __forceinline__ void bulk_load_row(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__global__ void softmax_rows_smem_kernel(const float* __restrict__ S, long long lds, __half* __restrict__ P,
                                         long long ldp, long long rows, int cols, float scale) {
  extern __shared__ __align__(16) float rowbuf[];          // [2][cols]
  __shared__ float red[32];
  __shared__ __align__(8) uint64_t full[2];
  const int tid = threadIdx.x, nw = blockDim.x >> 5;
  const uint32_t row_bytes = (uint32_t)cols * 4u;
  if (tid == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  long long r = blockIdx.x;
  if (tid == 0 && r < rows) {
    mbar_arrive_expect_tx(&full[0], row_bytes);
    bulk_load_row(rowbuf, S + r * lds, row_bytes, &full[0]);
  }
  const float sl2 = scale * 1.4426950408889634f;
  uint32_t phase[2] = {0u, 0u};
  int buf = 0;
  for (; r < rows; r += gridDim.x, buf ^= 1) {
    const long long rn = r + gridDim.x;
    if (tid == 0 && rn < rows) {
      // the other buffer was last touched by generic-proxy stores of the previous iteration (all threads are past the
      // trailing __syncthreads): order them before the async-proxy write
      fence_proxy_async_smem();
      mbar_arrive_expect_tx(&full[buf ^ 1], row_bytes);
      bulk_load_row(rowbuf + (size_t)(buf ^ 1) * cols, S + rn * lds, row_bytes, &full[buf ^ 1]);
    }
    mbar_wait(&full[buf], phase[buf]);
    phase[buf] ^= 1u;
    float* row = rowbuf + (size_t)buf * cols;
    __half* p = P + r * ldp;
    float m = -INFINITY;
    for (int c = tid * 4; c < cols; c += blockDim.x * 4) {
      const float4 v = *reinterpret_cast<const float4*>(row + c);
      m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    }
    m = warp_max(m);
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    m = red[0];
    for (int i = 1; i < nw; ++i) m = fmaxf(m, red[i]);
    __syncthreads();
    const float ms = m * sl2;
    float sum = 0.f;
    for (int c = tid * 4; c < cols; c += blockDim.x * 4) {      // each thread re-reads exactly what it writes
      float4 v = *reinterpret_cast<const float4*>(row + c);
      v.x = exp2f(v.x * sl2 - ms); v.y = exp2f(v.y * sl2 - ms); v.z = exp2f(v.z * sl2 - ms); v.w = exp2f(v.w * sl2 - ms);
      *reinterpret_cast<float4*>(row + c) = v;
      sum += (v.x + v.y) + (v.z + v.w);
    }
    sum = warp_sum(sum);
    if ((tid & 31) == 0) red[tid >> 5] = sum;
    __syncthreads();
    sum = 0.f;
    for (int i = 0; i < nw; ++i) sum += red[i];
    const float inv = 1.0f / sum;
    for (int c = tid * 4; c < cols; c += blockDim.x * 4) {
      const float4 v = *reinterpret_cast<const float4*>(row + c);
      __half2 a = __floats2half2_rn(v.x * inv, v.y * inv), b = __floats2half2_rn(v.z * inv, v.w * inv);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&a);
      u.y = *reinterpret_cast<uint32_t*>(&b);
      *reinterpret_cast<uint2*>(p + c) = u;
    }
    __syncthreads();                                          // `red` and this row buffer are free again
  }
}

// ------------------------------------------------------------------------------ grouped softmax
// Constant-context cross-attention (SURVEY.md §8 f1): logits [rows][ld_in] fp32 hold heads x S scores per query
// row (column j = head * S + s); softmax over the S keys of each head -> fp16 [rows][ld_out], padding columns
// (>= heads*S) written as zeros so the row is a K-padded GEMM operand.  One thread per row.
__global__ void softmax_groups_kernel(const float* __restrict__ lg, int ld_in, long long rows, int heads, int S,
                                      __half* __restrict__ p, int ld_out) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const float* src = lg + r * ld_in;
  __half* dst = p + r * ld_out;
  const int J = heads * S;
  for (int h = 0; h < heads; ++h) {
    float m = -INFINITY;
    for (int s = 0; s < S; ++s) m = fmaxf(m, src[h * S + s]);
    float sum = 0.f;
    for (int s = 0; s < S; ++s) sum += __expf(src[h * S + s] - m);
    const float inv = 1.0f / sum;
    for (int s = 0; s < S; ++s) dst[h * S + s] = __float2half_rn(__expf(src[h * S + s] - m) * inv);
  }
  for (int j = J; j < ld_out; ++j) dst[j] = __float2half_rn(0.f);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_softmax_groups(const float* logits, int ld_in, long long rows, int heads, int S, void* P,
                                   int ld_out, void* stream) {
  B200_CHECK_ARG(logits && P && rows > 0 && heads > 0 && S > 0, "b200_softmax_groups: bad arguments");
  B200_CHECK_ARG(heads * S <= ld_in && heads * S <= ld_out, "b200_softmax_groups: heads*S=%d exceeds ld (%d, %d)",
                 heads * S, ld_in, ld_out);
  softmax_groups_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      logits, ld_in, rows, heads, S, (__half*)P, ld_out);
  B200_CHECK_LAUNCH("softmax_groups_kernel");
  return 0;
}

static int gn_common_check(const char* fn, const void* x1, int C1, const void* x2, int C2, int NB,
                           int HW, int groups) {
  const int C = C1 + C2;
  B200_CHECK_ARG(x1 && C1 > 0 && NB > 0 && HW > 0, "%s: bad arguments", fn);
  B200_CHECK_ARG((C2 == 0) == (x2 == nullptr), "%s: x2/C2 mismatch", fn);
  B200_CHECK_ARG(C1 % 8 == 0 && C2 % 8 == 0, "%s: channel counts must be multiples of 8 (C1=%d C2=%d)", fn, C1, C2);
  B200_CHECK_ARG(groups > 0 && C % groups == 0, "%s: C=%d not divisible by groups=%d", fn, C, groups);
  B200_CHECK_ARG(gn_block(C) > 0 && gn_block(C) <= 1024, "%s: C=%d unsupported", fn, C);
  return 0;
}

static int gn_chunks(int NB, int HW, int rows_per_pass) {
  // ~8 CTAs per SM across the batch (2048 threads/SM: maximum bytes in flight), at least rows_per_pass pixels per CTA
  int target = (sm_count() * 8 + NB - 1) / NB;
  int ppc = (HW + target - 1) / target;
  if (ppc < rows_per_pass * 4) ppc = rows_per_pass * 4;
  return ppc;
}

extern "C" int b200_group_norm_stats(const void* x1, int C1, const void* x2, int C2, int in_f32, int NB,
                                     int HW, int groups, double* sums, void* stream) {
  int r = gn_common_check("b200_group_norm_stats", x1, C1, x2, C2, NB, HW, groups);
  if (r) return r;
  B200_CHECK_ARG(sums, "b200_group_norm_stats: null sums");
  // slices of gs whole groups: the fewest groups whose channels fill 8-channel vectors, doubled up to 16 channels
  const int cpg = (C1 + C2) / groups;
  int gs = 1;
  while ((gs * cpg) % 8 != 0) ++gs;
  while (2 * gs * cpg <= 16 && 2 * gs <= groups) gs *= 2;
  const int VS = gs * cpg / 8;
  const int rpb = VS >= 256 ? 1 : 256 / VS;
  const int T = VS * rpb;
  const int R = cluster_ctas(HW, 16LL * rpb);
  const dim3 grid(R, (groups + gs - 1) / gs, NB), cluster(R, 1, 1);
  const size_t smem = ((size_t)(rpb + 1) * 2 * gs * cpg + 2 * gs) * sizeof(double);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32) {
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(gn_stats_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    launch_clustered(gn_stats_kernel<float>, grid, dim3(T), smem, st, cluster, (const float*)x1, C1, (const float*)x2,
                     C2, HW, groups, gs, sums);
  } else {
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(gn_stats_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    launch_clustered(gn_stats_kernel<__half>, grid, dim3(T), smem, st, cluster, (const __half*)x1, C1,
                     (const __half*)x2, C2, HW, groups, gs, sums);
  }
  B200_CHECK_LAUNCH("gn_stats_kernel");
  return 0;
}

extern "C" int b200_group_norm_apply(const void* x1, int C1, const void* x2, int C2, int in_f32, int NB,
                                     int HW, int groups, const double* sums, const float* gamma,
                                     const float* beta, float eps, int silu, void* y, void* raw_copy,
                                     void* stream) {
  int r = gn_common_check("b200_group_norm_apply", x1, C1, x2, C2, NB, HW, groups);
  if (r) return r;
  B200_CHECK_ARG(sums && gamma && beta && y, "b200_group_norm_apply: null pointer");
  const int C = C1 + C2;
  const int T = gn_block(C);
  const int ppc = gn_chunks(NB, HW, T / (C / 8));
  dim3 grid((HW + ppc - 1) / ppc, NB);
  const size_t smem = (2 * C + 2 * groups) * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    gn_apply_kernel<float><<<grid, T, smem, st>>>((const float*)x1, C1, (const float*)x2, C2, HW, groups, ppc, sums,
                                                  nullptr, nullptr, gamma, beta, eps, silu, (__half*)y, (__half*)raw_copy);
  else
    gn_apply_kernel<__half><<<grid, T, smem, st>>>((const __half*)x1, C1, (const __half*)x2, C2, HW, groups, ppc, sums,
                                                   nullptr, nullptr, gamma, beta, eps, silu, (__half*)y, (__half*)raw_copy);
  B200_CHECK_LAUNCH("gn_apply_kernel");
  return 0;
}

extern "C" int b200_group_norm_apply_cs(const void* x1, int C1, const double* cs1, const void* x2, int C2,
                                        const double* cs2, int in_f32, int NB, int HW, int groups,
                                        const float* gamma, const float* beta, float eps, int silu, void* y,
                                        void* raw_copy, void* stream) {
  int r = gn_common_check("b200_group_norm_apply_cs", x1, C1, x2, C2, NB, HW, groups);
  if (r) return r;
  B200_CHECK_ARG(cs1 && (C2 == 0 || cs2) && gamma && beta && y, "b200_group_norm_apply_cs: null pointer");
  const int C = C1 + C2;
  const int T = gn_block(C);
  const int ppc = gn_chunks(NB, HW, T / (C / 8));
  dim3 grid((HW + ppc - 1) / ppc, NB);
  const size_t smem = (2 * C + 2 * groups) * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    gn_apply_kernel<float><<<grid, T, smem, st>>>((const float*)x1, C1, (const float*)x2, C2, HW, groups, ppc, nullptr,
                                                  cs1, cs2, gamma, beta, eps, silu, (__half*)y, (__half*)raw_copy);
  else
    gn_apply_kernel<__half><<<grid, T, smem, st>>>((const __half*)x1, C1, (const __half*)x2, C2, HW, groups, ppc, nullptr,
                                                   cs1, cs2, gamma, beta, eps, silu, (__half*)y, (__half*)raw_copy);
  B200_CHECK_LAUNCH("gn_apply_kernel(cs)");
  return 0;
}

extern "C" int b200_layer_norm(const void* x, int in_f32, long long rows, int C, const float* gamma,
                               const float* beta, float eps, void* y, void* stream) {
  B200_CHECK_ARG(x && y && gamma && beta && rows > 0, "b200_layer_norm: bad arguments");
  B200_CHECK_ARG(C % 8 == 0 && C <= 2048, "b200_layer_norm: C=%d must be a multiple of 8 and <= 2048", C);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    launch_layer_norm<float>((const float*)x, rows, C, gamma, beta, eps, (__half*)y, st);
  else
    launch_layer_norm<__half>((const __half*)x, rows, C, gamma, beta, eps, (__half*)y, st);
  B200_CHECK_LAUNCH("layer_norm_kernel");
  return 0;
}

extern "C" int b200_softmax_rows(const float* S, long long lds, void* P, long long ldp, long long rows,
                                 int cols, float scale, void* stream) {
  B200_CHECK_ARG(S && P && rows > 0 && cols > 0, "b200_softmax_rows: bad arguments");
  const bool vec = cols % 4 == 0 && lds % 4 == 0 && ldp % 4 == 0 && ((uintptr_t)S & 15) == 0 && ((uintptr_t)P & 7) == 0;
  if (vec && cols <= 16384) {
    static bool configured_dev[kMaxDevices] = {false};
    const int dev_ = current_device();
    bool& configured = configured_dev[dev_ < 0 ? 0 : dev_];
    if (!configured || dev_ < 0) {
      cudaFuncSetAttribute(softmax_rows_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 65536);
      configured = true;
    }
    const size_t smem = (size_t)cols * 8;                         // two row buffers
    const long long per_sm = (220 * 1024) / (long long)(smem + 1024);
    long long grid = (long long)sm_count() * (per_sm < 1 ? 1 : per_sm);
    if (grid > rows) grid = rows;
    softmax_rows_smem_kernel<<<(unsigned)grid, 256, smem, (cudaStream_t)stream>>>(S, lds, (__half*)P, ldp, rows, cols, scale);
  } else if (vec)
    softmax_rows_kernel<4><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(S, lds, (__half*)P, ldp, cols, scale);
  else
    softmax_rows_kernel<1><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(S, lds, (__half*)P, ldp, cols, scale);
  B200_CHECK_LAUNCH("softmax_rows_kernel");
  return 0;
}
