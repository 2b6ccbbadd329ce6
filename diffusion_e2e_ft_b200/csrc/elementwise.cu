// Small HBM-bound helpers around the tensor-core kernels: patch extraction for the tiny-Cin input
// convolutions, nearest upsample, timestep sinusoid, latent channel mixes, decode post-ops,
// boundary casts.
#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

// out[pixel][tap*C + c] (fp16, row length Kpad, zero padded), x NCHW.  One thread per pixel: it gathers the
// 9*C (<= 72) neighbours (L1/L2-served: neighbouring threads share them) and writes its whole patch row with
// 16-byte stores, so the 64-128 byte rows leave as full sectors.
template <typename T, int KPAD>
__global__ void im2col3x3_kernel(const T* __restrict__ x, int NB, int C, int H, int W,
                                 __half* __restrict__ out) {
  const long long total = (long long)NB * H * W;
  for (long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x; pix < total;
       pix += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const int n = (int)(pix / ((long long)W * H));
    constexpr int CC = KPAD == 32 ? 3 : (KPAD == 40 ? 4 : 8);       // compile-time channel count: row[] stays in registers
    __align__(16) __half row[KPAD];
#pragma unroll
    for (int k = 0; k < KPAD; ++k) row[k] = __float2half_rn(0.f);
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int hh = h + tap / 3 - 1, ww = w + tap % 3 - 1;
      const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W;
#pragma unroll
      for (int c = 0; c < CC; ++c)
        row[tap * CC + c] = ok ? __float2half_rn((float)x[(((long long)n * CC + c) * H + hh) * W + ww])
                               : __float2half_rn(0.f);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + pix * KPAD);
    const uint4* src = reinterpret_cast<const uint4*>(row);
#pragma unroll
    for (int v = 0; v < KPAD / 8; ++v) dst[v] = src[v];
  }
}

template <typename T>
__global__ void upsample_nearest_kernel(const T* __restrict__ x, int NB, int H, int W, int C, int OH,
                                        int OW, __half* __restrict__ y) {
  const int V = C / 8;
  const long long total = (long long)NB * OH * OW * V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % V);
    long long pix = i / V;
    const int ow = (int)(pix % OW);
    const int oh = (int)((pix / OW) % OH);
    const int n = (int)(pix / ((long long)OW * OH));
    // torch nearest: src = floor(dst * in / out)
    const int ih = min((int)(((long long)oh * H) / OH), H - 1);
    const int iw = min((int)(((long long)ow * W) / OW), W - 1);
    const T* src = x + (((long long)n * H + ih) * W + iw) * C + v * 8;
    __half* dst = y + pix * C + v * 8;
    if constexpr (sizeof(T) == 2) {
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    } else {
      float4 a = reinterpret_cast<const float4*>(src)[0], b = reinterpret_cast<const float4*>(src)[1];
      __half2 h0 = __floats2half2_rn(a.x, a.y), h1 = __floats2half2_rn(a.z, a.w);
      __half2 h2 = __floats2half2_rn(b.x, b.y), h3 = __floats2half2_rn(b.z, b.w);
      uint4 u;
      u.x = *reinterpret_cast<uint32_t*>(&h0);
      u.y = *reinterpret_cast<uint32_t*>(&h1);
      u.z = *reinterpret_cast<uint32_t*>(&h2);
      u.w = *reinterpret_cast<uint32_t*>(&h3);
      *reinterpret_cast<uint4*>(dst) = u;
    }
  }
}

// emb[b] = [cos(t*f_0..f_{h-1}), sin(t*f_0..)], f_i = exp(-ln(1e4) * i / half)   (flip_sin_to_cos)
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int B, int dim,
                                          __half* __restrict__ out) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * half) return;
  const int b = i / half, j = i - b * half;
  const float freq = expf(-9.210340371976184f * (float)j / (float)half);
  const float a = t[b] * freq;
  out[(long long)b * dim + j] = __float2half_rn(cosf(a));
  out[(long long)b * dim + half + j] = __float2half_rn(sinf(a));
}

// CLIP text embeddings (transformers modeling_clip CLIPTextEmbeddings): out[b*L + l][c] = tok[ids[b*L + l]][c] + pos[l][c],
// fp32 residual stream out; the tables are fp16 or fp32 (the module's parameter dtype).  One warp-strided pass, 8 B+ per lane.
template <typename T>
__global__ void embed_tokens_kernel(const long long* __restrict__ ids, const T* __restrict__ tok, const T* __restrict__ pos,
                                    long long rows, int L, int C, int vocab, float* __restrict__ out) {
  const long long total = rows * (long long)(C / 4);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / (C / 4);
    const int c = (int)(i - r * (C / 4)) * 4;
    long long id = ids[r];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const T* a = tok + id * C + c;
    const T* b = pos + (r % L) * C + c;
    float4 o;
    if constexpr (sizeof(T) == 2) {
      const __half2 a0 = reinterpret_cast<const __half2*>(a)[0], a1 = reinterpret_cast<const __half2*>(a)[1];
      const __half2 b0 = reinterpret_cast<const __half2*>(b)[0], b1 = reinterpret_cast<const __half2*>(b)[1];
      const float2 fa0 = __half22float2(a0), fa1 = __half22float2(a1), fb0 = __half22float2(b0), fb1 = __half22float2(b1);
      o = make_float4(fa0.x + fb0.x, fa0.y + fb0.y, fa1.x + fb1.x, fa1.y + fb1.y);
    } else {
      const float4 fa = *reinterpret_cast<const float4*>(a), fb = *reinterpret_cast<const float4*>(b);
      o = make_float4(fa.x + fb.x, fa.y + fb.y, fa.z + fb.z, fa.w + fb.w);
    }
    *reinterpret_cast<float4*>(out + r * C + c) = o;
  }
}

__global__ void pointwise_nchw_kernel(const float* __restrict__ in1, float a1,
                                      const float* __restrict__ in2, float a2, int in_cstride,
                                      const float* __restrict__ Wm, const float* __restrict__ bias,
                                      int Cin, int Cout, long long HW, float* __restrict__ out) {
  __shared__ float w[64 + 8];
  if (threadIdx.x < Cin * Cout) w[threadIdx.x] = Wm[threadIdx.x];
  if (threadIdx.x < Cout) w[64 + threadIdx.x] = bias ? bias[threadIdx.x] : 0.f;
  __syncthreads();
  const int n = blockIdx.y;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW;
       p += (long long)gridDim.x * blockDim.x) {
    float v[8];
    for (int ci = 0; ci < Cin; ++ci) {
      float t = a1 * in1[((long long)n * in_cstride + ci) * HW + p];
      if (in2) t += a2 * in2[((long long)n * in_cstride + ci) * HW + p];
      v[ci] = t;
    }
    for (int co = 0; co < Cout; ++co) {
      float acc = w[64 + co];
      for (int ci = 0; ci < Cin; ++ci) acc += w[co * Cin + ci] * v[ci];
      out[((long long)n * Cout + co) * HW + p] = acc;
    }
  }
}

__global__ void decode_post_kernel(const float* __restrict__ x, long long HW, int mode, float sign,
                                   float* __restrict__ out) {
  const int n = blockIdx.y;
  const float* xb = x + (long long)n * 3 * HW;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW;
       p += (long long)gridDim.x * blockDim.x) {
    const float a = xb[p], b = xb[HW + p], c = xb[2 * HW + p];
    if (mode == 0 || mode == 2) {
      float m = (a + b + c) / 3.0f;
      m = fminf(fmaxf(m, -1.0f), 1.0f);
      out[(long long)n * HW + p] = mode == 0 ? (m + 1.0f) / 2.0f : m;     // mode 2: training (train.py:533-534)
    } else {
      const float inv = sign / (sqrtf(a * a + b * b + c * c) + 1e-5f);
      float* ob = out + (long long)n * 3 * HW;
      float v0 = a * inv, v1 = b * inv, v2 = c * inv;
      if (mode == 3) {                                                     // training: clamp (train.py:539)
        v0 = fminf(fmaxf(v0, -1.f), 1.f); v1 = fminf(fmaxf(v1, -1.f), 1.f); v2 = fminf(fmaxf(v2, -1.f), 1.f);
      }
      ob[p] = v0;
      ob[HW + p] = v1;
      ob[2 * HW + p] = v2;
    }
  }
}

// diffusers DDIMScheduler.step with eta = 0, in fp32 and in diffusers' order of operations (each product and sum
// rounded on its own, no contraction): x0 / eps for the prediction type, then prev = sqrt(a_prev) x0 + sqrt(1-a_prev)
// eps.  `prev` may alias `sample` (each element is read before it is written).  UI: 0 = no UNet-input copy, 1 = fp16,
// 2 = fp32 copy of prev into a channel slice of the next UNet input.
template <typename MO, int UI>
__global__ void ddim_step_kernel(const MO* __restrict__ mo, long long mo_bs, const float* x, long long s_bs,
                                 long long CHW, int ptype, float a_t, float a_prev, float* prev,
                                 float* __restrict__ x0_out, void* __restrict__ ui, long long ui_bs) {
  const int n = blockIdx.y;
  const float beta = __fsub_rn(1.0f, a_t);
  const float sa = sqrtf(a_t), sb = sqrtf(beta);
  const float sp = sqrtf(a_prev), sd = sqrtf(__fsub_rn(1.0f, a_prev));
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < CHW;
       i += (long long)gridDim.x * blockDim.x) {
    const float m = (float)mo[n * mo_bs + i];
    const float s = x ? x[n * s_bs + i] : 0.0f;
    float x0, eps;
    if (ptype == B200_PRED_V) {
      x0 = __fsub_rn(__fmul_rn(sa, s), __fmul_rn(sb, m));
      eps = __fadd_rn(__fmul_rn(sa, m), __fmul_rn(sb, s));
    } else if (ptype == B200_PRED_EPSILON) {
      x0 = __fdiv_rn(__fsub_rn(s, __fmul_rn(sb, m)), sa);
      eps = m;
    } else {                                                   // B200_PRED_SAMPLE
      x0 = m;
      eps = __fdiv_rn(__fsub_rn(s, __fmul_rn(sa, x0)), sb);
    }
    const float p = __fadd_rn(__fmul_rn(sp, x0), __fmul_rn(sd, eps));
    prev[n * CHW + i] = p;
    if (x0_out) x0_out[n * CHW + i] = x0;
    if constexpr (UI == 1) reinterpret_cast<__half*>(ui)[n * ui_bs + i] = __float2half_rn(p);
    if constexpr (UI == 2) reinterpret_cast<float*>(ui)[n * ui_bs + i] = p;
  }
}

// DDPM add_noise + get_velocity + the UNet-input concatenation of the diffusion objective, one pass over [2B][C][HW]:
// unet_in[n] = [rgb[n mod B] | sqrt(a) x0 + sqrt(1-a) eps], target[n] = eps (epsilon) or sqrt(a) eps - sqrt(1-a) x0
// (v_prediction), a = alphas_cumprod[t[n]].  Each product and sum rounded on its own, as torch evaluates diffusers'
// expressions; eps = 0 when noise is null.
__global__ void diffusion_inputs_kernel(const float* __restrict__ rgb, const float* __restrict__ x0,
                                        const float* __restrict__ noise, const long long* __restrict__ t,
                                        const float* __restrict__ ac, int B, long long CHW, int ptype,
                                        float* __restrict__ unet_in, float* __restrict__ target) {
  const int n = blockIdx.y;
  const float a = ac[t[n]];
  const float sa = __fsqrt_rn(a), sb = __fsqrt_rn(__fsub_rn(1.0f, a));
  const float* xr = rgb + (long long)(n % B) * CHW;
  const float* xb = x0 + (long long)n * CHW;
  const float* nb = noise ? noise + (long long)n * CHW : nullptr;
  float* ui = unet_in + (long long)n * 2 * CHW;
  float* tg = target + (long long)n * CHW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < CHW; i += (long long)gridDim.x * blockDim.x) {
    const float x = xb[i];
    const float e = nb ? nb[i] : 0.0f;
    ui[i] = xr[i];
    ui[CHW + i] = __fadd_rn(__fmul_rn(sa, x), __fmul_rn(sb, e));
    tg[i] = ptype == B200_PRED_V ? __fsub_rn(__fmul_rn(sa, e), __fmul_rn(sb, x)) : e;
  }
}

__global__ void cast_f32_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    y[i] = __float2half_rn(x[i]);
}

// NHWC -> NCHW fp32 through a 32x32 smem transpose tile (coalesced both sides).
template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ x, int C, long long HW, float* __restrict__ y) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const long long p0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const long long p = p0 + r;
    const int c = c0 + threadIdx.x;
    if (p < HW && c < C) tile[r][threadIdx.x] = (float)x[((long long)n * HW + p) * C + c];
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int c = c0 + r;
    const long long p = p0 + threadIdx.x;
    if (p < HW && c < C) y[((long long)n * C + c) * HW + p] = tile[threadIdx.x][r];
  }
}

static int grid_for(long long n, int block) {
  long long g = (n + block - 1) / block;
  long long cap = (long long)sm_count() * 16;
  return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_im2col3x3_nchw(const void* x, int x_f32, int NB, int C, int H, int W, void* out,
                                   int Kpad, void* stream) {
  B200_CHECK_ARG(x && out && NB > 0 && C > 0 && H > 0 && W > 0, "b200_im2col3x3_nchw: bad arguments");
  B200_CHECK_ARG(Kpad >= 9 * C && Kpad % 8 == 0, "b200_im2col3x3_nchw: Kpad=%d must be >= 9*C and %%8==0", Kpad);
  B200_CHECK_ARG((Kpad == 32 && C == 3) || (Kpad == 40 && C == 4) || (Kpad == 72 && C == 8),
                 "b200_im2col3x3_nchw: (C=%d, Kpad=%d) unsupported: C must be 3, 4 or 8 with Kpad = round_up(9C, 8)", C, Kpad);
  const long long total = (long long)NB * H * W;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(total, 128);
#define B200_IM2COL(T, K) im2col3x3_kernel<T, K><<<g, 128, 0, st>>>((const T*)x, NB, C, H, W, (__half*)out)
  if (x_f32) {
    if (Kpad == 32) B200_IM2COL(float, 32); else if (Kpad == 40) B200_IM2COL(float, 40); else B200_IM2COL(float, 72);
  } else {
    if (Kpad == 32) B200_IM2COL(__half, 32); else if (Kpad == 40) B200_IM2COL(__half, 40); else B200_IM2COL(__half, 72);
  }
#undef B200_IM2COL
  B200_CHECK_LAUNCH("im2col3x3_kernel");
  return 0;
}

extern "C" int b200_upsample_nearest_nhwc(const void* x, int in_f32, int NB, int H, int W, int C, int OH,
                                          int OW, void* y, void* stream) {
  B200_CHECK_ARG(x && y && NB > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, "b200_upsample_nearest_nhwc: bad arguments");
  B200_CHECK_ARG(C % 8 == 0, "b200_upsample_nearest_nhwc: C=%d must be a multiple of 8", C);
  const long long total = (long long)NB * OH * OW * (C / 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    upsample_nearest_kernel<float><<<grid_for(total, 256), 256, 0, st>>>((const float*)x, NB, H, W, C, OH, OW, (__half*)y);
  else
    upsample_nearest_kernel<__half><<<grid_for(total, 256), 256, 0, st>>>((const __half*)x, NB, H, W, C, OH, OW, (__half*)y);
  B200_CHECK_LAUNCH("upsample_nearest_kernel");
  return 0;
}

extern "C" int b200_timestep_embedding(const float* t, int B, int dim, void* out, void* stream) {
  B200_CHECK_ARG(t && out && B > 0 && dim > 0 && dim % 2 == 0, "b200_timestep_embedding: bad arguments");
  const int n = B * (dim / 2);
  timestep_embedding_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(t, B, dim, (__half*)out);
  B200_CHECK_LAUNCH("timestep_embedding_kernel");
  return 0;
}

extern "C" int b200_embed_tokens(const long long* ids, const void* tok, const void* pos, int w_f32, long long rows, int L,
                                 int C, int vocab, float* out, void* stream) {
  B200_CHECK_ARG(ids && tok && pos && out && rows > 0 && L > 0 && vocab > 0, "b200_embed_tokens: bad arguments");
  B200_CHECK_ARG(C > 0 && C % 4 == 0, "b200_embed_tokens: C=%d must be a multiple of 4", C);
  const long long total = rows * (long long)(C / 4);
  cudaStream_t st = (cudaStream_t)stream;
  if (w_f32)
    embed_tokens_kernel<float><<<grid_for(total, 256), 256, 0, st>>>(ids, (const float*)tok, (const float*)pos, rows, L, C, vocab, out);
  else
    embed_tokens_kernel<__half><<<grid_for(total, 256), 256, 0, st>>>(ids, (const __half*)tok, (const __half*)pos, rows, L, C, vocab, out);
  B200_CHECK_LAUNCH("embed_tokens_kernel");
  return 0;
}

extern "C" int b200_pointwise_nchw(const float* in1, float a1, const float* in2, float a2, int in_cstride,
                                   const float* Wm, const float* bias, int NB, int Cin, int Cout,
                                   long long HW, float* out, void* stream) {
  B200_CHECK_ARG(in1 && Wm && out && NB > 0 && HW > 0, "b200_pointwise_nchw: bad arguments");
  B200_CHECK_ARG(Cin >= 1 && Cin <= 8 && Cout >= 1 && Cout <= 8 && in_cstride >= Cin,
                 "b200_pointwise_nchw: Cin=%d Cout=%d must be in [1,8]", Cin, Cout);
  dim3 grid(grid_for(HW, 256), NB);
  pointwise_nchw_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in1, a1, in2, a2, in_cstride, Wm, bias, Cin, Cout, HW, out);
  B200_CHECK_LAUNCH("pointwise_nchw_kernel");
  return 0;
}

extern "C" int b200_decode_post(const float* x, int NB, long long HW, int mode, float sign, float* out,
                                void* stream) {
  B200_CHECK_ARG(x && out && NB > 0 && HW > 0 && mode >= 0 && mode <= 3, "b200_decode_post: bad arguments");
  dim3 grid(grid_for(HW, 256), NB);
  decode_post_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, HW, mode, sign, out);
  B200_CHECK_LAUNCH("decode_post_kernel");
  return 0;
}

extern "C" int b200_ddim_step(const void* model_out, int mo_f16, long long mo_bstride, const float* sample,
                              long long s_bstride, int B, int C, long long HW, int prediction_type,
                              float alpha_prod_t, float alpha_prod_t_prev, float* prev_sample,
                              float* pred_original_sample, void* unet_in, int unet_in_f16, long long ui_bstride,
                              void* stream) {
  B200_CHECK_ARG(model_out && prev_sample, "b200_ddim_step: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && C >= 1 && HW >= 1, "b200_ddim_step: bad shape B=%d C=%d HW=%lld", B, C, HW);
  const long long CHW = (long long)C * HW;
  B200_CHECK_ARG(mo_bstride >= CHW && (!sample || s_bstride >= CHW) && (!unet_in || ui_bstride >= CHW),
                 "b200_ddim_step: batch strides must be >= C*HW");
  B200_CHECK_ARG((const void*)prev_sample != (const void*)sample || s_bstride == CHW,
                 "b200_ddim_step: prev_sample may alias sample only when sample is contiguous (s_bstride = C*HW)");
  B200_CHECK_ARG(prediction_type == B200_PRED_EPSILON || prediction_type == B200_PRED_V ||
                 prediction_type == B200_PRED_SAMPLE, "b200_ddim_step: unknown prediction_type %d", prediction_type);
  B200_CHECK_ARG(alpha_prod_t > 0.0f && alpha_prod_t < 1.0f && alpha_prod_t_prev >= 0.0f && alpha_prod_t_prev <= 1.0f,
                 "b200_ddim_step: alpha_prod_t must be in (0, 1) and alpha_prod_t_prev in [0, 1]");
  dim3 grid(grid_for(CHW, 256), B);
  cudaStream_t st = (cudaStream_t)stream;
  const int ui = unet_in ? (unet_in_f16 ? 1 : 2) : 0;
#define B200_DDIM(MO, UI)                                                                                        \
  ddim_step_kernel<MO, UI><<<grid, 256, 0, st>>>((const MO*)model_out, mo_bstride, sample, s_bstride, CHW,      \
                                                 prediction_type, alpha_prod_t, alpha_prod_t_prev, prev_sample, \
                                                 pred_original_sample, unet_in, ui_bstride)
  if (mo_f16) {
    if (ui == 0) B200_DDIM(__half, 0); else if (ui == 1) B200_DDIM(__half, 1); else B200_DDIM(__half, 2);
  } else {
    if (ui == 0) B200_DDIM(float, 0); else if (ui == 1) B200_DDIM(float, 1); else B200_DDIM(float, 2);
  }
#undef B200_DDIM
  B200_CHECK_LAUNCH("ddim_step_kernel");
  return 0;
}

extern "C" int b200_diffusion_inputs(const float* rgb_latents, const float* x0, const float* noise,
                                     const long long* timesteps, const float* alphas_cumprod, int B, int C,
                                     long long HW, int prediction_type, float* unet_in, float* target,
                                     void* stream) {
  B200_CHECK_ARG(rgb_latents && x0 && timesteps && alphas_cumprod && unet_in && target,
                 "b200_diffusion_inputs: null pointer");
  B200_CHECK_ARG(B >= 1 && 2 * B <= 65535 && C >= 1 && HW >= 1, "b200_diffusion_inputs: bad shape B=%d C=%d HW=%lld",
                 B, C, HW);
  B200_CHECK_ARG(prediction_type == B200_PRED_EPSILON || prediction_type == B200_PRED_V,
                 "b200_diffusion_inputs: prediction_type %d is not epsilon or v_prediction", prediction_type);
  const long long CHW = (long long)C * HW;
  dim3 grid(grid_for(CHW, 256), 2 * B);
  diffusion_inputs_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(rgb_latents, x0, noise, timesteps, alphas_cumprod, B,
                                                                  CHW, prediction_type, unet_in, target);
  B200_CHECK_LAUNCH("diffusion_inputs_kernel");
  return 0;
}

extern "C" int b200_cast_f32_to_f16(const float* x, void* y, long long n, void* stream) {
  B200_CHECK_ARG(x && y && n > 0, "b200_cast_f32_to_f16: bad arguments");
  cast_f32_f16_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, (__half*)y, n);
  B200_CHECK_LAUNCH("cast_f32_f16_kernel");
  return 0;
}

extern "C" int b200_nhwc_to_nchw_f32(const void* x, int in_f32, int NB, int C, long long HW, float* y,
                                     void* stream) {
  B200_CHECK_ARG(x && y && NB > 0 && C > 0 && HW > 0, "b200_nhwc_to_nchw_f32: bad arguments");
  dim3 grid((unsigned)((HW + 31) / 32), (C + 31) / 32, NB), block(32, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (in_f32)
    nhwc_to_nchw_kernel<float><<<grid, block, 0, st>>>((const float*)x, C, HW, y);
  else
    nhwc_to_nchw_kernel<__half><<<grid, block, 0, st>>>((const __half*)x, C, HW, y);
  B200_CHECK_LAUNCH("nhwc_to_nchw_kernel");
  return 0;
}
