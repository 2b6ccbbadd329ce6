// Optimizer-side kernels of the fine-tuning step over FLAT fp32 buffers (all UNet parameters / gradients /
// moments live in one contiguous allocation each): squared-gradient-norm reduction for
// `clip_grad_norm_` and a fused clip + AdamW update.  Reference: training/train.py:346-353 (AdamW:
// lr 3e-5, betas (0.9, 0.999), weight_decay 1e-2, eps 1e-8) and :564-566 (clip to max_grad_norm, step).
// HBM-bound: 16 B read + 12 B written per parameter.
#include "cluster_reduce.cuh"
#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

// *out += sum x^2 in fp64.  One cluster of CTAs: CTA `rank` sums a fixed contiguous share of the float4s
// thread-sequentially (the last CTA also takes the n % 4 tail), block_sum_fixed combines the threads and rank 0 adds the
// CTAs' partials in rank order (cluster_reduce.cuh): the same bits on every run and every H100.
__global__ void __launch_bounds__(1024) sumsq_kernel(const float* __restrict__ x, long long n, double* __restrict__ out) {
  __shared__ double part[1];
  const int rank = (int)cooperative_groups::this_cluster().block_rank(), R = gridDim.x;
  double acc[1] = {0.0};
  const long long n4 = n / 4;
  long long lo, hi;
  cluster_share(n4, R, rank, lo, hi);
  const float4* x4 = reinterpret_cast<const float4*>(x);
#pragma unroll 4
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const float4 v = x4[i];
    acc[0] += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
  }
  if (rank == R - 1)
    for (long long i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) acc[0] += (double)x[i] * x[i];
  block_sum_fixed(acc, part);
  cluster_add_partials(part, 1, [&](int) { return out; });
}

// torch.optim.AdamW (decoupled weight decay, bias-corrected), gradient pre-scaled by the clip coefficient
// min(1, max_norm / (||g|| + 1e-6)) read from the device (no host sync between norm and step).
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, long long n, float lr, float beta1, float beta2, float eps,
                             float wd, float bc1, float bc2, const double* __restrict__ gnorm_sq, float max_norm,
                             float unscale) {
  // `unscale` = 1 / loss scale: the buffer holds S * g; the norm (of S * g) and the gradient are brought back first
  float clip = unscale;
  if (gnorm_sq != nullptr && !isfinite(*gnorm_sq)) return;        // a non-finite gradient must not poison the moments
  if (gnorm_sq != nullptr && max_norm > 0.f) {
    const float nrm = (float)sqrt(*gnorm_sq) * unscale;
    clip = unscale * fminf(1.0f, max_norm / (nrm + 1e-6f));
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * clip;
    float pi = p[i] * (1.0f - lr * wd);
    const float mi = beta1 * m[i] + (1.0f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.0f - beta2) * gi * gi;
    const float denom = sqrtf(vi) / sqrtf(bc2) + eps;
    pi -= (lr / bc1) * (mi / denom);
    p[i] = pi; m[i] = mi; v[i] = vi;
  }
}

// 1 - beta^step, evaluated in fp64 and rounded to fp32 once.  In fp32 the subtraction cancels: for beta2 = 0.999 at
// step 2 even a correctly rounded powf leaves the result about 110 fp32 ulps (6.7e-6 relative) from 1 - beta^step.
__host__ __device__ __forceinline__ float bias_correction(float beta, float step) {
  return (float)(1.0 - pow((double)beta, (double)step));
}

// ---- optimizer step with device-side state: skipped steps + dynamic loss scaling, no host sync ----------------
// state (fp32[8], device): [0] loss scale S (the trainer multiplies the loss by it before backward), [1] growth
// tracker, [2] applied optimizer steps, [3] skipped steps, [4] this step skipped (0/1), [5] gradient multiplier of
// this step (clip coefficient / (S * world)), [6] bc1, [7] bc2.
// A step is SKIPPED — parameters and both moments untouched, like torch.optim.AdamW for parameters whose .grad is None
// — when the gradient norm is non-finite (an fp16 overflow in the loss-scaled backward; the scale is then halved) or
// exactly zero (every micro-batch had an empty validity mask / NaN loss: training/train.py:503,546-551 then
// back-propagates a constant 0).
__global__ void optim_prepare_kernel(const double* __restrict__ gnorm_sq, float* __restrict__ state, float max_norm,
                                     float inv_world, float beta1, float beta2, int dynamic, float growth_interval,
                                     float min_scale, float max_scale) {
  float S = state[0], tracker = state[1];
  const double nsq = *gnorm_sq;
  const bool finite = isfinite(nsq);
  const float unscale = inv_world / S;
  if (!finite || nsq == 0.0) {
    state[3] += 1.f;
    state[4] = 1.f;
    state[5] = 0.f;
    if (!finite && dynamic) { S = fmaxf(S * 0.5f, min_scale); tracker = 0.f; }
  } else {
    const float step = state[2] + 1.f;
    state[2] = step;
    state[4] = 0.f;
    float clip = unscale;
    if (max_norm > 0.f) {
      const float nrm = (float)sqrt(nsq) * unscale;
      clip = unscale * fminf(1.0f, max_norm / (nrm + 1e-6f));
    }
    state[5] = clip;
    state[6] = bias_correction(beta1, step);
    state[7] = bias_correction(beta2, step);
    if (dynamic) {
      tracker += 1.f;
      if (tracker >= growth_interval) { S = fminf(S * 2.0f, max_scale); tracker = 0.f; }
    }
  }
  state[0] = S;
  state[1] = tracker;
}

// Per-group learning rate / weight decay (torch.optim.AdamW parameter groups, ABI 11): the flat buffer is cut into
// RUNS, contiguous ranges [run_start[r], run_start[r+1]) each belonging to one group; run_start is increasing, starts
// at 0 and every start is a multiple of 4 (each parameter view starts 16-byte aligned), so a float4 never straddles
// two groups.  The run table (device) is staged in shared memory and a float4's run found by binary search; the
// per-group (lr, weight_decay) pairs travel as launch arguments.  run_start == nullptr: one run, group 0, taking
// the one-group loops of the kernel before ABI 11 unchanged.
struct AdamwGroupHP {
  float lr[B200_ADAMW_MAX_GROUPS];
  float wd[B200_ADAMW_MAX_GROUPS];
};

__global__ void adamw_state_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                   float* __restrict__ v, long long n, const long long* __restrict__ run_start,
                                   const int* __restrict__ run_group, int n_runs, AdamwGroupHP hp, int n_groups,
                                   float beta1, float beta2, float eps, const float* __restrict__ state) {
  __shared__ long long s_start[B200_ADAMW_MAX_RUNS];
  __shared__ int s_group[B200_ADAMW_MAX_RUNS];
  __shared__ float s_decay[B200_ADAMW_MAX_GROUPS], s_step[B200_ADAMW_MAX_GROUPS];
  if (state[4] != 0.f) return;                                   // skipped step: nothing is touched (block-uniform)
  const float clip = state[5], bc1 = state[6], rbc2 = rsqrtf(state[7]);
  const long long n4 = n / 4;
  float4* p4 = reinterpret_cast<float4*>(p);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  auto upd = [&](float& pi, float gi, float& mi, float& vi, float decay, float step_size) {
    gi *= clip;
    mi = beta1 * mi + (1.0f - beta1) * gi;
    vi = beta2 * vi + (1.0f - beta2) * gi * gi;
    pi = pi * decay - step_size * (mi / (sqrtf(vi) * rbc2 + eps));
  };
  if (run_start == nullptr) {
    // one group: the loops of the kernel before ABI 11, with decay / step_size held in registers, so the compiled
    // update (and its rounding) is the one b200_adamw_step_state always had
    const float decay = 1.0f - hp.lr[0] * hp.wd[0], step_size = hp.lr[0] / bc1;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
      float4 pp = p4[i], mm = m4[i], vv = v4[i];
      const float4 gg = g4[i];
      upd(pp.x, gg.x, mm.x, vv.x, decay, step_size); upd(pp.y, gg.y, mm.y, vv.y, decay, step_size);
      upd(pp.z, gg.z, mm.z, vv.z, decay, step_size); upd(pp.w, gg.w, mm.w, vv.w, decay, step_size);
      p4[i] = pp; m4[i] = mm; v4[i] = vv;
    }
    for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
      upd(p[i], g[i], m[i], v[i], decay, step_size);
    return;
  }
  for (int r = threadIdx.x; r < n_runs; r += blockDim.x) {
    s_start[r] = run_start[r];
    s_group[r] = min(max(run_group[r], 0), n_groups - 1);
  }
  if ((int)threadIdx.x < n_groups) {
    const float lr = hp.lr[threadIdx.x], wd = hp.wd[threadIdx.x];
    s_decay[threadIdx.x] = 1.0f - lr * wd;
    s_step[threadIdx.x] = lr / bc1;
  }
  __syncthreads();
  auto group_of = [&](long long e) {                             // the last run starting at or before element e
    int lo = 0, hi = n_runs - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_start[mid] <= e) lo = mid; else hi = mid - 1;
    }
    return s_group[lo];
  };
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const int k = group_of(4 * i);
    const float decay = s_decay[k], step_size = s_step[k];
    float4 pp = p4[i], mm = m4[i], vv = v4[i];
    const float4 gg = g4[i];
    upd(pp.x, gg.x, mm.x, vv.x, decay, step_size); upd(pp.y, gg.y, mm.y, vv.y, decay, step_size);
    upd(pp.z, gg.z, mm.z, vv.z, decay, step_size); upd(pp.w, gg.w, mm.w, vv.w, decay, step_size);
    p4[i] = pp; m4[i] = mm; v4[i] = vv;
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int k = group_of(i);
    upd(p[i], g[i], m[i], v[i], s_decay[k], s_step[k]);
  }
}

// diffusers EMAModel.step: s_param.sub_(one_minus_decay * (s_param - param)), each operation rounded on its own.
// 8 B read + 4 B written per parameter.
__global__ void ema_update_kernel(float* __restrict__ ema, const float* __restrict__ p, long long n, float omd) {
  const long long n4 = n / 4;
  float4* e4 = reinterpret_cast<float4*>(ema);
  const float4* p4 = reinterpret_cast<const float4*>(p);
  auto upd = [&](float e, float q) { return __fsub_rn(e, __fmul_rn(omd, __fsub_rn(e, q))); };
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 e = e4[i];
    const float4 q = p4[i];
    e.x = upd(e.x, q.x); e.y = upd(e.y, q.y); e.z = upd(e.z, q.z); e.w = upd(e.w, q.w);
    e4[i] = e;
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    ema[i] = upd(ema[i], p[i]);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_ema_update(float* ema, const float* param, long long n, float one_minus_decay, void* stream) {
  B200_CHECK_ARG(ema && param && n > 0, "b200_ema_update: bad arguments");
  B200_CHECK_ARG((((uintptr_t)ema | (uintptr_t)param) & 15) == 0, "b200_ema_update: buffers must be 16-byte aligned");
  long long g = (n / 4 + 255) / 256;
  long long cap = (long long)sm_count() * 8;
  ema_update_kernel<<<(unsigned)(g < 1 ? 1 : (g > cap ? cap : g)), 256, 0, (cudaStream_t)stream>>>(ema, param, n,
                                                                                                    one_minus_decay);
  B200_CHECK_LAUNCH("ema_update_kernel");
  return 0;
}

extern "C" int b200_adamw_step_state_groups(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                            long long n, const long long* run_start, const int* run_group, int n_runs,
                                            const float* group_lr, const float* group_wd, int n_groups, float beta1,
                                            float beta2, float eps, const double* grad_norm_sq, float max_grad_norm,
                                            float inv_world, float* state, int dynamic_scale, float growth_interval,
                                            float min_scale, float max_scale, void* stream) {
  B200_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && grad_norm_sq && state && n > 0 && inv_world > 0.f,
                 "b200_adamw_step_state_groups: bad arguments");
  B200_CHECK_ARG((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0,
                 "b200_adamw_step_state_groups: buffers must be 16-byte aligned");
  B200_CHECK_ARG(group_lr && group_wd && n_groups >= 1 && n_groups <= B200_ADAMW_MAX_GROUPS,
                 "b200_adamw_step_state_groups: 1..%d groups with host lr / weight_decay arrays", B200_ADAMW_MAX_GROUPS);
  B200_CHECK_ARG(n_runs >= 1 && n_runs <= B200_ADAMW_MAX_RUNS && (n_runs == 1 || (run_start && run_group)),
                 "b200_adamw_step_state_groups: 1..%d runs (device run_start / run_group needed for more than one)",
                 B200_ADAMW_MAX_RUNS);
  AdamwGroupHP hp{};
  for (int k = 0; k < n_groups; ++k) { hp.lr[k] = group_lr[k]; hp.wd[k] = group_wd[k]; }
  cudaStream_t st = (cudaStream_t)stream;
  optim_prepare_kernel<<<1, 1, 0, st>>>(grad_norm_sq, state, max_grad_norm, inv_world, beta1, beta2, dynamic_scale,
                                        growth_interval, min_scale, max_scale);
  long long g = (n / 4 + 255) / 256;
  long long cap = (long long)sm_count() * 8;
  adamw_state_kernel<<<(unsigned)(g < 1 ? 1 : (g > cap ? cap : g)), 256, 0, st>>>(
      param, grad, exp_avg, exp_avg_sq, n, n_runs == 1 ? nullptr : run_start, run_group, n_runs, hp, n_groups, beta1,
      beta2, eps, state);
  B200_CHECK_LAUNCH("adamw_state_kernel");
  return 0;
}

extern "C" int b200_adamw_step_state(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                                     float lr, float beta1, float beta2, float eps, float weight_decay,
                                     const double* grad_norm_sq, float max_grad_norm, float inv_world, float* state,
                                     int dynamic_scale, float growth_interval, float min_scale, float max_scale,
                                     void* stream) {
  return b200_adamw_step_state_groups(param, grad, exp_avg, exp_avg_sq, n, nullptr, nullptr, 1, &lr, &weight_decay, 1,
                                      beta1, beta2, eps, grad_norm_sq, max_grad_norm, inv_world, state, dynamic_scale,
                                      growth_interval, min_scale, max_scale, stream);
}

extern "C" int b200_sumsq(const float* x, long long n, double* out, void* stream) {
  B200_CHECK_ARG(x && out && n > 0 && ((uintptr_t)x & 15) == 0, "b200_sumsq: bad arguments (x must be 16-byte aligned)");
  const int R = cluster_ctas(n / 4, 1024LL * 16, kMaxSingleSlotCtas);
  launch_clustered(sumsq_kernel, dim3(R), dim3(1024), 0, (cudaStream_t)stream, dim3(R, 1, 1), x, n, out);
  B200_CHECK_LAUNCH("sumsq_kernel");
  return 0;
}

extern "C" int b200_adamw_step_scaled(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                                      float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                                      const double* grad_norm_sq, float max_grad_norm, float grad_unscale,
                                      void* stream) {
  B200_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && n > 0 && step >= 1 && grad_unscale > 0.f,
                 "b200_adamw_step: bad arguments");
  const float bc1 = bias_correction(beta1, (float)step), bc2 = bias_correction(beta2, (float)step);
  long long g = (n + 255) / 256;
  long long cap = (long long)sm_count() * 8;
  adamw_kernel<<<(unsigned)(g > cap ? cap : g), 256, 0, (cudaStream_t)stream>>>(
      param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_norm_sq, max_grad_norm, grad_unscale);
  B200_CHECK_LAUNCH("adamw_kernel");
  return 0;
}

extern "C" int b200_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                               float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                               const double* grad_norm_sq, float max_grad_norm, void* stream) {
  return b200_adamw_step_scaled(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step,
                                grad_norm_sq, max_grad_norm, 1.0f, stream);
}
