// Task losses of the E2E fine-tuning step (forward): scale-and-shift-invariant L1 (depth) and angular (normals).
// Reference: training/util/loss.py:13-47 (ScaleAndShiftInvariantLoss, compute_scale_and_shift_masked) and
// :51-67 (AngularLoss), called at training/train.py:542-556.  HBM-bound masked reductions in fp64.  Every sum is
// reduced in a fixed order by one thread-block cluster per output slot (cluster_reduce.cuh): thread-sequential over a
// fixed share of the pixels, a fixed xor butterfly, the warps in index order, then the cluster's CTAs in rank order,
// added to the zeroed workspace by one plain read-modify-write.  No floating-point atomics; the grid depends only on
// the problem size, so two runs (on any H100) give the same bits.
#include "cluster_reduce.cuh"
#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

constexpr int kLossThreads = 512;

// ws[b*5 + {0..4}] += (sum m p p, sum m p, sum m, sum m p y, sum m y); grid (R, B), one cluster per image b
__global__ void __launch_bounds__(kLossThreads) ssi_moments_kernel(const float* __restrict__ pred,
                                                                   const float* __restrict__ tgt,
                                                                   const uint8_t* __restrict__ mask, long long HW,
                                                                   double* __restrict__ ws) {
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

// ws[B*5] += sum m |s p + t - y| ; ws[B*5+1] += sum m      with (s,t) the per-image least-squares fit.
// grid (R): one cluster over the whole batch, each CTA taking the same share of every image, images in order.
__global__ void __launch_bounds__(kLossThreads) ssi_l1_kernel(const float* __restrict__ pred,
                                                              const float* __restrict__ tgt,
                                                              const uint8_t* __restrict__ mask, long long HW, int B,
                                                              double* __restrict__ ws) {
  __shared__ double part[2];
  double v[2] = {0, 0};
  long long lo, hi;
  cluster_share(HW, gridDim.x, blockIdx.x, lo, hi);
  for (int b = 0; b < B; ++b) {
    const double a00 = ws[b * 5 + 0], a01 = ws[b * 5 + 1], a11 = ws[b * 5 + 2], b0 = ws[b * 5 + 3], b1 = ws[b * 5 + 4];
    const double det = a00 * a11 - a01 * a01;
    float s = 0.f, t = 0.f;                                     // loss.py:41-46: only a positive determinant is solved
    if (det > 0) { s = (float)((a11 * b0 - a01 * b1) / det); t = (float)((-a01 * b0 + a00 * b1) / det); }
    const float* p = pred + (long long)b * HW;
    const float* y = tgt + (long long)b * HW;
    const uint8_t* m = mask + (long long)b * HW;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x)
      if (m[i]) { v[0] += fabsf(s * p[i] + t - y[i]); v[1] += 1.0; }
  }
  block_sum_fixed(v, part);
  cluster_add_partials(part, 2, [&](int k) { return ws + B * 5 + k; });
}

// ws[0] += sum m acos(clamp(<p, y>)), ws[1] += sum m; grid (R): one cluster over the whole batch
__global__ void __launch_bounds__(kLossThreads) angular_kernel(const float* __restrict__ pred,
                                                               const float* __restrict__ tgt,
                                                               const uint8_t* __restrict__ mask, long long HW, int B,
                                                               double* __restrict__ ws) {
  __shared__ double part[2];
  double v[2] = {0, 0};
  long long lo, hi;
  cluster_share(HW, gridDim.x, blockIdx.x, lo, hi);
  for (int b = 0; b < B; ++b) {
    const float* p = pred + (long long)b * 3 * HW;
    const float* y = tgt + (long long)b * 3 * HW;
    const uint8_t* m = mask + (long long)b * HW;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x)
      if (m[i]) {
        float d = p[i] * y[i] + p[HW + i] * y[HW + i] + p[2 * HW + i] * y[2 * HW + i];
        d = fminf(fmaxf(d, -1.0f), 1.0f);
        v[0] += acosf(d);
        v[1] += 1.0;
      }
  }
  block_sum_fixed(v, part);
  cluster_add_partials(part, 2, [&](int k) { return ws + k; });
}

__global__ void mean_finalize_kernel(const double* __restrict__ ws, float* __restrict__ out) {
  out[0] = (float)(ws[0] / ws[1]);                            // empty mask -> nan, like torch's mean of an empty tensor
}

// Masked latent MSE of the diffusion objective (train_depth_normal.py:607-609,712-714).  One thread per latent pixel
// (b, p): the pixel is valid iff all 64 pixels of its 8x8 block of val_mask are (~max_pool2d(~val_mask, 8, 8), floor
// cropping); the mask is stored for the backward and, when valid, the squared differences of the 2 halves x C channels
// of that pixel are summed in fp64.  ws[0] += sum, ws[1] += count (exact in fp64).  grid (R): one cluster over the batch.
template <typename T>
__global__ void __launch_bounds__(kLossThreads) masked_latent_mse_kernel(const T* __restrict__ pred,
                                                                         const float* __restrict__ tgt,
                                                                         const uint8_t* __restrict__ vm, int B, int C,
                                                                         int H, int W, int h, int w,
                                                                         uint8_t* __restrict__ lm,
                                                                         double* __restrict__ ws) {
  __shared__ double part[2];
  const long long hw = (long long)h * w;
  double v[2] = {0, 0};
  long long lo, hi;
  cluster_share(hw, gridDim.x, blockIdx.x, lo, hi);
  for (int b = 0; b < B; ++b)
    for (long long p = lo + threadIdx.x; p < hi; p += blockDim.x) {
      const int y = (int)(p / w), x = (int)(p - (long long)y * w);
      const uint8_t* blk = vm + ((long long)b * H + 8 * y) * W + 8 * x;
      bool ok = true;
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int s = 0; s < 8; ++s) ok = ok && blk[(long long)r * W + s] != 0;
      lm[(long long)b * hw + p] = ok;
      if (ok) {
#pragma unroll 1
        for (int half = 0; half < 2; ++half)
          for (int c = 0; c < C; ++c) {
            const long long idx = (((long long)half * B + b) * C + c) * hw + p;
            const double d = (double)(float)pred[idx] - (double)tgt[idx];
            v[0] += d * d;
          }
        v[1] += 2.0 * C;
      }
    }
  block_sum_fixed(v, part);
  cluster_add_partials(part, 2, [&](int k) { return ws + k; });
}

__global__ void masked_mean_finalize_kernel(const double* __restrict__ ws, float* __restrict__ out) {
  out[0] = ws[1] > 0 ? (float)(ws[0] / ws[1]) : 0.0f;          // empty mask: 0, not nan
}

// grad[n][c][p] = mask ? grad_out * 2 (pred - target) / count : 0, in pred's dtype
template <typename T>
__global__ void masked_latent_mse_bwd_kernel(const T* __restrict__ pred, const float* __restrict__ tgt,
                                             const uint8_t* __restrict__ lm, const double* __restrict__ ws,
                                             const float* __restrict__ grad_out, int B, int C, long long hw,
                                             T* __restrict__ grad) {
  const double cnt = ws[1];
  const float s = cnt > 0 ? (float)(2.0 * (double)grad_out[0] / cnt) : 0.0f;
  const long long total = 2LL * B * C * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % hw;
    const int b = (int)((i / (hw * C)) % B);
    float g = 0.0f;
    if (lm[(long long)b * hw + p]) g = __fmul_rn(s, __fsub_rn((float)pred[i], tgt[i]));
    grad[i] = (T)g;
  }
}

// CTAs per cluster for a reduction over `elems` elements per slot: at least 8 elements per thread; up to 16 CTAs when
// the whole batch is one slot
static int loss_ctas(long long elems, int max_ctas) { return cluster_ctas(elems, 8LL * kLossThreads, max_ctas); }

}  // namespace b200

using namespace b200;

extern "C" int b200_ssi_loss(const float* pred, const float* target, const unsigned char* mask, int B,
                             long long HW, double* workspace, float* out, void* stream) {
  B200_CHECK_ARG(pred && target && mask && workspace && out && B > 0 && HW > 0, "b200_ssi_loss: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int R = loss_ctas(HW, kMaxClusterCtas), R1 = loss_ctas((long long)B * HW, kMaxSingleSlotCtas);
  launch_clustered(ssi_moments_kernel, dim3(R, B), dim3(kLossThreads), 0, st, dim3(R, 1, 1), pred, target, mask, HW,
                   workspace);
  launch_clustered(ssi_l1_kernel, dim3(R1), dim3(kLossThreads), 0, st, dim3(R1, 1, 1), pred, target, mask, HW, B,
                   workspace);
  mean_finalize_kernel<<<1, 1, 0, st>>>(workspace + B * 5, out);
  B200_CHECK_LAUNCH("ssi_loss kernels");
  return 0;
}

extern "C" int b200_masked_latent_mse(const void* pred, int pred_f16, const float* target, const unsigned char* val_mask,
                                      int B, int C, int H, int W, int h, int w, unsigned char* latent_mask,
                                      double* workspace, float* out, void* stream) {
  B200_CHECK_ARG(pred && target && val_mask && latent_mask && workspace && out, "b200_masked_latent_mse: null pointer");
  B200_CHECK_ARG(B >= 1 && B <= 65535 && C >= 1 && h >= 1 && w >= 1 && H >= 1 && W >= 1,
                 "b200_masked_latent_mse: bad shape B=%d C=%d H=%d W=%d h=%d w=%d", B, C, H, W, h, w);
  B200_CHECK_ARG(h == H / 8 && w == W / 8, "b200_masked_latent_mse: latent %dx%d is not the 8x8-pooled mask %dx%d",
                 h, w, H / 8, W / 8);
  cudaStream_t st = (cudaStream_t)stream;
  const int R = loss_ctas((long long)B * h * w, kMaxSingleSlotCtas);
  const dim3 grid(R), block(kLossThreads), cluster(R, 1, 1);
  if (pred_f16)
    launch_clustered(masked_latent_mse_kernel<__half>, grid, block, 0, st, cluster, (const __half*)pred, target, val_mask,
                     B, C, H, W, h, w, latent_mask, workspace);
  else
    launch_clustered(masked_latent_mse_kernel<float>, grid, block, 0, st, cluster, (const float*)pred, target, val_mask,
                     B, C, H, W, h, w, latent_mask, workspace);
  masked_mean_finalize_kernel<<<1, 1, 0, st>>>(workspace, out);
  B200_CHECK_LAUNCH("masked_latent_mse kernels");
  return 0;
}

extern "C" int b200_masked_latent_mse_bwd(const void* pred, int pred_f16, const float* target,
                                          const unsigned char* latent_mask, const double* workspace,
                                          const float* grad_out, int B, int C, long long hw, void* grad, void* stream) {
  B200_CHECK_ARG(pred && target && latent_mask && workspace && grad_out && grad, "b200_masked_latent_mse_bwd: null pointer");
  B200_CHECK_ARG(B >= 1 && C >= 1 && hw >= 1, "b200_masked_latent_mse_bwd: bad shape");
  const long long total = 2LL * B * C * hw;
  long long g = (total + 255) / 256, cap = (long long)sm_count() * 16;
  const unsigned blocks = (unsigned)(g < cap ? g : cap);
  cudaStream_t st = (cudaStream_t)stream;
  if (pred_f16)
    masked_latent_mse_bwd_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)pred, target, latent_mask, workspace,
                                                                 grad_out, B, C, hw, (__half*)grad);
  else
    masked_latent_mse_bwd_kernel<float><<<blocks, 256, 0, st>>>((const float*)pred, target, latent_mask, workspace,
                                                                grad_out, B, C, hw, (float*)grad);
  B200_CHECK_LAUNCH("masked_latent_mse_bwd_kernel");
  return 0;
}

extern "C" int b200_angular_loss(const float* pred, const float* target, const unsigned char* mask, int B,
                                 long long HW, double* workspace, float* out, void* stream) {
  B200_CHECK_ARG(pred && target && mask && workspace && out && B > 0 && HW > 0, "b200_angular_loss: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int R = loss_ctas((long long)B * HW, kMaxSingleSlotCtas);
  launch_clustered(angular_kernel, dim3(R), dim3(kLossThreads), 0, st, dim3(R, 1, 1), pred, target, mask, HW, B,
                   workspace);
  mean_finalize_kernel<<<1, 1, 0, st>>>(workspace, out);
  B200_CHECK_LAUNCH("angular_loss kernels");
  return 0;
}
