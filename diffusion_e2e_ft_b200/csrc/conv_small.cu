// 3x3 convolution (stride 1, pad 1) with a tiny number of output channels (Cout <= 8): the UNet / VAE
// `conv_out` layers (320->4, 128->3, 512->8).  With N <= 8 the wgmma implicit GEMM is bound by
// re-fetching every activation tile nine times through L2; this
// kernel stages a halo tile in shared memory once per 64-channel chunk and reuses it for all nine taps.
// HBM-bound: reads the NHWC fp16 input exactly once, writes NCHW fp32.
// Tensor work is negligible (N padded to 8) and runs on mma.sync m16n8k16 (fp16 in, fp32 accumulate).
#include "common.cuh"
#include "../../include/b200_e2eft.h"

namespace b200 {

constexpr int kTH = 8, kTW = 32, kCC = 64;                 // tile rows / cols, channels per chunk
constexpr int kPixStride = kCC * 2 + 16;                  // bytes per halo pixel (+16 pad: conflict-free ldmatrix)
constexpr int kHaloBytes = (kTH + 2) * (kTW + 2) * kPixStride;
constexpr int kWChunkBytes = 9 * (kCC / 16) * 8 * 16 * 2;  // [tap][kstep][n=8][k=16] fp16
constexpr int kSmallSmem = kHaloBytes + kWChunkBytes;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int bytes = valid ? 16 : 0;                         // src-size 0 -> zero fill (conv padding)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(256, 2)
conv3x3_small_cout_kernel(const __half* __restrict__ x, int H, int W, int C,
                          const __half* __restrict__ wq, const float* __restrict__ bias, int Cout,
                          float* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t sm[];
  uint8_t* halo = sm;
  uint8_t* wsm = sm + kHaloBytes;
  const uint32_t halo_u = smem_u32(halo), wsm_u = smem_u32(wsm);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int w0 = blockIdx.x * kTW, h0 = blockIdx.y * kTH, n = blockIdx.z;
  const __half* xn = x + (long long)n * H * W * C;
  float acc[2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int g = lane >> 2, t = lane & 3;
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8;     // ldmatrix.x4 row supplied by this lane
  const int a_khalf = lane >> 4;

  for (int c0 = 0; c0 < C; c0 += kCC) {
    // ---- stage the halo tile (zero-filled outside the image) and this chunk's weights
    for (int i = tid; i < (kTH + 2) * (kTW + 2) * (kCC / 8); i += 256) {
      const int v = i % (kCC / 8);
      const int pix = i / (kCC / 8);
      const int pw = pix % (kTW + 2), ph = pix / (kTW + 2);
      const int hh = h0 + ph - 1, ww = w0 + pw - 1;
      const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W;
      const __half* src = ok ? xn + ((long long)hh * W + ww) * C + c0 + v * 8 : xn;
      cp_async16(halo_u + pix * kPixStride + v * 16, src, ok);
    }
    const __half* wsrc = wq + (long long)(c0 / kCC) * (kWChunkBytes / 2);
    for (int i = tid; i < kWChunkBytes / 16; i += 256) cp_async16(wsm_u + i * 16, wsrc + i * 8, true);
    asm volatile("cp.async.commit_group;\n cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    // ---- warp `warp` owns tile row `warp`: two 16-pixel m-tiles, all 9 taps x 4 k-steps
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int dy = tap / 3, dx = tap % 3;                 // halo coordinates already include the -1
#pragma unroll
      for (int ks = 0; ks < kCC / 16; ++ks) {
        const uint32_t baddr = wsm_u + ((tap * (kCC / 16) + ks) * 8 + g) * 32 + t * 4;
        uint32_t b0, b1;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b0) : "r"(baddr));
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b1) : "r"(baddr + 16));
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const int pw = mt * 16 + a_row + dx;
          const uint32_t aaddr = halo_u + ((warp + dy) * (kTW + 2) + pw) * kPixStride + ks * 32 + a_khalf * 16;
          uint32_t a0, a1, a2, a3;
          asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                       : "=r"(a0), "=r"(a1), "=r"(a2), "=r"(a3) : "r"(aaddr));
          asm volatile(
              "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
              : "+f"(acc[mt][0]), "+f"(acc[mt][1]), "+f"(acc[mt][2]), "+f"(acc[mt][3])
              : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
        }
      }
    }
    __syncthreads();
  }
  // ---- epilogue: c0,c1 -> (pixel g, cout 2t, 2t+1); c2,c3 -> pixel g+8
  const int hh = h0 + warp;
  if (hh < H) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int co = 2 * t + (j & 1);
        const int ww = w0 + mt * 16 + g + (j >> 1) * 8;
        if (co < Cout && ww < W)
          out[(((long long)n * Cout + co) * H + hh) * W + ww] = acc[mt][j] + (bias ? bias[co] : 0.f);
      }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_conv3x3_small_cout(const void* x, int NB, int H, int W, int C, const void* wq,
                                       const float* bias, int Cout, float* out, void* stream) {
  B200_CHECK_ARG(x && wq && out && NB > 0 && H > 0 && W > 0, "b200_conv3x3_small_cout: bad arguments");
  B200_CHECK_ARG(C % kCC == 0 && Cout >= 1 && Cout <= 8, "b200_conv3x3_small_cout: C=%d must be a multiple of 64, Cout=%d <= 8", C, Cout);
  B200_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)wq & 15) == 0, "b200_conv3x3_small_cout: 16-byte alignment");
  static bool configured_dev[kMaxDevices] = {false};      // per device: function attributes live in the context
  const int dev_ = current_device();
  bool& configured = configured_dev[dev_ < 0 ? 0 : dev_];
  if (!configured || dev_ < 0) {
    cudaError_t e = cudaFuncSetAttribute(conv3x3_small_cout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmallSmem);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(conv_small smem=%d): %s", kSmallSmem, cudaGetErrorString(e));
      return (int)e;
    }
    configured = true;
  }
  dim3 grid((W + kTW - 1) / kTW, (H + kTH - 1) / kTH, NB);
  conv3x3_small_cout_kernel<<<grid, 256, kSmallSmem, (cudaStream_t)stream>>>(
      (const __half*)x, H, W, C, (const __half*)wq, bias, Cout, out);
  B200_CHECK_LAUNCH("conv3x3_small_cout_kernel");
  return 0;
}
