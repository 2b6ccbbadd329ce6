// Fixed-order reductions over the CTAs of a thread-block cluster (sm_90a), used by every training-path reduction that
// feeds a gradient, a loss or the gradient norm (backward.cu, loss.cu, optim.cu, gn_stats_kernel in norm.cu).
//
// Each output slot (an image's channel slice, a column slice, an image's loss moments, the gradient norm) is owned by
// ONE cluster of up to kMaxClusterCtas CTAs.  Every CTA reduces a fixed slice of the input in a fixed order into a
// partial array in its shared memory; rank 0 reads the partials of ranks 0, 1, 2, ... through distributed shared
// memory, sums them in that order and adds the total to the output with one plain read-modify-write.  A slot has a
// single writer and no floating-point atomics are involved, so the result depends only on the inputs and the shapes.
// Callers pick the grid and the cluster size from the problem size alone, never from the device's SM count, so two
// H100 variants give the same bits.  Slots that have many siblings (channel or column slices) use at most 8 CTAs, the
// portable limit; the few reductions with a single slot (the gradient norm, LayerNorm's d_gamma / d_beta, the batch
// loss sums) use up to 16, Hopper's non-portable limit, to read through more SMs.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace b200 {

constexpr int kMaxClusterCtas = 8;         // portable
constexpr int kMaxSingleSlotCtas = 16;     // non-portable, for reductions with one output slot

// CTAs per cluster for `work` units when one CTA should get at least `per_cta` of them: 1..max_ctas.
static inline int cluster_ctas(long long work, long long per_cta, int max_ctas = kMaxClusterCtas) {
  long long r = (work + per_cta - 1) / per_cta;
  return (int)(r < 1 ? 1 : (r > max_ctas ? max_ctas : r));
}

// [lo, hi): the contiguous share of [0, n) that CTA `rank` of `ranks` reduces.
__device__ __forceinline__ void cluster_share(long long n, int ranks, int rank, long long& lo, long long& hi) {
  const long long per = (n + ranks - 1) / ranks;
  lo = min(n, (long long)rank * per);
  hi = min(n, lo + per);
}

// part[0..K) (shared memory, written by this CTA before the call) -> rank 0 adds part_0[k] + part_1[k] + ... (ranks in
// order) to *dst(k).  Every thread of every CTA of the cluster must call it: it holds the two cluster barriers that
// publish the partials and keep them alive until rank 0 has read them.
template <typename T, typename Dst>
__device__ __forceinline__ void cluster_add_partials(T* part, int K, Dst dst) {
  namespace cg = cooperative_groups;
  cg::cluster_group cl = cg::this_cluster();
  const int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  const int nt = blockDim.x * blockDim.y * blockDim.z;
  if (cl.num_blocks() == 1) {                  // launched without a cluster: the CTA is the slot's only writer
    __syncthreads();
    for (int k = tid; k < K; k += nt) {
      T* o = dst(k);
      *o = *o + part[k];
    }
    return;
  }
  cl.sync();
  if (cl.block_rank() == 0) {
    const unsigned R = cl.num_blocks();
    for (int k = tid; k < K; k += nt) {
      T s = part[k];
      for (unsigned r = 1; r < R; ++r) s += cl.map_shared_rank(part, r)[k];
      T* o = dst(k);
      *o = *o + s;
    }
  }
  cl.sync();
}

// Block-wide fixed-order sum of NF per-thread values (a fixed xor butterfly over each warp, then the warps in index
// order) into part[0..NF) (shared memory) by thread 0; blockDim.x a multiple of 32, at most 1024.
template <int NF, typename T>
__device__ __forceinline__ void block_sum_fixed(T (&v)[NF], T* part) {
  __shared__ T s[32][NF];
#pragma unroll
  for (int f = 0; f < NF; ++f) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[f] += __shfl_xor_sync(0xffffffffu, v[f], o);
  }
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int f = 0; f < NF; ++f) s[warp][f] = v[f];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int f = 0; f < NF; ++f) {
      T t = s[0][f];
      for (int w = 1; w < nw; ++w) t += s[w][f];
      part[f] = t;
    }
  }
}

// Launch `kernel` with a (cx, cy, cz) cluster shape (a plain launch for 1 x 1 x 1); launch errors surface through
// cudaGetLastError as for <<<>>>.
template <typename... KArgs, typename... Args>
static inline void launch_clustered(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                    dim3 cluster, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster.x;
  attr[0].val.clusterDim.y = cluster.y;
  attr[0].val.clusterDim.z = cluster.z;
  cfg.attrs = attr;
  cfg.numAttrs = cluster.x * cluster.y * cluster.z > 1 ? 1 : 0;
  if (cluster.x * cluster.y * cluster.z > kMaxClusterCtas)
    cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace b200
