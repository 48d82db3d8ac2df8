// block_scan.h — the block-wide prefix sum of the CUDA kernels (device code only): warp scans, then every warp scans the warp
// totals and takes its own prefix by shuffle.
#pragma once
#include <cstdint>

namespace horae {

// inclusive scan of one value per lane across lanes [0, W) of the calling warp (all 32 lanes call it)
template <int W = 32>
__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
  for (int d = 1; d < W; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += t;
  }
  return v;
}

// Exclusive scan of one value per thread across an NT-thread block (every thread calls it); returns the thread's exclusive
// prefix, *total = the block sum.  s_w: NT / 32 + 1 words of shared memory.  Ends with a barrier, so the caller may call it
// again with the same s_w right away.
template <int NT>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total, uint32_t* s_w) {
  static_assert(NT % 32 == 0 && NT <= 1024, "one warp scans the warp totals");
  constexpr int kWarps = NT / 32;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const uint32_t inc = warp_incl_scan(v, lane);
  if (lane == 31) s_w[w] = inc;
  __syncthreads();
  const uint32_t x = lane < kWarps ? s_w[lane] : 0;       // every warp scans the warp totals
  const uint32_t xi = warp_incl_scan<kWarps>(x, lane);
  const uint32_t before = __shfl_sync(0xffffffffu, xi - x, w);
  *total = __shfl_sync(0xffffffffu, xi, kWarps - 1);
  __syncthreads();
  return before + inc - v;
}

}  // namespace horae
