// Block-wide exclusive prefix sum used by the compaction-style kernels (probe index, replay-pool filter, local map,
// marching cubes).
#pragma once
#include "common.cuh"

namespace pinb {

// every thread of the block calls it; `s_warp` = 64 ints of shared memory; returns the exclusive prefix of `v` over
// the block in thread order and the block total
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(FULL, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = lane < (blockDim.x >> 5) ? s_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(FULL, w, o);
      if (lane >= o) w += t;
    }
    s_warp[32 + lane] = w;  // inclusive over warps
  }
  __syncthreads();
  total = s_warp[32 + (blockDim.x >> 5) - 1];
  const int warp_off = warp == 0 ? 0 : s_warp[32 + warp - 1];
  return warp_off + inc - v;
}

// one block of blockDim.x (a multiple of 32, <= 1024) threads turns the per-block counts `in` [n_blocks] of a
// count-then-scatter pair of kernels into exclusive offsets `out` (may alias `in`) and returns the grand total to every
// thread; the running total is 64-bit, the partial sums of one pass over blockDim.x counts are not
template <typename T>
__device__ long long scan_block_sums(const int* in, T* out, int n_blocks) {
  __shared__ int s_warp[64];
  long long carry = 0;
  for (int base = 0; base < n_blocks; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int v = i < n_blocks ? in[i] : 0;
    int total;
    const int ex = block_exclusive_scan(v, s_warp, total);
    if (i < n_blocks) out[i] = (T)(carry + ex);
    carry += total;
    __syncthreads();
  }
  return carry;
}

}  // namespace pinb
