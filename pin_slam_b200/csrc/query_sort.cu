// Spatial order of a query batch for the split pipeline's search launch (query.cu: pinb200_query_sdf).
//
// Batches of random queries (bench, the mapper's replay pool) make the 32 lanes of a search tile probe 32 unrelated
// cells: every load instruction of the probe loop touches ~32 different 128-byte lines of the probe index.  Searched in
// spatial order, the lanes of a tile lie on a small patch of surface: lanes in the same cell issue the same addresses,
// neighbouring cells share lines and L1.  The order only buys locality -- it is never compared with anything, so the
// queries of one bucket may come in any order and the outputs do not depend on it.
//
// A counting sort into buckets = Morton code of the query's cell at twice the map resolution, b bits per axis
// (wrapped; b = 7 when the workspace has room for the 2^21-entry histogram, fewer otherwise):
//   memset           histogram
//   sort_key_kernel  thread per query: bucket (after the optional transform), rank inside the bucket (atomicAdd)
//   cub scan         exclusive prefix sum of the histogram, in place -> first position of every bucket
//   sort_scatter     perm[start[bucket] + rank] = query index
// (cub::DeviceRadixSort over a 30-bit key of the same order cost 50 us at 200 k queries on an H100, most of the
// search launch's gain: its onesweep passes run ~26 tiles of 7.7 k items each, latency-bound.)
#include <algorithm>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace pinb {

constexpr int SORT_MAX_AXIS_BITS = 7;
constexpr float SORT_CELL = 2.f;  // bucket cell edge in map resolutions

// bits 0..9 of v -> bits 0, 3, 6, ..., 27
__device__ __forceinline__ uint32_t morton_spread3(uint32_t v) {
  v &= 0x3ffu;
  v = (v | (v << 16)) & 0x030000ffu;
  v = (v | (v << 8)) & 0x0300f00fu;
  v = (v | (v << 4)) & 0x030c30c3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

__global__ void __launch_bounds__(256) sort_key_kernel(const float* __restrict__ xyz, const double* __restrict__ T,
                                                       long long n, float inv_cell, uint32_t axis_mask,
                                                       uint32_t* __restrict__ hist, uint32_t* __restrict__ bucket,
                                                       uint32_t* __restrict__ rank) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
    if (T) {  // where the search looks (a1_tile); any assignment would do for the order
      const float tx = fmaf(z, (float)T[2], fmaf(y, (float)T[1], x * (float)T[0])) + (float)T[3];
      const float ty = fmaf(z, (float)T[6], fmaf(y, (float)T[5], x * (float)T[4])) + (float)T[7];
      const float tz = fmaf(z, (float)T[10], fmaf(y, (float)T[9], x * (float)T[8])) + (float)T[11];
      x = tx;
      y = ty;
      z = tz;
    }
    const uint32_t cx = (uint32_t)__float2int_rd(x * inv_cell) & axis_mask,
                   cy = (uint32_t)__float2int_rd(y * inv_cell) & axis_mask,
                   cz = (uint32_t)__float2int_rd(z * inv_cell) & axis_mask;
    const uint32_t b = morton_spread3(cx) | (morton_spread3(cy) << 1) | (morton_spread3(cz) << 2);
    bucket[i] = b;
    rank[i] = atomicAdd(hist + b, 1u);
  }
}

__global__ void __launch_bounds__(256) sort_scatter_kernel(long long n, const uint32_t* __restrict__ start,
                                                           const uint32_t* __restrict__ bucket,
                                                           const uint32_t* __restrict__ rank, int32_t* __restrict__ perm) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    perm[__ldg(start + __ldg(bucket + i)) + __ldg(rank + i)] = (int32_t)i;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Sorts the n queries into spatial order and sets *perm to the sorted original indices (inside `scratch`).  Needs
// 3 arrays of n words, the histogram and the scan's temp storage; with less than the smallest histogram's worth of
// `scratch_bytes` (or more than 2^31 - 1 queries) *perm stays nullptr and nothing is launched.  No allocation, no
// host sync.
int sort_queries(const float* xyz, const double* transform, long long n, float resolution, void* scratch,
                 size_t scratch_bytes, const int32_t** perm, cudaStream_t stream) {
  *perm = nullptr;
  if (n <= 0 || n > INT32_MAX || !(resolution > 0.f)) return PINB200_OK;
  const uintptr_t base = reinterpret_cast<uintptr_t>(scratch);
  const size_t pad = align256(base) - base, arr = align256((size_t)n * 4);
  for (int bits = SORT_MAX_AXIS_BITS; bits >= 4; --bits) {
    const int nb = 1 << (3 * bits);
    size_t temp = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, temp, (uint32_t*)nullptr, nb, stream);
    if (e != cudaSuccess) {
      set_error("sort_queries: scan temp size: %s", cudaGetErrorString(e));
      return PINB200_ERR_CUDA;
    }
    const size_t hist_bytes = align256((size_t)nb * 4);
    if (pad + 3 * arr + hist_bytes + temp > scratch_bytes) continue;
    char* s = static_cast<char*>(scratch) + pad;
    int32_t* out = reinterpret_cast<int32_t*>(s);
    uint32_t* bucket = reinterpret_cast<uint32_t*>(s + arr);
    uint32_t* rank = reinterpret_cast<uint32_t*>(s + 2 * arr);
    uint32_t* hist = reinterpret_cast<uint32_t*>(s + 3 * arr);
    e = cudaMemsetAsync(hist, 0, (size_t)nb * 4, stream);
    if (e != cudaSuccess) {
      set_error("sort_queries: memset: %s", cudaGetErrorString(e));
      return PINB200_ERR_CUDA;
    }
    const int grid = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 8);
    sort_key_kernel<<<grid, 256, 0, stream>>>(xyz, transform, n, 1.f / (SORT_CELL * resolution), (1u << bits) - 1u,
                                              hist, bucket, rank);
    int rc = check_launch("sort_key_kernel");
    if (rc) return rc;
    e = cub::DeviceScan::ExclusiveSum(s + 3 * arr + hist_bytes, temp, hist, nb, stream);
    if (e != cudaSuccess) {
      set_error("sort_queries: scan: %s", cudaGetErrorString(e));
      return PINB200_ERR_CUDA;
    }
    sort_scatter_kernel<<<grid, 256, 0, stream>>>(n, hist, bucket, rank, out);
    rc = check_launch("sort_scatter_kernel");
    if (rc) return rc;
    *perm = out;
    return PINB200_OK;
  }
  return PINB200_OK;
}

}  // namespace pinb
