// Spatial order of a query batch for the split pipeline's search launch (query.cu: pinb200_query_sdf).
//
// Batches of random queries (bench, the mapper's replay pool) make the 32 lanes of a search tile probe 32 unrelated
// cells: every load instruction of the probe loop touches ~32 different 128-byte lines of the probe index.  Searched in
// spatial order, the lanes of a tile lie on a small patch of surface: lanes in the same cell issue the same addresses,
// neighbouring cells share lines and L1.  The order only buys locality -- it is never compared with anything, so the
// queries of one bucket may come in any order and the outputs do not depend on it.
//
// A counting sort into buckets = Morton code of the query's cell at twice the map resolution, b bits per axis
// (wrapped; b = 7 when the workspace has room for the 2^21-entry histogram, fewer otherwise), in two launches:
//   sort_key_kernel      cooperative, one grid of co-resident CTAs, phases separated by grid syncs:
//                        (a) every CTA zeroes its slice of the histogram
//                        (b) thread per query: bucket (after the optional transform), rank inside the bucket (atomicAdd)
//                        (c) every CTA scans its slice in place (exclusive) and stores the slice total in totals[]
//   sort_scatter_kernel  every CTA scans totals[] in shared memory; then thread per query:
//                        sorted[start[bucket] + slice offset + rank] = {x, y, z, query index} (the untransformed query)
// The search launch reads one 16-byte record per lane.  The histogram's size does not shrink with N, so the sort is
// bound by launch latency and by one write + one read-modify-write of the histogram, all in L2.
// (cub::DeviceRadixSort over a 30-bit key of the same order cost 50 us at 200 k queries on an H100, most of the
// search launch's gain: its onesweep passes run ~26 tiles of 7.7 k items each, latency-bound.  A memset, the key
// kernel, cub::DeviceScan's two kernels and the scatter cost 26 us.)
#include <cooperative_groups.h>

#include <algorithm>

#include "common.cuh"

namespace pinb {

constexpr int SORT_MAX_AXIS_BITS = 7;
constexpr float SORT_CELL = 2.f;      // bucket cell edge in map resolutions
constexpr int SORT_KEY_THREADS = 1024;  // 2 CTAs per SM: few CTAs make the grid syncs cheap
constexpr int SORT_SCATTER_THREADS = 256;

// bits 0..9 of v -> bits 0, 3, 6, ..., 27
__device__ __forceinline__ uint32_t morton_spread3(uint32_t v) {
  v &= 0x3ffu;
  v = (v | (v << 16)) & 0x030000ffu;
  v = (v | (v << 8)) & 0x0300f00fu;
  v = (v | (v << 4)) & 0x030c30c3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

// Exclusive prefix sum of one value per thread over the CTA (blockDim.x a multiple of 32, <= 1024); `total` = the
// CTA's sum.  Every thread of the CTA calls it; s_warp holds 33 words.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* s_warp, uint32_t& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(FULL, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    const uint32_t t = lane < nwarp ? s_warp[lane] : 0u;
    uint32_t s = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(FULL, s, o);
      if (lane >= o) s += y;
    }
    s_warp[lane] = s - t;  // exclusive prefix of the warp totals
    if (lane == 31) s_warp[32] = s;
  }
  __syncthreads();
  const uint32_t r = s_warp[warp] + x - v;
  total = s_warp[32];
  __syncthreads();  // s_warp is free for the next call
  return r;
}

// Bucket of query i: where the search looks (a1_tile: after the optional transform); any assignment would do for the
// order.
__device__ __forceinline__ uint32_t query_bucket(const float* __restrict__ xyz, const double* __restrict__ T, uint32_t i,
                                                 float inv_cell, uint32_t axis_mask) {
  const float* q = xyz + 3ull * i;
  float x = __ldg(q), y = __ldg(q + 1), z = __ldg(q + 2);
  if (T) {
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
  return morton_spread3(cx) | (morton_spread3(cy) << 1) | (morton_spread3(cz) << 2);
}

// Launched cooperatively only (grid.sync): gridDim.x CTAs, all co-resident.  The histogram has 2^(3 bits) entries in
// 2^(3 bits - slice_log2) slices of 2^slice_log2 (>= 4) entries, at most one per CTA.
__global__ void __launch_bounds__(SORT_KEY_THREADS, 2)
    sort_key_kernel(const float* __restrict__ xyz, const double* __restrict__ T, long long n, float inv_cell, int bits,
                    int slice_log2, uint32_t* __restrict__ hist, uint32_t* __restrict__ totals,
                    uint32_t* __restrict__ bucket, uint32_t* __restrict__ rank) {
  __shared__ uint32_t s_warp[33];
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  const uint32_t axis_mask = (1u << bits) - 1u;
  const int nslices = 1 << (3 * bits - slice_log2);
  const int slice4 = 1 << (slice_log2 - 2);  // uint4 per slice
  const bool has_slice = (int)blockIdx.x < nslices;
  uint4* h4 = reinterpret_cast<uint4*>(hist) + (size_t)blockIdx.x * slice4;
  // n < 2^31 (sort_queries): i + stride stays below 2^32
  const uint32_t stride = gridDim.x * blockDim.x;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  // (the grid covers a bench-sized batch in one pass: the first query's loads are in flight under the zeroing)
  uint32_t b = i < n ? query_bucket(xyz, T, i, inv_cell, axis_mask) : 0u;
  if (has_slice)
    for (int j = threadIdx.x; j < slice4; j += blockDim.x) h4[j] = make_uint4(0u, 0u, 0u, 0u);
  grid.sync();
  while (i < n) {
    bucket[i] = b;
    rank[i] = atomicAdd(hist + b, 1u);
    i += stride;
    if (i < n) b = query_bucket(xyz, T, i, inv_cell, axis_mask);
  }
  grid.sync();
  if (!has_slice) return;
  uint32_t carry = 0;
  for (int c = 0; c < slice4; c += blockDim.x) {
    const int j = c + threadIdx.x;
    const uint4 v = j < slice4 ? h4[j] : make_uint4(0u, 0u, 0u, 0u);
    uint32_t chunk;
    const uint32_t e = carry + block_exclusive_scan(v.x + v.y + v.z + v.w, s_warp, chunk);
    if (j < slice4) h4[j] = make_uint4(e, e + v.x, e + v.x + v.y, e + v.x + v.y + v.z);
    carry += chunk;
  }
  if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(SORT_SCATTER_THREADS)
    sort_scatter_kernel(const float* __restrict__ xyz, long long n, int slice_log2, int nslices,
                        const uint32_t* __restrict__ start, const uint32_t* __restrict__ totals,
                        const uint32_t* __restrict__ bucket, const uint32_t* __restrict__ rank,
                        float4* __restrict__ sorted) {
  extern __shared__ uint32_t s_off[];  // [nslices] first position of every slice
  __shared__ uint32_t s_warp[33];
  const uint32_t stride = gridDim.x * blockDim.x;  // n < 2^31: i + stride stays below 2^32
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  // everything of the first query but its slice offset is loaded before the scan of the slice totals
  uint32_t b = 0, pos = 0;
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n) {
    b = __ldg(bucket + i);
    pos = __ldg(start + b) + __ldg(rank + i);
    r = make_float4(__ldg(xyz + 3ull * i), __ldg(xyz + 3ull * i + 1), __ldg(xyz + 3ull * i + 2), __int_as_float((int)i));
  }
  // each thread sums a run of consecutive slice totals: one CTA-wide scan for any nslices
  const int per = (nslices + blockDim.x - 1) / blockDim.x, j0 = threadIdx.x * per, j1 = min(j0 + per, nslices);
  uint32_t s = 0, all;
  for (int j = j0; j < j1; ++j) s += __ldg(totals + j);
  uint32_t e = block_exclusive_scan(s, s_warp, all);
  for (int j = j0; j < j1; ++j) {
    s_off[j] = e;
    e += __ldg(totals + j);
  }
  __syncthreads();
  while (i < n) {
    sorted[pos + s_off[b >> slice_log2]] = r;
    i += stride;
    if (i < n) {
      b = __ldg(bucket + i);
      pos = __ldg(start + b) + __ldg(rank + i);
      r = make_float4(__ldg(xyz + 3ull * i), __ldg(xyz + 3ull * i + 1), __ldg(xyz + 3ull * i + 2), __int_as_float((int)i));
    }
  }
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Sorts the n queries into spatial order and sets *sorted to the queries' records {x, y, z, original index} in that
// order (inside `scratch`).  Needs two arrays of n words, the n records, the histogram and one word per CTA of the
// key launch; with less than the smallest histogram's worth of `scratch_bytes` (or more than 2^31 - 1 queries)
// *sorted stays nullptr and nothing is launched.  No allocation, no host sync.
int sort_queries(const float* xyz, const double* transform, long long n, float resolution, void* scratch,
                 size_t scratch_bytes, const float4** sorted, cudaStream_t stream) {
  *sorted = nullptr;
  if (n <= 0 || n > INT32_MAX || !(resolution > 0.f)) return PINB200_OK;
  // co-resident CTAs of the cooperative launch (the occupancy query costs microseconds: once per device and thread)
  static thread_local int occ_dev = -1, occ = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev != occ_dev) {
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, sort_key_kernel, SORT_KEY_THREADS, 0);
    if (e != cudaSuccess || occ < 1) {
      set_error("sort_key_kernel: occupancy %d: %s", occ, cudaGetErrorString(e));
      return PINB200_ERR_CUDA;
    }
    occ_dev = dev;
  }
  const int grid = occ * sm_count();
  const uintptr_t base = reinterpret_cast<uintptr_t>(scratch);
  const size_t pad = align256(base) - base, arr = align256((size_t)n * 4), rec = align256((size_t)n * 16),
               tot = align256((size_t)grid * 4);
  for (int bits = SORT_MAX_AXIS_BITS; bits >= 4; --bits) {
    const int nb = 1 << (3 * bits);
    const size_t hist_bytes = align256((size_t)nb * 4);
    if (pad + rec + 2 * arr + hist_bytes + tot > scratch_bytes) continue;
    char* s = static_cast<char*>(scratch) + pad;
    float4* out = reinterpret_cast<float4*>(s);
    uint32_t* bucket = reinterpret_cast<uint32_t*>(s + rec);
    uint32_t* rank = reinterpret_cast<uint32_t*>(s + rec + arr);
    uint32_t* hist = reinterpret_cast<uint32_t*>(s + rec + 2 * arr);
    uint32_t* totals = reinterpret_cast<uint32_t*>(s + rec + 2 * arr + hist_bytes);
    // the fewest power-of-two slices of >= 4 entries such that every slice has a CTA
    int slice_log2 = 2;
    while ((nb >> slice_log2) > grid) ++slice_log2;
    float inv_cell = 1.f / (SORT_CELL * resolution);
    void* args[] = {(void*)&xyz, (void*)&transform, (void*)&n, (void*)&inv_cell, (void*)&bits, (void*)&slice_log2,
                    (void*)&hist, (void*)&totals, (void*)&bucket, (void*)&rank};
    const cudaError_t e = cudaLaunchCooperativeKernel((const void*)sort_key_kernel, dim3(grid), dim3(SORT_KEY_THREADS),
                                                      args, 0, stream);
    if (e != cudaSuccess) {
      cudaGetLastError();
      set_error("sort_key_kernel: cooperative launch of %d CTAs: %s", grid, cudaGetErrorString(e));
      return PINB200_ERR_CUDA;
    }
    const int nslices = nb >> slice_log2;
    const int sgrid = (int)std::min<long long>((n + SORT_SCATTER_THREADS - 1) / SORT_SCATTER_THREADS, (long long)sm_count() * 8);
    sort_scatter_kernel<<<sgrid, SORT_SCATTER_THREADS, nslices * sizeof(uint32_t), stream>>>(
        xyz, n, slice_log2, nslices, hist, totals, bucket, rank, out);
    const int rc = check_launch("sort_scatter_kernel");
    if (rc) return rc;
    *sorted = out;
    return PINB200_OK;
  }
  return PINB200_OK;
}

}  // namespace pinb
