// Replay-pool window filter (SURVEY.md section 8 row f2): utils/mapper.py:404-438 of the reference keeps the samples
// within `window_radius` of the sensor with boolean-mask indexing of five (six with colour) pool tensors -- five
// reallocations of ~5 M-row tensors per frame, which on the benchmark loop cost tens of milliseconds of allocator
// time.  Here the pool lives in two fixed-capacity arenas (pin_slam_b200/utils/mapper.py: _PoolArena) and the filter
// is ONE order-preserving compaction from one arena into the other: flags + block sums, a scan of the block sums,
// and a scatter of all arrays.  The distance test uses the reference's arithmetic (the pool is fp32, the sensor
// origin fp64: torch promotes the difference to fp64), every product and sum rounded on its own: a contracted DFMA
// would decide samples within an ulp of the radius differently from torch.
#include <algorithm>

#include "scan.cuh"

namespace pinb {

constexpr int PF_TPB = 256;
constexpr int PF_IPT = 4;  // items per thread
constexpr int PF_IPB = PF_TPB * PF_IPT;

struct PoolPtrs {
  const float *coord, *gcoord, *label, *weight, *color;
  const int32_t* ts;
  float *o_coord, *o_gcoord, *o_label, *o_weight, *o_color;
  int32_t* o_ts;
  int cc;
};

__device__ __forceinline__ bool pool_keep(const float* __restrict__ g, long long i, const double* __restrict__ origin,
                                          double r2) {
  const double dx = (double)g[3 * i] - origin[0], dy = (double)g[3 * i + 1] - origin[1], dz = (double)g[3 * i + 2] - origin[2];
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) < r2;
}

__global__ void __launch_bounds__(PF_TPB) pool_count_kernel(const float* __restrict__ gcoord, long long n,
                                                            const double* __restrict__ origin, double r2, int* bsum) {
  __shared__ int s_warp[64];
  const long long i0 = (long long)blockIdx.x * PF_IPB + threadIdx.x * PF_IPT;
  int c = 0;
#pragma unroll
  for (int j = 0; j < PF_IPT; ++j)
    if (i0 + j < n && pool_keep(gcoord, i0 + j, origin, r2)) ++c;
  int total;
  block_exclusive_scan(c, s_warp, total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) pool_scan_kernel(int* bsum, int n_blocks, long long* counts) {
  const long long kept = scan_block_sums(bsum, bsum, n_blocks);
  if (threadIdx.x == 0) counts[0] = kept;  // counts[1] (kept among the last n_tail) is set by the scatter
}

__global__ void __launch_bounds__(PF_TPB) pool_scatter_kernel(const PoolPtrs p, long long n, long long n_tail,
                                                              const double* __restrict__ origin, double r2,
                                                              const int* __restrict__ bsum, long long* counts) {
  __shared__ int s_warp[64];
  const long long i0 = (long long)blockIdx.x * PF_IPB + threadIdx.x * PF_IPT;
  bool k[PF_IPT];
  int c = 0;
#pragma unroll
  for (int j = 0; j < PF_IPT; ++j) {
    k[j] = i0 + j < n && pool_keep(p.gcoord, i0 + j, origin, r2);
    c += k[j] ? 1 : 0;
  }
  int total;
  long long pos = (long long)bsum[blockIdx.x] + block_exclusive_scan(c, s_warp, total);
#pragma unroll
  for (int j = 0; j < PF_IPT; ++j) {
    const long long i = i0 + j;
    if (i == n - n_tail) counts[1] = counts[0] - pos;  // kept samples from the first "fresh" one on
    if (!k[j]) continue;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      p.o_coord[3 * pos + a] = p.coord[3 * i + a];
      p.o_gcoord[3 * pos + a] = p.gcoord[3 * i + a];
    }
    p.o_label[pos] = p.label[i];
    p.o_weight[pos] = p.weight[i];
    p.o_ts[pos] = p.ts[i];
    for (int a = 0; a < p.cc; ++a) p.o_color[pos * p.cc + a] = p.color[i * p.cc + a];
    ++pos;
  }
}

}  // namespace pinb

using namespace pinb;

extern "C" int64_t pinb200_pool_filter_scratch(int64_t n) { return (n + PF_IPB - 1) / PF_IPB + 1; }

extern "C" int pinb200_pool_filter(const float* coord, const float* gcoord, const float* label, const float* weight,
                                   const int32_t* ts, const float* color, int32_t color_channels, int64_t n,
                                   int64_t n_tail, const double* origin, double radius2, float* o_coord, float* o_gcoord,
                                   float* o_label, float* o_weight, int32_t* o_ts, float* o_color, int32_t* scratch,
                                   int64_t* counts, void* stream) {
  if (!coord || !gcoord || !label || !weight || !ts || !origin || !o_coord || !o_gcoord || !o_label || !o_weight || !o_ts ||
      !scratch || !counts || n < 0 || n_tail < 0 || n_tail > n || (color_channels > 0 && (!color || !o_color))) {
    set_error("pool_filter: bad argument");
    return PINB200_ERR_BAD_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    cudaMemsetAsync(counts, 0, 16, st);
    return PINB200_OK;
  }
  const int n_blocks = (int)((n + PF_IPB - 1) / PF_IPB);
  PoolPtrs p{coord, gcoord, label, weight, color, ts, o_coord, o_gcoord, o_label, o_weight, o_color, o_ts, color_channels};
  cudaMemsetAsync(counts, 0, 16, st);
  pool_count_kernel<<<n_blocks, PF_TPB, 0, st>>>(gcoord, n, origin, radius2, scratch);
  pool_scan_kernel<<<1, 1024, 0, st>>>(scratch, n_blocks, (long long*)counts);
  pool_scatter_kernel<<<n_blocks, PF_TPB, 0, st>>>(p, n, n_tail, origin, radius2, scratch, (long long*)counts);
  return check_launch("pool_filter");
}
