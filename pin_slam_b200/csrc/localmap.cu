// Local-map reset (SURVEY.md section 8 row f1): model/neural_points.py:424-513 (reset_local_map) of the reference keeps
// the neural points that are recent (travel-distance or time-stamp window; everything if fewer than 100 are recent) and
// within `local_map_radius` of the sensor, and gathers them -- ~25 torch ops and a boolean-mask compaction per tensor.
// Two entry points around the one unavoidable host sync (the local point count shapes the local tensors):
//   pinb200_local_map_select: recent flags + their count, keep flags (written as the class's `local_mask`), block sums,
//                             scan -> counts = {recent, n_local}
//   pinb200_local_map_gather: ordered scatter of the index list, global2local (incl. the reference's fill-value quirk,
//                             DESIGN.md Q1) and the gathers of positions / orientations / certainties / update stamps
#include <algorithm>

#include "scan.cuh"

namespace pinb {

constexpr int LM_TPB = 256;

struct LocalSel {
  const float* points;
  const int32_t *ts_create, *ts_update;
  const float* travel;
  long long n;
  int cur_ts, temporal_on, use_mid_ts, use_travel, diff_ts_local, reboot_map, reboot_ts, sensor_f64;
  float diff_travel, radius2_f;
  double radius2_d;
  const void* sensor;
  unsigned char* mask;  // [n+1] bool: recent flags after kernel A, keep flags after kernel B
  int* bsum;
  long long* counts;  // {recent points, local points}
};

__global__ void __launch_bounds__(LM_TPB) local_recent_kernel(const LocalSel p) {
  __shared__ int s_warp[64];
  const long long i = (long long)blockIdx.x * LM_TPB + threadIdx.x;
  int r = 0;
  if (i < p.n) {
    r = 1;
    if (p.temporal_on) {
      int ts = p.ts_create[i];
      if (p.use_mid_ts) ts = (int)(((float)ts + (float)p.ts_update[i]) / 2.f);  // ((create + update) / 2).int()
      if (p.use_travel)
        r = fabsf(__fsub_rn(p.travel[p.cur_ts], p.travel[ts])) < p.diff_travel;
      else
        r = abs(p.cur_ts - ts) < p.diff_ts_local;
      if (p.reboot_map) r = r && (ts >= p.reboot_ts);
    }
    p.mask[i] = (unsigned char)r;
  }
  int total;
  block_exclusive_scan(r, s_warp, total);
  if (threadIdx.x == 0 && total) atomicAdd(reinterpret_cast<unsigned long long*>(p.counts), (unsigned long long)total);
}

__global__ void __launch_bounds__(LM_TPB) local_keep_kernel(const LocalSel p) {
  __shared__ int s_warp[64];
  const long long i = (long long)blockIdx.x * LM_TPB + threadIdx.x;
  int k = 0;
  if (i < p.n) {
    const bool recent = p.mask[i] || (p.temporal_on && p.counts[0] < 100);  // fewer than 100 recent points: keep all
    bool near;
    if (p.sensor_f64) {  // float32 points minus a float64 sensor position: torch promotes to float64 (no DFMA)
      const double* s = reinterpret_cast<const double*>(p.sensor);
      const double dx = (double)p.points[3 * i] - s[0], dy = (double)p.points[3 * i + 1] - s[1], dz = (double)p.points[3 * i + 2] - s[2];
      near = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) < p.radius2_d;
    } else {
      const float* s = reinterpret_cast<const float*>(p.sensor);
      const float dx = __fsub_rn(p.points[3 * i], s[0]), dy = __fsub_rn(p.points[3 * i + 1], s[1]), dz = __fsub_rn(p.points[3 * i + 2], s[2]);
      near = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)) < p.radius2_f;
    }
    k = (recent && near) ? 1 : 0;
    p.mask[i] = (unsigned char)k;
  } else if (i == p.n) {
    p.mask[i] = 1;  // the padding row travels with the local map
  }
  int total;
  block_exclusive_scan(k, s_warp, total);
  if (threadIdx.x == 0) p.bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) local_scan_kernel(int* bsum, int n_blocks, long long* counts) {
  __shared__ int s_warp[64];
  int carry = 0;
  for (int base = 0; base < n_blocks; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < n_blocks ? bsum[i] : 0;
    int total;
    const int ex = block_exclusive_scan(v, s_warp, total);
    if (i < n_blocks) bsum[i] = carry + ex;
    carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[1] = carry;
}

struct LocalGather {
  const float *points, *orient, *certainty;
  const int32_t* ts_update;
  const unsigned char* mask;
  const int* bsum;
  long long n, n_local;
  int miss;
  long long* idx_pad;  // [n_local + 1]
  int32_t* g2l;        // [n + 1]
  float *l_points, *l_orient, *l_cert;
  int32_t* l_ts;
};

__global__ void __launch_bounds__(LM_TPB) local_gather_kernel(const LocalGather p) {
  __shared__ int s_warp[64];
  const long long i = (long long)blockIdx.x * LM_TPB + threadIdx.x;
  const int k = i < p.n ? p.mask[i] : 0;
  int total;
  const long long pos = (long long)p.bsum[blockIdx.x] + block_exclusive_scan(k, s_warp, total);
  if (i < p.n) {
    p.g2l[i] = k ? (int)pos : p.miss;
    if (k) {
      p.idx_pad[pos] = i;
      p.l_points[3 * pos] = p.points[3 * i];
      p.l_points[3 * pos + 1] = p.points[3 * i + 1];
      p.l_points[3 * pos + 2] = p.points[3 * i + 2];
      reinterpret_cast<float4*>(p.l_orient)[pos] = reinterpret_cast<const float4*>(p.orient)[i];
      p.l_cert[pos] = p.certainty[i];
      p.l_ts[pos] = p.ts_update[i];
    }
  } else if (i == p.n) {
    p.g2l[i] = -1;
    p.idx_pad[p.n_local] = p.n;
  }
}

}  // namespace pinb

using namespace pinb;

extern "C" int64_t pinb200_local_map_scratch(int64_t n) { return (n + 1 + LM_TPB - 1) / LM_TPB + 1; }

extern "C" int pinb200_local_map_select(const float* points, const int32_t* ts_create, const int32_t* ts_update,
                                        const float* travel_dist, int64_t n, int32_t cur_ts, int32_t temporal_on,
                                        int32_t use_mid_ts, int32_t use_travel_dist, int32_t diff_ts_local, int32_t reboot_map,
                                        int32_t reboot_ts, float diff_travel, const void* sensor_pos, int32_t sensor_is_f64,
                                        double radius2, uint8_t* local_mask, int32_t* scratch, int64_t* counts, void* stream) {
  // an empty map (torch gives its tensors a null data pointer) still writes the padding row's mask and the counts
  if ((n > 0 && !points) || !sensor_pos || !local_mask || !scratch || !counts || n < 0 ||
      (temporal_on && n > 0 && (!ts_create || (use_mid_ts && !ts_update) || (use_travel_dist && !travel_dist)))) {
    set_error("local_map_select: bad argument");
    return PINB200_ERR_BAD_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(counts, 0, 16, st);
  LocalSel p{};
  p.points = points;
  p.ts_create = ts_create;
  p.ts_update = ts_update;
  p.travel = travel_dist;
  p.n = n;
  p.cur_ts = cur_ts;
  p.temporal_on = temporal_on;
  p.use_mid_ts = use_mid_ts;
  p.use_travel = use_travel_dist;
  p.diff_ts_local = diff_ts_local;
  p.reboot_map = reboot_map;
  p.reboot_ts = reboot_ts;
  p.sensor_f64 = sensor_is_f64;
  p.diff_travel = diff_travel;
  p.radius2_f = (float)radius2;
  p.radius2_d = radius2;
  p.sensor = sensor_pos;
  p.mask = local_mask;
  p.bsum = scratch;
  p.counts = reinterpret_cast<long long*>(counts);
  const int n_blocks = (int)((n + 1 + LM_TPB - 1) / LM_TPB);
  if (n > 0) local_recent_kernel<<<n_blocks, LM_TPB, 0, st>>>(p);
  local_keep_kernel<<<n_blocks, LM_TPB, 0, st>>>(p);
  local_scan_kernel<<<1, 1024, 0, st>>>(scratch, n_blocks, p.counts);
  return check_launch("local_map_select");
}

extern "C" int pinb200_local_map_gather(const float* points, const float* orient, const float* certainty,
                                        const int32_t* ts_update, const uint8_t* local_mask, const int32_t* scratch, int64_t n,
                                        int64_t n_local, int32_t miss_value, int64_t* idx_pad, int32_t* global2local,
                                        float* l_points, float* l_orient, float* l_certainty, int32_t* l_ts_update,
                                        void* stream) {
  if ((n > 0 && (!points || !orient || !certainty || !ts_update)) || !local_mask || !scratch || !idx_pad ||
      !global2local || n < 0 ||
      n_local < 0 || (n_local > 0 && (!l_points || !l_orient || !l_certainty || !l_ts_update))) {
    set_error("local_map_gather: bad argument");
    return PINB200_ERR_BAD_ARG;
  }
  LocalGather p{points, orient, certainty, ts_update, local_mask, scratch, n, n_local, miss_value,
                reinterpret_cast<long long*>(idx_pad), global2local, l_points, l_orient, l_certainty, l_ts_update};
  const int n_blocks = (int)((n + 1 + LM_TPB - 1) / LM_TPB);
  local_gather_kernel<<<n_blocks, LM_TPB, 0, (cudaStream_t)stream>>>(p);
  return check_launch("local_map_gather");
}
