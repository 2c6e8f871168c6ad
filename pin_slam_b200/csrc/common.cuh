// Shared device/host helpers for the pinb200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/pinb200.h"
#include "knn_select.cuh"

namespace pinb {

constexpr long long PRIME0 = 73856093LL;  // model/neural_points.py:82-84
constexpr long long PRIME1 = 19349669LL;
constexpr long long PRIME2 = 83492791LL;

constexpr int TILE = 128;        // rows (queries or query-neighbour pairs) per CTA tile == threads per CTA
constexpr int ACT_LD = TILE + 1; // leading dimension of the transposed activation tile (odd => conflict-free both ways)
constexpr unsigned FULL = 0xffffffffu;
constexpr float INVALID_D2 = 9e3f;  // model/neural_points.py:583
constexpr float IDW_EPS = 1e-15f;   // model/neural_points.py:665

void set_error(const char* fmt, ...);
int check_launch(const char* what);
int sm_count();
int nccl_allreduce_sum(void* comm, float* buf, int64_t count, cudaStream_t stream);  // collective.cu

// Lets kernel `fn` use up to 227 KB of dynamic shared memory and, with `occ`, stores its resident CTAs per SM (>= 1)
// at `threads` threads and `smem_bytes` of dynamic shared memory.  The attribute and occupancy calls cost a few
// microseconds each, so they run once per (device, kernel, smem_bytes).  Returns PINB200_OK or PINB200_ERR_CUDA.
int prepare_kernel(const void* fn, const char* what, size_t smem_bytes, int threads = 0, int* occ = nullptr);

__host__ __device__ inline int align4(int x) { return (x + 3) & ~3; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}

// floor-mod of a signed 64-bit value: equals torch.fmod(v, B) followed by the
// negative-index wrap torch applies when the result is used as an index
// (model/neural_points.py:972-978).
__device__ __host__ __forceinline__ uint32_t floormod_u32(long long v, long long B) {
  long long r = v % B;
  if (r < 0) r += B;
  return (uint32_t)r;
}

// Passive rotation by the conjugate quaternion, utils/tools.py:428-437.
__device__ __forceinline__ void quat_rotate_passive(float qw, float qx, float qy, float qz, float vx,
                                                    float vy, float vz, float& ox, float& oy, float& oz) {
  const float ax = -qx, ay = -qy, az = -qz;
  const float tx = 2.f * (ay * vz - az * vy);
  const float ty = 2.f * (az * vx - ax * vz);
  const float tz = 2.f * (ax * vy - ay * vx);
  ox = vx + qw * tx + (ay * tz - az * ty);
  oy = vy + qw * ty + (az * tx - ax * tz);
  oz = vz + qw * tz + (ax * ty - ay * tx);
}
// Transpose of the above (rotation by the quaternion itself): maps a gradient
// w.r.t. the rotated vector back to the unrotated one.
__device__ __forceinline__ void quat_rotate_active(float qw, float qx, float qy, float qz, float vx,
                                                   float vy, float vz, float& ox, float& oy, float& oz) {
  quat_rotate_passive(qw, -qx, -qy, -qz, vx, vy, vz, ox, oy, oz);
}

// Lane-distributed result of the per-query neighbour search: lanes [0,K) hold
// the K nearest valid neural points in ascending distance order.
struct Knn {
  float d2;   // squared distance, INVALID_D2 if idx < 0
  int idx;    // id in the queried index space, -1 invalid
  int gidx;   // id of the same neighbour in the GLOBAL arrays (what the distance was measured to)
  int count;  // nn_counts: valid probes before top-K (warp-uniform)
};

// Precompute, once per CTA, the hash-slot delta of every probe offset:
// floormod(sum_d dx_d * prime_d, B).  slot(cell+dx) = (r0 + delta) mod B.
__device__ __forceinline__ void fill_probe_deltas(const pinb200_map_view& m, uint32_t* s_delta) {
  for (int c = threadIdx.x; c < m.n_probe; c += blockDim.x) {
    long long d = (long long)m.probe_dx[3 * c + 0] * PRIME0 + (long long)m.probe_dx[3 * c + 1] * PRIME1 +
                  (long long)m.probe_dx[3 * c + 2] * PRIME2;
    s_delta[c] = floormod_u32(d, m.buffer_size);
  }
}

__device__ __forceinline__ uint32_t base_slot(const pinb200_map_view& m, float qx, float qy, float qz) {
  // fp32 true division then floor (model/neural_points.py:963)
  const long long cx = (long long)floorf(__fdiv_rn(qx, m.resolution));
  const long long cy = (long long)floorf(__fdiv_rn(qy, m.resolution));
  const long long cz = (long long)floorf(__fdiv_rn(qz, m.resolution));
  return floormod_u32(cx * PRIME0 + cy * PRIME1 + cz * PRIME2, m.buffer_size);
}

// One probe: returns validity, squared distance and the id in the queried index space.
__device__ __forceinline__ bool probe_cell(const pinb200_map_view& m, uint32_t r0, uint32_t delta, float qx,
                                           float qy, float qz, float td_cur, float& d2, int& li, int& gi_out) {
  uint32_t slot = r0 + delta;
  if (slot >= (uint32_t)m.buffer_size) slot -= (uint32_t)m.buffer_size;
  const int gi = __ldg(m.slot_table + slot);
  gi_out = gi;
  li = -1;
  d2 = m.max_valid_dist2;
  if (gi < 0) return false;
  bool ok = true;
  if (m.time_filter) {
    const int ts = __ldg(m.ts_create + gi);
    const float dtd = fabsf(td_cur - __ldg(m.travel_dist + ts));
    ok = dtd < m.diff_travel_dist_local;  // model/neural_points.py:983-988
  }
  const float dx = __fsub_rn(__ldg(m.points + 3 * (size_t)gi + 0), qx);
  const float dy = __fsub_rn(__ldg(m.points + 3 * (size_t)gi + 1), qy);
  const float dz = __fsub_rn(__ldg(m.points + 3 * (size_t)gi + 2), qz);
  const float dd = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
  if (!ok) {  // aged out: reference sets idx=-1 first, so dist2 becomes max_valid_dist2 (:988,:996)
    gi_out = -1;
    return false;
  }
  d2 = dd;
  if (dd > m.max_valid_dist2) {  // hash collision / too far (:999)
    gi_out = -1;
    return false;
  }
  li = m.global2local ? __ldg(m.global2local + gi) : gi;
  return li >= 0;
}

// Warp-cooperative voxel-hash kNN for ONE query (all 32 lanes call this).
__device__ __forceinline__ Knn knn_search_warp(const pinb200_map_view& m, const uint32_t* s_delta, float qx,
                                               float qy, float qz, int K, int lane) {
  Knn r;
  r.d2 = INVALID_D2;
  r.idx = -1;
  r.gidx = -1;
  r.count = 0;
  const uint32_t r0 = base_slot(m, qx, qy, qz);
  const float td_cur = m.time_filter ? __ldg(m.travel_dist + m.cur_ts) : 0.f;
  const uint32_t INF_BITS = 0x7f800000u;
  for (int base = 0; base < m.n_probe; base += 32) {
    const int c = base + lane;
    bool valid = false;
    float d2 = 0.f;
    int li = -1, gi = -1;
    if (c < m.n_probe) valid = probe_cell(m, r0, s_delta[c], qx, qy, qz, td_cur, d2, li, gi);
    r.count += __popc(__ballot_sync(FULL, valid));
    uint32_t cand = valid ? __float_as_uint(d2) : INF_BITS;  // d2 >= 0: uint order == float order
    while (true) {
      const uint32_t mn = __reduce_min_sync(FULL, cand);
      if (mn == INF_BITS) break;
      const float mnf = __uint_as_float(mn);
      const float worst = __shfl_sync(FULL, r.d2, K - 1);
      if (!(mnf < worst)) break;
      const int src = __ffs(__ballot_sync(FULL, cand == mn)) - 1;
      const int cidx = __shfl_sync(FULL, li, src);
      const int cgi = __shfl_sync(FULL, gi, src);
      if (lane == src) cand = INF_BITS;
      const int pos = __popc(__ballot_sync(FULL, (lane < K) && (r.d2 <= mnf)));
      const float up_d2 = __shfl_up_sync(FULL, r.d2, 1);
      const int up_idx = __shfl_up_sync(FULL, r.idx, 1);
      const int up_gi = __shfl_up_sync(FULL, r.gidx, 1);
      if (lane > pos && lane < K) {
        r.d2 = up_d2;
        r.idx = up_idx;
        r.gidx = up_gi;
      }
      if (lane == pos) {
        r.d2 = mnf;
        r.idx = cidx;
        r.gidx = cgi;
      }
    }
  }
  if (lane >= K) {
    r.d2 = INVALID_D2;
    r.idx = -1;
    r.gidx = -1;
  }
  return r;
}

// Normalised inverse-distance weights over lanes [0,K) (model/neural_points.py:665-683).
// Returns this lane's weight; `u_out` = unnormalised 1/(d2+eps) (0 for invalid / nn_count==0).
__device__ __forceinline__ float idw_weight(float d2, bool valid, int nn_count, int K, int lane, float& u_out,
                                            float& inv_sum) {
  float u = 0.f;
  if (lane < K) {
    if (nn_count == 0)
      u = IDW_EPS;
    else if (valid)
      u = __fdiv_rn(1.0f, d2 + IDW_EPS);
  }
  const float s = warp_sum(u);
  float w = __fdiv_rn(u, s);
  if (!valid) w = 0.f;
  u_out = (valid && nn_count > 0) ? u : 0.f;
  inv_sum = 1.f / s;
  return w;
}

// Sum K (<= 8) per-lane values over the 32 lanes with 9 shuffles (vs 5 per value):
// after the call, lane l holds the warp total of value k = 4*bit4(l) + 2*bit3(l) + bit2(l).
__device__ __forceinline__ float warp_reduce8(float (&p)[8], int lane) {
  float a[4];
  {
    const bool hi = (lane & 16) != 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float send = hi ? p[i] : p[4 + i];
      const float keep = hi ? p[4 + i] : p[i];
      a[i] = keep + __shfl_xor_sync(FULL, send, 16);
    }
  }
  float b[2];
  {
    const bool hi = (lane & 8) != 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float send = hi ? a[i] : a[2 + i];
      const float keep = hi ? a[2 + i] : a[i];
      b[i] = keep + __shfl_xor_sync(FULL, send, 8);
    }
  }
  float c;
  {
    const bool hi = (lane & 4) != 0;
    const float send = hi ? b[0] : b[1];
    const float keep = hi ? b[1] : b[0];
    c = keep + __shfl_xor_sync(FULL, send, 4);
  }
  c += __shfl_xor_sync(FULL, c, 2);
  c += __shfl_xor_sync(FULL, c, 1);
  return c;
}
__device__ __forceinline__ int warp_reduce8_owner(int lane) { return ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1); }

}  // namespace pinb
