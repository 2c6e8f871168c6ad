// Frame preparation (DESIGN.md row f6): the point work of SLAMDataset.preprocess_frame after the voxel down-sampling
// (dataset/slam_dataset.py:437-439 gathers, :1229-1248 crop_frame, :1251-1270 intrinsic_correct) and the deskewing of
// utils/tools.py:747-779, which the reference does with roma.rotmat_slerp.
//
// Crop: one order-preserving compaction over the down-sampling index, as in pool.cu: per-block survivor counts ->
// scan of the block sums (scan.cuh) -> scatter of the surviving rows, corrected on the way.  The range and the
// correction use the reference's fp32 arithmetic with every product and sum rounded on its own (a contracted FMA
// would decide rows within an ulp of a bound differently from torch.norm).
//
// Deskew: launch 1 reduces min/max of the timestamps into a two-float scratch (one block: no atomics, no memset);
// launch 2 moves every point by exp(s log R) p + s t, s = (ts - min) / (max - min) - ts_mid.  log R is the shortest-arc
// rotation vector of the fp32 pose, computed in fp64 once per block; per point, Rodrigues' formula in fp32 with a
// series for small angles.  Reproduced on purpose: all-equal timestamps give s = 0/0 = NaN (as torch does), and the
// identity pose adds exact zeros, so it leaves the points bit-identical.
#include "../scan.cuh"

namespace pinb {

constexpr int FP_TPB = 256;
constexpr int FP_IPT = 4;  // index entries per thread
constexpr int FP_IPB = FP_TPB * FP_IPT;
constexpr int DS_TPB = 256;

struct CropArgs {
  const float* points;
  const float* ts;
  const int64_t* index;
  long long m;
  int cols;
  float min_z, max_z, min_range, max_range;
};

// row j kept iff min_range < r < max_range and min_z < z < max_z, r = |xyz| in fp32 (torch.norm of three floats)
__device__ __forceinline__ bool crop_keep(const CropArgs& a, long long j, float& r) {
  const float* p = a.points + j * a.cols;
  const float x = p[0], y = p[1], z = p[2];
  r = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
  return r > a.min_range && r < a.max_range && z > a.min_z && z < a.max_z;
}

__global__ void __launch_bounds__(FP_TPB) crop_count_kernel(const CropArgs a, int* bsum) {
  __shared__ int s_warp[64];
  const long long i0 = (long long)blockIdx.x * FP_IPB + threadIdx.x;
  int c = 0;
#pragma unroll
  for (int k = 0; k < FP_IPT; ++k) {
    const long long i = i0 + k * FP_TPB;
    float r;
    if (i < a.m && crop_keep(a, a.index[i], r)) ++c;
  }
  int total;
  block_exclusive_scan(c, s_warp, total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) crop_scan_kernel(int* bsum, int n_blocks, long long* n_kept) {
  const long long kept = scan_block_sums(bsum, bsum, n_blocks);
  if (threadIdx.x == 0) *n_kept = kept;
}

// thread t owns the FP_IPT consecutive index entries from i0, so that survivors are written in index order (the count
// kernel strides by FP_TPB for coalesced index loads: it only needs the block total)
__global__ void __launch_bounds__(FP_TPB) crop_scatter_kernel(const CropArgs a, const int* __restrict__ bsum,
                                                              float corr, float* out, float* ts_out) {
  __shared__ int s_warp[64];
  const long long i0 = (long long)blockIdx.x * FP_IPB + (long long)threadIdx.x * FP_IPT;
  int keep = 0;  // bit k: entry i0 + k survives
#pragma unroll
  for (int k = 0; k < FP_IPT; ++k) {
    float r;
    if (i0 + k < a.m && crop_keep(a, a.index[i0 + k], r)) keep |= 1 << k;
  }
  int total;
  long long pos = (long long)bsum[blockIdx.x] + block_exclusive_scan(__popc(keep), s_warp, total);
#pragma unroll
  for (int k = 0; k < FP_IPT; ++k) {
    if (!(keep >> k & 1)) continue;
    const long long j = a.index[i0 + k];
    const float* p = a.points + j * a.cols;
    float* o = out + pos * a.cols;
    float x = p[0], y = p[1], z = p[2];
    if (corr != 0.f) {  // intrinsic_correct: v = asin(z / r), vc = v + corr
      float r;
      crop_keep(a, j, r);
      const float v = asinf(__fdiv_rn(z, r));
      const float vc = __fadd_rn(v, corr);
      const float s = __fdiv_rn(cosf(vc), cosf(v));
      x = __fmul_rn(x, s);
      y = __fmul_rn(y, s);
      z = __fmul_rn(r, sinf(vc));
    }
    o[0] = x;
    o[1] = y;
    o[2] = z;
    for (int c2 = 3; c2 < a.cols; ++c2) o[c2] = p[c2];
    if (ts_out) ts_out[pos] = a.ts[j];
    ++pos;
  }
}

// one block: mm[0] = min(ts), mm[1] = max(ts)
__global__ void __launch_bounds__(1024) deskew_minmax_kernel(const float* __restrict__ ts, long long n, float* mm) {
  __shared__ float s_lo[32], s_hi[32];
  float lo = INFINITY, hi = -INFINITY;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float t = ts[i];
    lo = fminf(lo, t);
    hi = fmaxf(hi, t);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(FULL, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(FULL, hi, o));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_lo[warp] = lo;
    s_hi[warp] = hi;
  }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    lo = lane < nw ? s_lo[lane] : INFINITY;
    hi = lane < nw ? s_hi[lane] : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = fminf(lo, __shfl_xor_sync(FULL, lo, o));
      hi = fmaxf(hi, __shfl_xor_sync(FULL, hi, o));
    }
    if (lane == 0) {
      mm[0] = lo;
      mm[1] = hi;
    }
  }
}

// shortest-arc rotation vector of the (nearly orthonormal) fp32 rotation block of `pose` [4,4] row-major, in fp64:
// quaternion by the largest of (trace, diagonal) (Shepperd), normalised, w >= 0, then 2 atan2(|v|, w) v / |v|
__device__ void rotation_log(const float* __restrict__ pose, double w_out[3]) {
  double R[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r][c] = pose[4 * r + c];
  const double tr = R[0][0] + R[1][1] + R[2][2];
  double q[4];  // w, x, y, z
  if (tr >= R[0][0] && tr >= R[1][1] && tr >= R[2][2]) {
    const double s = 2.0 * sqrt(1.0 + tr);
    q[0] = 0.25 * s, q[1] = (R[2][1] - R[1][2]) / s, q[2] = (R[0][2] - R[2][0]) / s, q[3] = (R[1][0] - R[0][1]) / s;
  } else if (R[0][0] >= R[1][1] && R[0][0] >= R[2][2]) {
    const double s = 2.0 * sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]);
    q[0] = (R[2][1] - R[1][2]) / s, q[1] = 0.25 * s, q[2] = (R[0][1] + R[1][0]) / s, q[3] = (R[0][2] + R[2][0]) / s;
  } else if (R[1][1] >= R[2][2]) {
    const double s = 2.0 * sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]);
    q[0] = (R[0][2] - R[2][0]) / s, q[1] = (R[0][1] + R[1][0]) / s, q[2] = 0.25 * s, q[3] = (R[1][2] + R[2][1]) / s;
  } else {
    const double s = 2.0 * sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]);
    q[0] = (R[1][0] - R[0][1]) / s, q[1] = (R[0][2] + R[2][0]) / s, q[2] = (R[1][2] + R[2][1]) / s, q[3] = 0.25 * s;
  }
  const double qn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double sg = q[0] < 0.0 ? -1.0 / qn : 1.0 / qn;
  const double w = q[0] * sg, x = q[1] * sg, y = q[2] * sg, z = q[3] * sg;
  const double vn = sqrt(x * x + y * y + z * z);
  const double f = vn > 0.0 ? 2.0 * atan2(vn, w) / vn : 0.0;
  w_out[0] = f * x, w_out[1] = f * y, w_out[2] = f * z;
}

__global__ void __launch_bounds__(DS_TPB) deskew_apply_kernel(float* points, long long stride, const float* __restrict__ ts,
                                                              long long n, const float* __restrict__ pose, float ts_mid,
                                                              const float* __restrict__ mm) {
  __shared__ float s_w[3];
  if (threadIdx.x == 0) {
    double w[3];
    rotation_log(pose, w);
    s_w[0] = (float)w[0], s_w[1] = (float)w[1], s_w[2] = (float)w[2];
  }
  __syncthreads();
  const long long i = (long long)blockIdx.x * DS_TPB + threadIdx.x;
  if (i >= n) return;
  const float wx = s_w[0], wy = s_w[1], wz = s_w[2];
  const float tx = pose[3], ty = pose[7], tz = pose[11];
  const float lo = mm[0], hi = mm[1];
  // torch: ts = (ts - min) / (max - min); ts -= ts_mid
  const float s = __fsub_rn(__fdiv_rn(__fsub_rn(ts[i], lo), __fsub_rn(hi, lo)), ts_mid);
  float* p = points + i * stride;
  const float px = p[0], py = p[1], pz = p[2];
  const float fx = s * wx, fy = s * wy, fz = s * wz;  // phi = s log R, theta = |phi|
  const float th2 = fx * fx + fy * fy + fz * fz;
  const float th = sqrtf(th2);
  float A, B;  // R(phi) = I + A [phi]x + B [phi]x^2
  if (th < 1e-2f) {
    A = 1.f - th2 * (1.f / 6.f) * (1.f - th2 * (1.f / 20.f));
    B = 0.5f - th2 * (1.f / 24.f) * (1.f - th2 * (1.f / 30.f));
  } else {
    float sh, ch;
    sincosf(0.5f * th, &sh, &ch);
    A = 2.f * sh * ch / th;        // sin(theta) / theta
    B = 2.f * sh * sh / th2;       // (1 - cos(theta)) / theta^2 without the cancellation
  }
  const float cx = fy * pz - fz * py, cy = fz * px - fx * pz, cz = fx * py - fy * px;  // phi x p
  const float dx = fy * cz - fz * cy, dy = fz * cx - fx * cz, dz = fx * cy - fy * cx;  // phi x (phi x p)
  p[0] = px + (A * cx + B * dx + s * tx);
  p[1] = py + (A * cy + B * dy + s * ty);
  p[2] = pz + (A * cz + B * dz + s * tz);
}

}  // namespace pinb

using namespace pinb;

extern "C" int pinb200_frame_crop(const float* points, int64_t n, int32_t cols, const int64_t* index, int64_t m,
                                  const float* ts, float min_z, float max_z, float min_range, float max_range,
                                  double correction_deg, int32_t* scratch, int64_t scratch_len, int64_t* n_kept,
                                  float* points_out, float* ts_out, void* stream) {
  const long long n_blocks = (m + FP_IPB - 1) / FP_IPB;
  if ((n > 0 && !points) || (m > 0 && !index) || n < 0 || m < 0 || cols < 3 || cols > 7 || !n_kept ||
      (m > 0 && (!points_out || !scratch || scratch_len < n_blocks || (ts == nullptr) != (ts_out == nullptr))) ||
      n_blocks > INT32_MAX) {
    set_error("frame_crop: bad argument");
    return PINB200_ERR_BAD_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (m == 0) {
    cudaMemsetAsync(n_kept, 0, sizeof(int64_t), st);
    return check_launch("frame_crop");
  }
  // the Python scalar correct_deg / 180 * pi, rounded once to the points' fp32 (slam_dataset.py:1261)
  const float corr = (float)(correction_deg / 180.0 * 3.141592653589793);
  const CropArgs a{points, ts, index, m, cols, min_z, max_z, min_range, max_range};
  crop_count_kernel<<<(unsigned)n_blocks, FP_TPB, 0, st>>>(a, scratch);
  crop_scan_kernel<<<1, 1024, 0, st>>>(scratch, (int)n_blocks, (long long*)n_kept);
  crop_scatter_kernel<<<(unsigned)n_blocks, FP_TPB, 0, st>>>(a, scratch, corr, points_out, ts_out);
  return check_launch("frame_crop");
}

extern "C" int pinb200_deskew(float* points, int64_t n, int64_t row_stride, const float* ts, const float* pose,
                              float ts_mid, float* scratch, void* stream) {
  if (n < 0 || (n > 0 && (!points || !ts || !pose || !scratch)) || row_stride < 3) {
    set_error("deskew: bad argument");
    return PINB200_ERR_BAD_ARG;
  }
  if (n == 0) return PINB200_OK;
  cudaStream_t st = (cudaStream_t)stream;
  deskew_minmax_kernel<<<1, 1024, 0, st>>>(ts, n, scratch);
  deskew_apply_kernel<<<(unsigned)((n + DS_TPB - 1) / DS_TPB), DS_TPB, 0, st>>>(points, row_stride, ts, n, pose, ts_mid,
                                                                                scratch);
  return check_launch("deskew");
}
