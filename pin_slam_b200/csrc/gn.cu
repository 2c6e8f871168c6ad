// K4: point-to-implicit registration step.
//   pass 1 (gn_accumulate_kernel): per source point validity mask, Geman-McClure
//          robust weights and the 6x6 normal equations J^T W J / -J^T W r, reduced
//          warp -> block -> fp64 atomics (27 unique scalars + 4 counters);
//   pass 2 (gn_solve): weight normalisation w /= 2 mean(w), LM damping, fp64 6x6 solve,
//          expmap, T <- dT @ T -- run by the LAST block of pass 1 to finish (threadfence +
//          ticket counter), so a registration step is one launch; gn_solve_kernel remains
//          for the empty-input case.
// Replaces utils/tracker.py:409-524 (registration_step) and :652-679 (implicit_reg)
// without any host synchronisation.
#include <algorithm>
#include <math.h>

#include "common.cuh"

namespace pinb {

constexpr int GN_NSUM = 46;    // 36 N + 6 g + sum_w + sum|r| + count + sum w r^2
constexpr int GN_TICKET = 63;  // sums[63] (zeroed with the sums): finished-block counter of the fused solve
__device__ void gn_solve(const double* sums, float lm_lambda, double* __restrict__ result, double* __restrict__ t_inout);
__device__ __forceinline__ void gn_finish(double* sums, float lm_lambda, double* result, double* t_inout);

__global__ void __launch_bounds__(256) gn_accumulate_kernel(
    const float* __restrict__ xyz, const float* __restrict__ sdf, const float* __restrict__ grad,
    const float* __restrict__ sdf_std, const int32_t* __restrict__ nn_count, const float* __restrict__ sdf_label,
    const float* __restrict__ normals, long long n, int min_nn, float min_gn, float max_gn, float max_std,
    float gm_dist, float gm_grad, const float* __restrict__ c_obs, const float* __restrict__ c_pred,
    const float* __restrict__ c_grad, int cc, int color_mode, float w_photo, double* __restrict__ sums, float lm_lambda,
    double* __restrict__ result, double* __restrict__ t_inout) {
  // 21 upper-triangular entries of N, 6 of g, 5 scalars
  constexpr int NA = 32;
  float acc[NA];
#pragma unroll
  for (int i = 0; i < NA; ++i) acc[i] = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gx = grad[3 * i], gy = grad[3 * i + 1], gz = grad[3 * i + 2];
    const float gn = sqrtf(gx * gx + gy * gy + gz * gz);
    const bool valid = (nn_count[i] >= min_nn) && (gn < max_gn) && (gn > min_gn) &&
                       (sdf_std ? sdf_std[i] < max_std : true);  // tracker.py:419-425
    if (!valid) continue;
    const float px = xyz[3 * i], py = xyz[3 * i + 1], pz = xyz[3 * i + 2];
    const float r = sdf[i] - (sdf_label ? sdf_label[i] : 0.f);  // tracker.py:459
    float w = 1.f;
    if (gm_grad > 0.f) {  // tracker.py:471-475
      const float a = gn - 1.f;
      const float t = gm_grad / (gm_grad + a * a);
      w *= t * t;
    }
    if (gm_dist > 0.f) {  // tracker.py:476-480
      const float t = gm_dist / (gm_dist + r * r);
      w *= t * t;
    }
    if (normals) {  // tracker.py:482-488
      const float inv = 1.f / gn;
      w *= 0.5f + fabsf(normals[3 * i] * gx * inv + normals[3 * i + 1] * gy * inv + normals[3 * i + 2] * gz * inv);
    }
    // colour: intensity of the measured / predicted colour and of the colour gradient (tools.py:408)
    float rc = 0.f, cgx = 0.f, cgy = 0.f, cgz = 0.f;
    if (color_mode) {
      float io, ip;
      if (cc == 3) {
        const float k0 = 0.299f, k1 = 0.587f, k2 = 0.114f;
        io = k0 * c_obs[3 * i] + k1 * c_obs[3 * i + 1] + k2 * c_obs[3 * i + 2];
        ip = k0 * c_pred[3 * i] + k1 * c_pred[3 * i + 1] + k2 * c_pred[3 * i + 2];
        if (c_grad) {
          const float* g3 = c_grad + 9 * i;
          cgx = k0 * g3[0] + k1 * g3[3] + k2 * g3[6];
          cgy = k0 * g3[1] + k1 * g3[4] + k2 * g3[7];
          cgz = k0 * g3[2] + k1 * g3[5] + k2 * g3[8];
        }
      } else {
        io = c_obs[i * cc];
        ip = c_pred[i * cc];
        if (c_grad) {
          cgx = c_grad[(i * cc) * 3];
          cgy = c_grad[(i * cc) * 3 + 1];
          cgz = c_grad[(i * cc) * 3 + 2];
        }
      }
      rc = ip - io;
      if (color_mode == 1) w *= expf(-fabsf(io - ip));  // consistency weight (tracker.py:509-514)
    }
    // J = [p x g, g]  (tracker.py:652-655)
    float J[6];
    J[0] = py * gz - pz * gy;
    J[1] = pz * gx - px * gz;
    J[2] = px * gy - py * gx;
    J[3] = gx;
    J[4] = gy;
    J[5] = gz;
    int e = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      const float wa = w * J[a];
#pragma unroll
      for (int b = a; b < 6; ++b) {
        acc[e] = fmaf(wa, J[b], acc[e]);
        ++e;
      }
      acc[21 + a] = fmaf(-wa, r, acc[21 + a]);
    }
    if (color_mode == 2) {  // photometric term (tracker.py:720-730)
      float Jc[6];
      Jc[0] = py * cgz - pz * cgy;
      Jc[1] = pz * cgx - px * cgz;
      Jc[2] = px * cgy - py * cgx;
      Jc[3] = cgx;
      Jc[4] = cgy;
      Jc[5] = cgz;
      int e2 = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        const float wa = w_photo * w * Jc[a];
#pragma unroll
        for (int b = a; b < 6; ++b) {
          acc[e2] = fmaf(wa, Jc[b], acc[e2]);
          ++e2;
        }
        acc[21 + a] = fmaf(-wa, rc, acc[21 + a]);
      }
    }
    acc[27] += w;
    acc[28] += fabsf(r);
    acc[29] += 1.f;
    acc[30] = fmaf(w * r, r, acc[30]);
    acc[31] += fabsf(rc);
  }
  __shared__ float s_red[8][NA];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NA; ++i) {
    const float v = warp_sum(acc[i]);
    if (lane == 0) s_red[warp][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < NA) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += (double)s_red[w][threadIdx.x];
    // scatter the packed triangle back to the full symmetric layout
    const int i = threadIdx.x;
    if (i < 21) {
      int a = 0, rem = i;
      while (rem >= 6 - a) {
        rem -= 6 - a;
        ++a;
      }
      const int b = a + rem;
      atomicAdd(sums + a * 6 + b, t);
      if (a != b) atomicAdd(sums + b * 6 + a, t);
    } else {
      atomicAdd(sums + 36 + (i - 21), t);
    }
  }
  gn_finish(sums, lm_lambda, result, t_inout);
}

__device__ void expmap_d(const double* w, double* R) {  // tracker.py:784-795
  const double angle = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double ax = 0, ay = 0, az = 0;
  if (angle > 0) {
    ax = w[0] / angle;
    ay = w[1] / angle;
    az = w[2] / angle;
  }
  const double s = sin(angle), c1 = 1.0 - cos(angle);
  const double S[9] = {0, -az, ay, az, 0, -ax, -ay, ax, 0};
  double S2[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double t = 0;
      for (int k = 0; k < 3; ++k) t += S[i * 3 + k] * S[k * 3 + j];
      S2[i * 3 + j] = t;
    }
  for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0 ? 1.0 : 0.0) + S[i] * s + S2[i] * c1;
}

// eigenvalues of a symmetric 3x3 (closed form), ascending not required
__device__ void sym3_eig(const double* A, double* ev) {
  const double p1 = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
  const double q = (A[0] + A[4] + A[8]) / 3.0;
  if (p1 == 0.0) {
    ev[0] = A[0];
    ev[1] = A[4];
    ev[2] = A[8];
    return;
  }
  const double p2 = (A[0] - q) * (A[0] - q) + (A[4] - q) * (A[4] - q) + (A[8] - q) * (A[8] - q) + 2.0 * p1;
  const double p = sqrt(p2 / 6.0);
  double B[9];
  for (int i = 0; i < 9; ++i) B[i] = (A[i] - (i % 4 == 0 ? q : 0.0)) / p;
  const double detB = B[0] * (B[4] * B[8] - B[5] * B[7]) - B[1] * (B[3] * B[8] - B[5] * B[6]) +
                      B[2] * (B[3] * B[7] - B[4] * B[6]);
  double r = detB / 2.0;
  r = r < -1.0 ? -1.0 : (r > 1.0 ? 1.0 : r);
  const double phi = acos(r) / 3.0;
  ev[0] = q + 2.0 * p * cos(phi);
  ev[2] = q + 2.0 * p * cos(phi + 2.0943951023931953);
  ev[1] = 3.0 * q - ev[0] - ev[2];
}

__device__ void gn_solve(const double* sums, float lm_lambda, double* __restrict__ result, double* __restrict__ t_inout) {
  const double cnt = sums[44];
  double dT[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  for (int i = 0; i < 32; ++i) result[i] = 0.0;
  result[16] = cnt;
  if (cnt >= 10.0) {  // tracker.py:430-432
    // w /= 2*mean(w) (tracker.py:524) scales N and g by cnt / (2 sum_w)
    const double sc = cnt / (2.0 * sums[42]);
    double N[36], g[6], A[36];
    // the reference holds N, g in fp32 before the fp64 solve (tracker.py:656-675)
    for (int i = 0; i < 36; ++i) N[i] = (double)(float)(sums[i] * sc);
    for (int i = 0; i < 6; ++i) g[i] = (double)(float)(sums[36 + i] * sc);
    for (int i = 0; i < 36; ++i) A[i] = N[i];
    for (int i = 0; i < 6; ++i) A[i * 7] = (double)(float)(N[i * 7] + (double)lm_lambda * N[i * 7]);
    // Gaussian elimination with partial pivoting: A t = g
    double t[6];
    for (int i = 0; i < 6; ++i) t[i] = g[i];
    bool singular = false;
    for (int c = 0; c < 6; ++c) {
      int piv = c;
      for (int r = c + 1; r < 6; ++r)
        if (fabs(A[r * 6 + c]) > fabs(A[piv * 6 + c])) piv = r;
      if (A[piv * 6 + c] == 0.0) {
        singular = true;
        break;
      }
      if (piv != c) {
        for (int k = 0; k < 6; ++k) {
          const double tmp = A[c * 6 + k];
          A[c * 6 + k] = A[piv * 6 + k];
          A[piv * 6 + k] = tmp;
        }
        const double tmp = t[c];
        t[c] = t[piv];
        t[piv] = tmp;
      }
      for (int r = c + 1; r < 6; ++r) {
        const double f = A[r * 6 + c] / A[c * 6 + c];
        for (int k = c; k < 6; ++k) A[r * 6 + k] -= f * A[c * 6 + k];
        t[r] -= f * t[c];
      }
    }
    if (!singular) {
      for (int c = 5; c >= 0; --c) {
        double s = t[c];
        for (int k = c + 1; k < 6; ++k) s -= A[c * 6 + k] * t[k];
        t[c] = s / A[c * 6 + c];
      }
      double R[9];
      expmap_d(t, R);
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) dT[i * 4 + j] = R[i * 3 + j];
        dT[i * 4 + 3] = t[3 + i];
      }
    }
    result[17] = sums[43] / cnt * 100.0;  // mean |r| in cm (tracker.py:461)
    double tr[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) tr[i * 3 + j] = N[(3 + i) * 6 + 3 + j];
    sym3_eig(tr, result + 18);            // eigenvalues of N_raw[3:,3:] (tracker.py:685-686)
    result[21] = sums[45] * sc / cnt;     // mean(w r^2) (tracker.py:692)
    for (int i = 0; i < 6; ++i) result[22 + i] = g[i];
    result[28] = sums[46] / cnt;          // mean |colour residual| (tracker.py:531)
  }
  for (int i = 0; i < 16; ++i) result[i] = dT[i];
  if (t_inout) {  // T <- dT @ T (tracker.py:147)
    double T[16], O[16];
    for (int i = 0; i < 16; ++i) T[i] = t_inout[i];
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) {
        double s = 0;
        for (int k = 0; k < 4; ++k) s += dT[i * 4 + k] * T[k * 4 + j];
        O[i * 4 + j] = s;
      }
    for (int i = 0; i < 16; ++i) t_inout[i] = O[i];
  }
}

__global__ void gn_solve_kernel(const double* __restrict__ sums, float lm_lambda, double* __restrict__ result,
                                double* __restrict__ t_inout) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  gn_solve(sums, lm_lambda, result, t_inout);
}

// the block that finishes last solves the normal equations (all other blocks' fp64 atomics are visible: every block
// fences before it takes its ticket)
__device__ __forceinline__ void gn_finish(double* sums, float lm_lambda, double* result, double* t_inout) {
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int* ticket = reinterpret_cast<unsigned int*>(sums + GN_TICKET);
    s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    double loc[GN_NSUM + 2];
    for (int i = 0; i < GN_NSUM + 2; ++i) loc[i] = __ldcg(sums + i);  // written by L2 atomics: bypass L1
    gn_solve(loc, lm_lambda, result, t_inout);
  }
}

}  // namespace pinb

using namespace pinb;

extern "C" int pinb200_gn_step(const float* xyz, const float* sdf, const float* grad, const float* sdf_std,
                               const int32_t* nn_count, const float* sdf_label, const float* normals, int64_t n,
                               int32_t min_nn, float min_grad_norm, float max_grad_norm, float max_sdf_std,
                               float gm_dist, float gm_grad, float lm_lambda, const float* color_obs,
                               const float* color_pred, const float* color_grad, int32_t color_channels,
                               int32_t color_mode, float w_photo, double* sums, double* result, double* t_inout,
                               void* stream) {
  // n == 0 (empty tensors have null data pointers) takes gn_solve_kernel: identity step, T unchanged
  if ((n > 0 && (!xyz || !sdf || !grad || !nn_count)) || !sums || !result || n < 0) {
    set_error("gn_step: null argument");
    return PINB200_ERR_BAD_ARG;
  }
  if (color_mode < 0 || color_mode > 2 ||
      (color_mode && (!color_obs || !color_pred || color_channels < 1 || (color_mode == 2 && !color_grad)))) {
    set_error("gn_step: colour mode %d needs color_obs/color_pred (and color_grad for the photometric term)",
              color_mode);
    return PINB200_ERR_BAD_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sums, 0, 64 * sizeof(double), st);
  if (e != cudaSuccess) {
    set_error("cudaMemsetAsync: %s", cudaGetErrorString(e));
    return PINB200_ERR_CUDA;
  }
  if (n > 0) {
    const int grid = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 2);
    gn_accumulate_kernel<<<grid, 256, 0, st>>>(xyz, sdf, grad, sdf_std, nn_count, sdf_label, normals, n, min_nn,
                                               min_grad_norm, max_grad_norm, max_sdf_std, gm_dist, gm_grad, color_obs, color_pred,
                                               color_grad, color_channels, color_mode, w_photo, sums, lm_lambda, result,
                                               t_inout);
    return check_launch("gn_accumulate_kernel");
  }
  gn_solve_kernel<<<1, 32, 0, st>>>(sums, lm_lambda, result, t_inout);
  return check_launch("gn_solve_kernel");
}


extern "C" int pinb200_track_iterations(const pinb200_map_view* map, const pinb200_decoder_view* sdf_dec,
                                        const pinb200_decoder_view* color_dec, const float* source_xyz, int64_t n,
                                        const pinb200_query_opts* opts, const pinb200_query_out* out,
                                        const pinb200_gn_opts* gn, int32_t n_iter, void* stream) {
  if (!opts || !out || !gn || !gn->sums || !gn->result) {
    set_error("track_iterations: null argument");
    return PINB200_ERR_BAD_ARG;
  }
  if (!opts->transform || !out->xyz || !out->sdf || !out->grad || !out->sdf_std || !out->nn_count) {
    set_error("track_iterations: needs opts->transform and the xyz/sdf/grad/sdf_std/nn_count outputs");
    return PINB200_ERR_BAD_ARG;
  }
  for (int it = 0; it < n_iter; ++it) {
    int rc = pinb200_query_sdf(map, sdf_dec, color_dec, source_xyz, nullptr, n, opts, out, stream);
    if (rc) return rc;
    rc = pinb200_gn_step(out->xyz, out->sdf, out->grad, out->sdf_std, out->nn_count, gn->sdf_label, gn->normals, n,
                         gn->min_nn, gn->min_grad_norm, gn->max_grad_norm, gn->max_sdf_std, gn->gm_dist, gn->gm_grad,
                         gn->lm_lambda, gn->color_mode ? gn->color_obs : nullptr, gn->color_mode ? out->color : nullptr,
                         gn->color_mode == 2 ? out->color_grad : nullptr, gn->color_channels, gn->color_mode,
                         gn->w_photo, gn->sums, gn->result, const_cast<double*>(opts->transform), stream);
    if (rc) return rc;
  }
  return PINB200_OK;
}
