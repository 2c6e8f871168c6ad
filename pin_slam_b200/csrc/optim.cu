// K3 (Adam) and the loss heads of one map-training iteration.
#include <algorithm>
#include <math.h>

#include "common.cuh"

namespace pinb {

// torch.optim.Adam single-tensor arithmetic (torch/optim/adam.py, _single_tensor_adam),
// as configured by the reference's setup_optimizer (utils/tools.py:153-203):
//   grad += wd * param ; m.lerp_(grad, 1-b1) ; v = v*b2 + (1-b2)*g*g ;
//   denom = sqrt(v)/sqrt(bc2) + eps ; param += -(lr/bc1) * m/denom
__global__ void adam_kernel(float* __restrict__ param, float* __restrict__ grad, float* __restrict__ m,
                            float* __restrict__ v, long long n, float one_minus_b1, float b2, float one_minus_b2,
                            float bc2_sqrt, float eps, float neg_step_size, float wd) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float g = grad[i];
    grad[i] = 0.f;  // opt.zero_grad() for the next iteration
    float p = param[i];
    if (wd != 0.f) g = fmaf(wd, p, g);
    float mi = m[i], vi = v[i];
    mi = mi + one_minus_b1 * (g - mi);
    vi = vi * b2 + one_minus_b2 * g * g;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p = p + neg_step_size * (mi / denom);
    m[i] = mi;
    v[i] = vi;
    param[i] = p;
  }
}

// BCE-with-logits on the main rows + Eikonal on the numerical-gradient rows.
// utils/mapper.py:728-780, utils/loss.py:45-63, utils/mapper.py:1002-1014.
__global__ void mapping_loss_kernel(const float* __restrict__ sdf, const float* __restrict__ label,
                                    const float* __restrict__ weight, long long n_main, long long n_eik, float sigma,
                                    int weighted, float weight_e, float eik_eps, float gscale, float* __restrict__ dl,
                                    float* __restrict__ losses) {
  float bce = 0.f, eik = 0.f;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const float inv_n = 1.f / (float)n_main;
  for (long long i = t0; i < n_main; i += stride) {
    const float z = sdf[i] / sigma;
    const float t = 1.f / (1.f + expf(-label[i] / sigma));
    const float w = weighted ? fabsf(weight[i]) : 1.f;  // |weight| (mapper.py:729)
    // (1-t)*z + log1p(exp(-|z|)) + max(-z,0)
    bce += w * ((1.f - t) * z + log1pf(expf(-fabsf(z))) + fmaxf(-z, 0.f));
    const float sg = 1.f / (1.f + expf(-z));
    dl[i] = gscale * w * (sg - t) * inv_n / sigma;
  }
  if (n_eik > 0) {
    const float* s = sdf + n_main;
    float* d = dl + n_main;
    const float inv2e = 1.f / (2.f * eik_eps);
    for (long long j = t0; j < n_eik; j += stride) {
      const float gx = (s[j] - s[n_eik + j]) * inv2e;
      const float gy = (s[2 * n_eik + j] - s[3 * n_eik + j]) * inv2e;
      const float gz = (s[4 * n_eik + j] - s[5 * n_eik + j]) * inv2e;
      const float nrm = sqrtf(gx * gx + gy * gy + gz * gz);
      const float e = nrm - 1.f;
      eik += e * e;
      const float c = nrm > 0.f ? gscale * weight_e * 2.f * e / ((float)n_eik * nrm) * inv2e : 0.f;
      d[j] = c * gx;
      d[n_eik + j] = -c * gx;
      d[2 * n_eik + j] = c * gy;
      d[3 * n_eik + j] = -c * gy;
      d[4 * n_eik + j] = c * gz;
      d[5 * n_eik + j] = -c * gz;
    }
  }
  if (losses) {
    bce = warp_sum(bce);
    eik = warp_sum(eik);
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(losses + 0, bce * inv_n);
      if (n_eik > 0) atomicAdd(losses + 1, eik / (float)n_eik);
    }
  }
}

// L1 colour loss on surface samples (utils/mapper.py:804-812, utils/loss.py:31-41)
__global__ void color_loss_kernel(const float* __restrict__ pred, const float* __restrict__ lab,
                                  const float* __restrict__ sdf_label, const float* __restrict__ weight, long long n,
                                  int cc, float surf, int weighted, float weight_i, float gscale,
                                  const float* __restrict__ n_surface, float* __restrict__ dl,
                                  float* __restrict__ loss) {
  const float cnt = fmaxf(*n_surface, 1.f) * (float)cc;
  float acc = 0.f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n * cc; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / cc;
    float g = 0.f;
    if (fabsf(sdf_label[i]) < surf) {
      const float w = weighted ? fabsf(weight[i]) : 1.f;
      const float d = pred[e] - lab[e];
      acc += w * fabsf(d);
      g = gscale * weight_i * w * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) / cnt;
    }
    dl[e] = g;
  }
  if (loss) {
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) atomicAdd(loss, acc / cnt);
  }
}

// one thread per sample: pool gathers + the six shifted numerical-gradient rows of every decimation-th sample
__global__ void assemble_batch_kernel(const float* __restrict__ cp, const float* __restrict__ lp,
                                      const int32_t* __restrict__ tp, const float* __restrict__ wp,
                                      const float* __restrict__ colp, int cc, const long long* __restrict__ index,
                                      long long n, int dec, float eps, float* __restrict__ rows,
                                      float* __restrict__ label, int32_t* __restrict__ ts, float* __restrict__ weight,
                                      float* __restrict__ color) {
  const long long ne = (n + dec - 1) / dec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long s = index[i];
    const float x = cp[3 * s], y = cp[3 * s + 1], z = cp[3 * s + 2];
    rows[3 * i] = x;
    rows[3 * i + 1] = y;
    rows[3 * i + 2] = z;
    label[i] = lp[s];
    ts[i] = tp[s];
    weight[i] = wp[s];
    if (colp)
      for (int c = 0; c < cc; ++c) color[i * cc + c] = colp[s * cc + c];
    if (dec > 0 && i % dec == 0) {
      const long long j = i / dec;
      float* r = rows + 3 * n;
      const float sh[6][3] = {{eps, 0, 0}, {-eps, 0, 0}, {0, eps, 0}, {0, -eps, 0}, {0, 0, eps}, {0, 0, -eps}};
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        float* o = r + 3 * (a * ne + j);
        o[0] = x + sh[a][0];
        o[1] = y + sh[a][1];
        o[2] = z + sh[a][2];
      }
    }
  }
}

}  // namespace pinb

using namespace pinb;

extern "C" int pinb200_assemble_batch(const float* coord_pool, const float* label_pool, const int32_t* ts_pool,
                                      const float* weight_pool, const float* color_pool, int32_t color_channels,
                                      const int64_t* index, int64_t n, int32_t decimation, float eps, float* rows,
                                      float* label, int32_t* ts, float* weight, float* color, void* stream) {
  if (!coord_pool || !label_pool || !ts_pool || !weight_pool || !index || !rows || !label || !ts || !weight ||
      (color_pool && !color)) {
    set_error("assemble_batch: null argument");
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 8);
  assemble_batch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(coord_pool, label_pool, ts_pool, weight_pool,
                                                                color_pool, color_channels,
                                                                reinterpret_cast<const long long*>(index), n, decimation,
                                                                eps, rows, label, ts, weight, color);
  return check_launch("assemble_batch_kernel");
}

extern "C" int pinb200_color_loss(const float* color_pred, const float* color_label, const float* sdf_label,
                                  const float* weight, int64_t n, int32_t color_channels, float surface_range,
                                  int32_t loss_weight_on, float weight_i, float grad_scale, const float* n_surface,
                                  float* dloss_dcolor, float* loss, void* stream) {
  if (!color_pred || !color_label || !sdf_label || !n_surface || !dloss_dcolor || color_channels < 1 ||
      (loss_weight_on && !weight)) {
    set_error("color_loss: null argument");
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  const long long work = n * color_channels;
  const int grid = (int)std::min<long long>((work + 255) / 256, (long long)sm_count() * 4);
  color_loss_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(color_pred, color_label, sdf_label, weight, n,
                                                            color_channels, surface_range, loss_weight_on, weight_i,
                                                            grad_scale, n_surface, dloss_dcolor, loss);
  return check_launch("color_loss_kernel");
}

extern "C" int pinb200_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double lr,
                                 double beta1, double beta2, double eps, double weight_decay, int32_t step,
                                 void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || step < 1) {
    set_error("adam_step: null argument or step < 1");
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  const double step_size = lr / bc1;
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 8);
  adam_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, n, (float)(1.0 - beta1),
                                                      (float)beta2, (float)(1.0 - beta2), (float)sqrt(bc2), (float)eps,
                                                      (float)(-step_size), (float)weight_decay);
  return check_launch("adam_kernel");
}

extern "C" int pinb200_mapping_loss(const float* sdf, const float* sdf_label, const float* weight, int64_t n_main,
                                    int64_t n_eik, float sigma, int32_t loss_weight_on, float weight_e, float eik_eps,
                                    float grad_scale, float* dloss_dsdf, float* losses, void* stream) {
  if (!sdf || !sdf_label || !dloss_dsdf || n_main <= 0 || (loss_weight_on && !weight)) {
    set_error("mapping_loss: null argument / empty batch");
    return PINB200_ERR_BAD_ARG;
  }
  if (losses) {
    const cudaError_t e = cudaMemsetAsync(losses, 0, 2 * sizeof(float), (cudaStream_t)stream);
    if (e != cudaSuccess) {
      set_error("cudaMemsetAsync: %s", cudaGetErrorString(e));
      return PINB200_ERR_CUDA;
    }
  }
  const long long work = std::max<long long>(n_main, n_eik);
  const int grid = (int)std::min<long long>((work + 255) / 256, (long long)sm_count() * 4);
  mapping_loss_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(sdf, sdf_label, weight, n_main, n_eik, sigma,
                                                              loss_weight_on, weight_e, eik_eps, grad_scale, dloss_dsdf, losses);
  return check_launch("mapping_loss_kernel");
}


extern "C" int pinb200_map_iterations(const pinb200_map_view* map, const pinb200_decoder_view* dec, int32_t nn_k,
                                      int32_t weighted_first, const pinb200_map_train_opts* t,
                                      const pinb200_query_out* out, int32_t n_iter, void* stream) {
  if (!map || !dec || !t || !out || !t->index || !t->rows || !t->label || !t->ts || !t->weight || !t->dloss ||
      !t->losses || !t->feat || !t->dec_flat || !t->grad_feat || !t->grad_dec || !t->m_feat || !t->v_feat ||
      !t->m_dec || !t->v_dec || !out->sdf || !out->knn_idx || !out->knn_weight) {
    set_error("map_iterations: null argument");
    return PINB200_ERR_BAD_ARG;
  }
  const int64_t n = t->bs;
  const int64_t ne = t->decimation > 0 ? (n + t->decimation - 1) / t->decimation : 0;
  const int64_t rows = n + 6 * ne;
  const int64_t n_feat = ((int64_t)map->n_nb + 1) * map->feature_dim;
  const int64_t n_dec = pinb200_decoder_param_count(dec);
  pinb200_query_opts qo{};
  qo.nn_k = nn_k;
  qo.weighted_first = weighted_first;
  qo.training_mode = 1;
  qo.need_grad = 0;
  qo.training_rows = n;
  qo.transform = nullptr;
  qo.workspace = t->workspace;
  qo.workspace_bytes = t->workspace_bytes;
  const bool do_fb = (t->stages & 1) != 0, do_opt = (t->stages & 2) != 0;
  for (int it = 0; it < n_iter; ++it) {
    int rc = PINB200_OK;
    if (do_fb) {
      rc = pinb200_assemble_batch(t->coord_pool, t->label_pool, t->ts_pool, t->weight_pool, nullptr, 0,
                                  t->index + (int64_t)it * n, n, t->decimation, t->eik_eps, t->rows, t->label, t->ts,
                                  t->weight, nullptr, stream);
      if (rc) return rc;
      rc = pinb200_query_sdf(map, dec, nullptr, t->rows, t->ts, rows, &qo, out, stream);
      if (rc) return rc;
      rc = pinb200_mapping_loss(out->sdf, t->label, t->weight, n, ne, t->sigma, t->loss_weight_on,
                                ne > 0 ? t->weight_e : 0.f, t->eik_eps, t->grad_scale, t->dloss, t->losses, stream);
      if (rc) return rc;
      rc = pinb200_train_backward(map, dec, t->feat, t->rows, out->knn_idx, out->knn_weight, t->dloss, rows, nn_k,
                                  weighted_first, t->grad_feat, t->grad_dec, stream);
      if (rc) return rc;
    }
    if (do_fb && do_opt && t->nccl_comm) {  // data-parallel: sum the gradient blocks over the ranks, on this stream
      if (!t->reduce_buf || t->reduce_count <= 0) {
        set_error("map_iterations: nccl_comm needs reduce_buf / reduce_count");
        return PINB200_ERR_BAD_ARG;
      }
      rc = nccl_allreduce_sum(t->nccl_comm, t->reduce_buf, t->reduce_count, (cudaStream_t)stream);
      if (rc) return rc;
    }
    if (!do_opt) continue;
    const int step = t->first_step + it;
    if (t->train_decoder) {
      rc = pinb200_adam_step(t->dec_flat, t->grad_dec, t->m_dec, t->v_dec, n_dec, t->lr, t->beta1, t->beta2, t->eps, 0.0,
                             step, stream);
      if (rc) return rc;
    } else {
      cudaError_t e = cudaMemsetAsync(t->grad_dec, 0, (size_t)n_dec * sizeof(float), (cudaStream_t)stream);
      if (e != cudaSuccess) {
        set_error("cudaMemsetAsync: %s", cudaGetErrorString(e));
        return PINB200_ERR_CUDA;
      }
    }
    rc = pinb200_adam_step(t->feat, t->grad_feat, t->m_feat, t->v_feat, n_feat, t->lr, t->beta1, t->beta2, t->eps,
                           t->weight_decay, step, stream);
    if (rc) return rc;
  }
  return PINB200_OK;
}
