// K2: backward pass of one map-training batch through the decoder and the IDW
// feature interpolation, from the kNN ids/weights the forward saved.
//
// Per 128-row tile (same row <-> thread mapping as K1):
//   A  thread per row : re-gather the decoder input rows from the saved kNN (float4 feature-row loads)
//   B  thread per row : forward, keeping every layer's activations in shared memory
//   C  tile reductions: dW_out, then for each layer l = L-1..0
//        dW_l  += G_l^T A_{l-1}   (128-row tile GEMM, thread-owned 4 x NI output blocks)
//        G_{l-1} = mask * (W_l^T G_l)  (thread per row)
//   D  thread per row : scatter d loss / d feature rows with 16-byte vector reductions
// Decoder gradients are accumulated per CTA in shared memory over all its tiles
// and flushed once with atomics.
//
// Replaces the autograd reverse pass of utils/mapper.py:816-817 through
// model/neural_points.py:597-731 (index_put_ accumulate) and model/decoder.py:61-85.
#include <algorithm>

#include "mlp.cuh"

#ifndef PINB_K2_MIN_CTAS
#define PINB_K2_MIN_CTAS 3  // resident CTAs per SM the register allocation targets (12 warps)
#endif

namespace pinb {

struct TrainLayout {
  DecSmem dec;
  int x, h, dW, go, idx, w, q, mask, total;
};

struct TrainParams {
  pinb200_map_view map;
  pinb200_decoder_view dec;
  const float* feat;
  const float* query_xyz;
  const int32_t* knn_idx;
  const float* knn_w;
  const float* dl;  // [N, out_dim] d loss / d decoder output (after out_scale / sigmoid)
  long long n;
  int K, wf, n_tiles, qpt;
  // the per-CTA shared-memory gradient accumulator: n_acc floats laid out [w0 | b0 | w1 | b1 | ... | w_out | b_out],
  // with a slot for every bias whether the decoder has it or not (the bias sums are computed either way); acc_*:
  // offset of each block
  int n_acc;
  int acc_w[PINB200_MAX_HIDDEN_LAYERS];
  int acc_b[PINB200_MAX_HIDDEN_LAYERS];
  int acc_wout, acc_bout;
  float* grad_feat;
  // where each parameter block's gradient goes in the caller's flat gradient vector, whose layout has no slot for an
  // absent bias (pinb200_decoder_param_count); NULL: the bias is absent and its partial sums are dropped
  float* gd_w[PINB200_MAX_HIDDEN_LAYERS];
  float* gd_b[PINB200_MAX_HIDDEN_LAYERS];
  float* gd_wout;
  float* gd_bout;
  TrainLayout lay;
};

// adds this CTA's partial sums of one parameter block (shared memory) to its block of the flat gradient vector
__device__ __forceinline__ void flush_block(const float* src, int count, float* dst, int tid) {
  if (!dst) return;
  for (int e = tid; e < count; e += TILE) {
    const float v = src[e];
    if (v != 0.f) atomicAdd(dst + e, v);
  }
}

// dW[j][i] += sum_r G[j][r] * A[i][r]; db[j] += sum_r G[j][r]   (thread-owned 4 x NI blocks)
template <int NI>
__device__ __forceinline__ void tile_gemm_acc(const float* __restrict__ G, const float* __restrict__ A, int n_in,
                                              float* __restrict__ dW, float* __restrict__ db, int tid) {
  const int j0 = (tid >> 3) * 4, ib = tid & 7;
  float acc[4][NI];
  float bacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int s = 0; s < NI; ++s) acc[a][s] = 0.f;
#pragma unroll 2
  for (int r = 0; r < TILE; ++r) {
    float g[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) g[a] = G[(j0 + a) * ACT_LD + r];
#pragma unroll
    for (int s = 0; s < NI; ++s) {
      const int i = ib + 8 * s;
      const float av = i < n_in ? A[i * ACT_LD + r] : 0.f;
#pragma unroll
      for (int a = 0; a < 4; ++a) acc[a][s] = fmaf(g[a], av, acc[a][s]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) bacc[a] += g[a];
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
#pragma unroll
    for (int s = 0; s < NI; ++s) {
      const int i = ib + 8 * s;
      if (i < n_in) dW[(j0 + a) * n_in + i] += acc[a][s];
    }
    if (ib == 0) db[j0 + a] += bacc[a];
  }
}

template <int H, int DP>
__global__ void __launch_bounds__(TILE, PINB_K2_MIN_CTAS) train_bwd_kernel(const __grid_constant__ TrainParams p) {
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const pinb200_map_view& m = p.map;
  const int K = p.K, F = m.feature_dim, D = F + 3, L = p.dec.n_hidden, OC = p.dec.out_dim;
  const bool wf = p.wf != 0, leaky = p.dec.leaky_relu != 0;
  const float* __restrict__ feat = p.feat;
  constexpr int NI0 = (DP + 7) / 8;

  float* s_x = smem + p.lay.x;
  float* s_h = smem + p.lay.h;  // L tiles of [H][ACT_LD]
  float* s_dW = smem + p.lay.dW;
  float* s_go = smem + p.lay.go;  // [TILE][4]
  int* s_idx = reinterpret_cast<int*>(smem + p.lay.idx);
  float* s_w = smem + p.lay.w;
  float* s_q = smem + p.lay.q;
  uint64_t* s_mask = reinterpret_cast<uint64_t*>(smem + p.lay.mask);

  stage_decoder(p.dec, p.lay.dec, smem, DP, true);
  for (int e = tid; e < p.n_acc; e += TILE) s_dW[e] = 0.f;
  __syncthreads();

  // accumulator block offsets (TrainParams::acc_*), copied once: read from the kernel parameters at their uses in
  // the layer loops they cost this kernel more spills (ptxas -v)
  int off_w[PINB200_MAX_HIDDEN_LAYERS], off_b[PINB200_MAX_HIDDEN_LAYERS];
#pragma unroll
  for (int l = 0; l < PINB200_MAX_HIDDEN_LAYERS; ++l) {
    off_w[l] = p.acc_w[l];
    off_b[l] = p.acc_b[l];
  }
  const int off_wout = p.acc_wout, off_bout = p.acc_bout;

  const int QPT = p.qpt;
  // feature rows are 16-byte aligned multiples of 4 floats: vector loads and vector reductions
  const bool vec_ok = (F % 4 == 0) && ((reinterpret_cast<uintptr_t>(feat) & 15) == 0) &&
                      ((reinterpret_cast<uintptr_t>(p.grad_feat) & 15) == 0);
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const long long q0 = (long long)tile * QPT;
    // ---------------- A: rebuild decoder inputs (thread per tile row) ----------------
    // every thread issues its own idx / weight / point / feature-row loads (a feature row is >= 16 contiguous
    // bytes, read as float4): one dependent round trip per tile instead of one per query
#pragma unroll
    for (int c = 0; c < 4; ++c) s_go[tid * 4 + c] = 0.f;
    if (!wf) {
      const int ql = tid / K, k = tid - ql * K;
      const long long qi = q0 + ql;
      int lk = -1;
      float w = 0.f, nx = 0.f, ny = 0.f, nz = 0.f;
      const bool live = ql < QPT && qi < p.n;
      if (live) {
        lk = __ldg(p.knn_idx + qi * K + k);
        w = __ldg(p.knn_w + qi * K + k);
      }
      if (ql < QPT) {
        s_idx[tid] = lk;
        s_w[tid] = w;
      }
      if (lk >= 0) {
        const float* pp = m.nb_points + 3 * (size_t)lk;
        nx = __fsub_rn(__ldg(p.query_xyz + 3 * qi), __ldg(pp));
        ny = __fsub_rn(__ldg(p.query_xyz + 3 * qi + 1), __ldg(pp + 1));
        nz = __fsub_rn(__ldg(p.query_xyz + 3 * qi + 2), __ldg(pp + 2));
        if (m.after_pgo) {
          const float* qq = m.nb_orient + 4 * (size_t)lk;
          quat_rotate_passive(__ldg(qq), __ldg(qq + 1), __ldg(qq + 2), __ldg(qq + 3), nx, ny, nz, nx, ny, nz);
        }
        const float* fr = feat + (size_t)lk * F;
        if (vec_ok) {
          for (int j = 0; j < F; j += 4) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(fr + j));
            s_x[(j + 0) * ACT_LD + tid] = v.x;
            s_x[(j + 1) * ACT_LD + tid] = v.y;
            s_x[(j + 2) * ACT_LD + tid] = v.z;
            s_x[(j + 3) * ACT_LD + tid] = v.w;
          }
        } else {
          for (int j = 0; j < F; ++j) s_x[j * ACT_LD + tid] = __ldg(fr + j);
        }
        for (int c = 0; c < OC; ++c) s_go[tid * 4 + c] = __ldg(p.dl + qi * OC + c) * w;
      } else {
        for (int j = 0; j < F; ++j) s_x[j * ACT_LD + tid] = 0.f;
      }
      s_x[(F + 0) * ACT_LD + tid] = nx;
      s_x[(F + 1) * ACT_LD + tid] = ny;
      s_x[(F + 2) * ACT_LD + tid] = nz;
    } else {
      const long long qi = q0 + tid;
      const bool live = qi < p.n;
      int lks[PINB200_MAX_K];
      float ws[PINB200_MAX_K];
      float sx = 0.f, sy = 0.f, sz = 0.f;
#pragma unroll
      for (int k = 0; k < PINB200_MAX_K; ++k) {
        lks[k] = (live && k < K) ? __ldg(p.knn_idx + qi * K + k) : -1;
        ws[k] = (live && k < K) ? __ldg(p.knn_w + qi * K + k) : 0.f;
        if (k < K) {
          s_idx[tid * K + k] = lks[k];
          s_w[tid * K + k] = ws[k];
        }
      }
      float qx = 0.f, qy = 0.f, qz = 0.f;
      if (live) {
        qx = __ldg(p.query_xyz + 3 * qi);
        qy = __ldg(p.query_xyz + 3 * qi + 1);
        qz = __ldg(p.query_xyz + 3 * qi + 2);
        for (int c = 0; c < OC; ++c) s_go[tid * 4 + c] = __ldg(p.dl + qi * OC + c);
      }
#pragma unroll
      for (int k = 0; k < PINB200_MAX_K; ++k) {
        if (lks[k] < 0) continue;
        const float* pp = m.nb_points + 3 * (size_t)lks[k];
        float nx = __fsub_rn(qx, __ldg(pp)), ny = __fsub_rn(qy, __ldg(pp + 1)), nz = __fsub_rn(qz, __ldg(pp + 2));
        if (m.after_pgo) {
          const float* qq = m.nb_orient + 4 * (size_t)lks[k];
          quat_rotate_passive(__ldg(qq), __ldg(qq + 1), __ldg(qq + 2), __ldg(qq + 3), nx, ny, nz, nx, ny, nz);
        }
        sx = fmaf(ws[k], nx, sx);
        sy = fmaf(ws[k], ny, sy);
        sz = fmaf(ws[k], nz, sz);
      }
      s_x[(F + 0) * ACT_LD + tid] = sx;
      s_x[(F + 1) * ACT_LD + tid] = sy;
      s_x[(F + 2) * ACT_LD + tid] = sz;
      if (vec_ok) {
        for (int j = 0; j < F; j += 4) {
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int k = 0; k < PINB200_MAX_K; ++k) {
            if (lks[k] < 0) continue;
            const float4 v = __ldg(reinterpret_cast<const float4*>(feat + (size_t)lks[k] * F + j));
            acc.x = fmaf(ws[k], v.x, acc.x);
            acc.y = fmaf(ws[k], v.y, acc.y);
            acc.z = fmaf(ws[k], v.z, acc.z);
            acc.w = fmaf(ws[k], v.w, acc.w);
          }
          s_x[(j + 0) * ACT_LD + tid] = acc.x;
          s_x[(j + 1) * ACT_LD + tid] = acc.y;
          s_x[(j + 2) * ACT_LD + tid] = acc.z;
          s_x[(j + 3) * ACT_LD + tid] = acc.w;
        }
      } else {
        for (int j = 0; j < F; ++j) {
          float acc = 0.f;
#pragma unroll
          for (int k = 0; k < PINB200_MAX_K; ++k)
            if (lks[k] >= 0) acc = fmaf(ws[k], __ldg(feat + (size_t)lks[k] * F + j), acc);
          s_x[j * ACT_LD + tid] = acc;
        }
      }
    }
    __syncthreads();

    // ---------------- B: forward, activations kept per layer ----------------
    float g[H];
    {
      float h[H];
      const float* col_in = s_x + tid;
      int n_in = D;
      for (int l = 0; l < L; ++l) {
        matvec_col<H>(smem + p.lay.dec.wt[l], smem + p.lay.dec.b[l], col_in, n_in, h);
        s_mask[l * TILE + tid] = activate<H>(h, leaky);
        float* col_out = s_h + l * H * ACT_LD + tid;
        store_col<H>(col_out, h, H);
        col_in = col_out;
        n_in = H;
      }
      float go[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        go[c] = 0.f;
        if (c < OC) {
          float dv = p.dec.out_scale;
          if (p.dec.sigmoid_out) {
            const float* wo = smem + p.lay.dec.wout + c * H;
            float o = smem[p.lay.dec.bout + c];
#pragma unroll
            for (int j = 0; j < H; ++j) o = fmaf(wo[j], h[j], o);
            const float v = 1.f / (1.f + expf(-o));
            dv = v * (1.f - v);
          }
          go[c] = s_go[tid * 4 + c] * dv;
          s_go[tid * 4 + c] = go[c];
        }
      }
#pragma unroll
      for (int j = 0; j < H; ++j) {
        float t = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < OC) t = fmaf(go[c], smem[p.lay.dec.wout + c * H + j], t);
        g[j] = t;
      }
      apply_mask<H>(g, s_mask[(L - 1) * TILE + tid], leaky);
    }
    __syncthreads();

    // ---------------- C: output layer gradients ----------------
    {
      const float* hl = s_h + (L - 1) * H * ACT_LD;
      if (tid < H) {
        for (int c = 0; c < OC; ++c) {
          float t = 0.f;
          for (int r = 0; r < TILE; ++r) t = fmaf(s_go[r * 4 + c], hl[tid * ACT_LD + r], t);
          s_dW[off_wout + c * H + tid] += t;
        }
      } else if (tid < H + OC) {
        const int c = tid - H;
        float t = 0.f;
        for (int r = 0; r < TILE; ++r) t += s_go[r * 4 + c];
        s_dW[off_bout + c] += t;
      }
    }
    __syncthreads();

    // ---------------- hidden layers, last to first ----------------
    for (int l = L - 1; l >= 0; --l) {
      float* gl = s_h + l * H * ACT_LD;  // overwrite h_l with G_l (pre-activation gradient)
      store_col<H>(gl + tid, g, H);
      __syncthreads();
      if (l > 0) {
        tile_gemm_acc<8>(gl, s_h + (l - 1) * H * ACT_LD, H, s_dW + off_w[l], s_dW + off_b[l], tid);
        matvec_col<H>(smem + p.lay.dec.w[l], nullptr, gl + tid, H, g);
        apply_mask<H>(g, s_mask[(l - 1) * TILE + tid], leaky);
        __syncthreads();
      } else {
        tile_gemm_acc<NI0>(gl, s_x, D, s_dW + off_w[0], s_dW + off_b[0], tid);
        float gx[DP];
        matvec_col<DP>(smem + p.lay.dec.w[0], nullptr, gl + tid, H, gx);
        __syncthreads();  // everyone is done reading the x tile
        store_col<DP>(s_x + tid, gx, D);
        __syncthreads();
      }
    }

    // ---------------- D: scatter feature gradients (thread per tile row, 16-byte vector reductions) ----------------
    if (!wf) {
      const int ql = tid / K;
      const int lk = ql < QPT ? s_idx[tid] : -1;
      if (lk >= 0) {
        float* gr = p.grad_feat + (size_t)lk * F;
        if (vec_ok) {
          for (int j = 0; j < F; j += 4)
            atomicAdd(reinterpret_cast<float4*>(gr + j),
                      make_float4(s_x[(j + 0) * ACT_LD + tid], s_x[(j + 1) * ACT_LD + tid], s_x[(j + 2) * ACT_LD + tid],
                                  s_x[(j + 3) * ACT_LD + tid]));
        } else {
          for (int j = 0; j < F; ++j) atomicAdd(gr + j, s_x[j * ACT_LD + tid]);
        }
      }
    } else if (q0 + tid < p.n) {
      for (int k = 0; k < K; ++k) {
        const int lk = s_idx[tid * K + k];
        if (lk < 0) continue;
        const float w = s_w[tid * K + k];
        float* gr = p.grad_feat + (size_t)lk * F;
        if (vec_ok) {
          for (int j = 0; j < F; j += 4)
            atomicAdd(reinterpret_cast<float4*>(gr + j),
                      make_float4(w * s_x[(j + 0) * ACT_LD + tid], w * s_x[(j + 1) * ACT_LD + tid],
                                  w * s_x[(j + 2) * ACT_LD + tid], w * s_x[(j + 3) * ACT_LD + tid]));
        } else {
          for (int j = 0; j < F; ++j) atomicAdd(gr + j, w * s_x[j * ACT_LD + tid]);
        }
      }
    }
    __syncthreads();
  }
  for (int l = 0; l < L; ++l) {
    flush_block(s_dW + off_w[l], H * (l == 0 ? D : H), p.gd_w[l], tid);
    flush_block(s_dW + off_b[l], H, p.gd_b[l], tid);
  }
  flush_block(s_dW + off_wout, OC * H, p.gd_wout, tid);
  flush_block(s_dW + off_bout, OC, p.gd_bout, tid);
}

}  // namespace pinb

#include "train_mma.cuh"

namespace pinb {

template <int H, int DP>
static int launch_train(TrainParams& p, cudaStream_t stream) {
  TrainLayout l{};
  int o = 0;
  l.dec = plan_decoder_smem(p.dec, DP, true, o);
  o = l.dec.end;
  l.x = o;
  o += align4(DP * ACT_LD);
  l.h = o;
  o += align4(p.dec.n_hidden * H * ACT_LD);
  l.dW = o;
  o += align4(p.n_acc);
  l.go = o;
  o += TILE * 4;
  l.idx = o;
  o += TILE * p.K;
  l.w = o;
  o += TILE * p.K;
  l.q = o;
  o += TILE * 3;
  o = (o + 1) & ~1;
  l.mask = o;
  o += 2 * TILE * p.dec.n_hidden;
  l.total = o;
  p.lay = l;
  const size_t smem_bytes = (size_t)o * sizeof(float);
  if (smem_bytes > 227 * 1024) {
    set_error("train kernel needs %zu B shared memory (> 227 KB)", smem_bytes);
    return PINB200_ERR_UNSUPPORTED;
  }
  auto kern = train_bwd_kernel<H, DP>;
  int occ = 1;
  if (const int rc = prepare_kernel((const void*)kern, "train_bwd_kernel", smem_bytes, TILE, &occ)) return rc;
  const int grid = (int)std::min<long long>(p.n_tiles, (long long)sm_count() * occ);
  kern<<<grid, TILE, smem_bytes, stream>>>(p);
  return check_launch("train_bwd_kernel");
}

// the tensor-core kernel for 1-2 hidden layers over a 16-byte aligned feature table, the SIMT kernel (by padded
// decoder input width) otherwise
static int dispatch_train(TrainParams& p, cudaStream_t st) {
  const int F = p.map.feature_dim, L = p.dec.n_hidden, D = p.dec.in_dim;
  const bool aligned = (reinterpret_cast<uintptr_t>(p.feat) & 15) == 0;
  if (aligned && (L == 1 || L == 2)) {
    switch (F) {
      case 4: return L == 1 ? launch_train_mma<4, 1>(p, st) : launch_train_mma<4, 2>(p, st);
      case 8: return L == 1 ? launch_train_mma<8, 1>(p, st) : launch_train_mma<8, 2>(p, st);
      case 16: return L == 1 ? launch_train_mma<16, 1>(p, st) : launch_train_mma<16, 2>(p, st);
      case 32: return L == 1 ? launch_train_mma<32, 1>(p, st) : launch_train_mma<32, 2>(p, st);
      case 64: return L == 1 ? launch_train_mma<64, 1>(p, st) : launch_train_mma<64, 2>(p, st);
      default: break;
    }
  }
  if (D <= 12) return launch_train<64, 12>(p, st);
  if (D <= 20) return launch_train<64, 20>(p, st);
  if (D <= 36) return launch_train<64, 36>(p, st);
  if (D <= 68) return launch_train<64, 68>(p, st);
  set_error("decoder in_dim %d unsupported (<= 68)", D);
  return PINB200_ERR_UNSUPPORTED;
}

}  // namespace pinb

using namespace pinb;

extern "C" int pinb200_train_backward(const pinb200_map_view* map, const pinb200_decoder_view* dec, const float* feat,
                                      const float* query_xyz, const int32_t* knn_idx, const float* knn_weight,
                                      const float* dloss_dout, int64_t n, int32_t nn_k, int32_t weighted_first,
                                      float* grad_feat, float* grad_dec, void* stream) {
  if (!map || !dec || !feat || !query_xyz || !knn_idx || !knn_weight || !dloss_dout || !grad_feat || !grad_dec ||
      !map->nb_points) {
    set_error("train_backward: null argument");
    return PINB200_ERR_BAD_ARG;
  }
  if (dec->hidden_dim != 64 || dec->n_hidden < 1 || dec->n_hidden > PINB200_MAX_HIDDEN_LAYERS || dec->out_dim < 1 ||
      dec->out_dim > 4 || dec->in_dim != map->feature_dim + 3) {
    set_error("train_backward: unsupported decoder shape (hidden 64, 1..4 layers, out 1..4, in = F+3)");
    return PINB200_ERR_UNSUPPORTED;
  }
  if (nn_k < 1 || nn_k > PINB200_MAX_K) {
    set_error("nn_k %d out of range", nn_k);
    return PINB200_ERR_BAD_ARG;
  }
  if (map->after_pgo && !map->nb_orient) {
    set_error("map view: after_pgo needs nb_orient");
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  TrainParams p{};
  p.map = *map;
  p.dec = *dec;
  p.feat = feat;
  p.query_xyz = query_xyz;
  p.knn_idx = knn_idx;
  p.knn_w = knn_weight;
  p.dl = dloss_dout;
  p.n = n;
  p.K = nn_k;
  p.wf = weighted_first;
  p.qpt = weighted_first ? TILE : TILE / nn_k;
  p.n_tiles = (int)((n + p.qpt - 1) / p.qpt);
  p.grad_feat = grad_feat;
  {
    // each parameter block's place in the shared-memory accumulator (acc) and in the caller's gradient vector (g)
    const int H = dec->hidden_dim;
    int acc = 0;
    float* g = grad_dec;
    for (int l = 0; l < dec->n_hidden; ++l) {
      const int nw = H * (l == 0 ? dec->in_dim : H);
      p.acc_w[l] = acc;
      p.gd_w[l] = g;
      acc += nw;
      g += nw;
      p.acc_b[l] = acc;
      p.gd_b[l] = dec->b[l] ? g : nullptr;
      acc += H;
      if (dec->b[l]) g += H;
    }
    p.acc_wout = acc;
    p.gd_wout = g;
    acc += dec->out_dim * H;
    g += dec->out_dim * H;
    p.acc_bout = acc;
    p.gd_bout = dec->b_out ? g : nullptr;
    p.n_acc = acc + dec->out_dim;
  }
  return dispatch_train(p, (cudaStream_t)stream);
}
