// K2 on the tensor cores: the training backward pass with every contraction issued as warp-level
// mma.sync.m16n8k8 TF32 instructions (3xTF32 split, fp32 accumulate -- see mlp_chain.cuh).
//
// A CTA is 4 warps and works on 128-row tiles (row = query when weighted_first, else (query, neighbour) pair):
//   A   thread per row : re-gather the decoder input row from the saved kNN (float4 feature-row loads)
//   B   warp per 32 rows: forward layers; the output-layer gradients and G_{L-1} come straight from the
//       accumulator fragments
//   C   for l = L-1 .. 0:   (two block barriers per layer)
//         every warp stores its G_l rows over h_l                       | per warp
//         dW_l[16w..16w+16, :] += G_l^T A_{l-1}  over all 128 tile rows | warp w owns a 16-row slab of dW_l and
//                                                                       | keeps it in REGISTERS across all tiles
//         g_{l-1} = mask(G_l W_l)                                       | per warp, own 32 rows
//   D   thread per row : scatter d loss / d feature rows with 16-byte vector reductions
// The dW slabs are flushed once per CTA with global atomics; biases and the output layer go through a small
// shared-memory accumulator.
//
// Replaces the autograd reverse pass of utils/mapper.py:816-817 through model/neural_points.py:597-731
// (index_put_ accumulate) and model/decoder.py:61-85.  Included by train.cu (needs TrainParams).
#pragma once
#include "mlp_chain.cuh"

namespace pinb {

constexpr int LDH = 68;  // leading dimension of the hidden-activation tiles (== 4 mod 32)

struct TrainMmaLayout {
  WarpDecSmem dec;
  int x, h, dW, go, idx, w, total;
};

// dacc[nt] (16 x 8 C fragments of the slab  dW[j0 .. j0+16][8 nt .. 8 nt + 8]) += G^T A over the 128 tile rows
//   G: [128][LDG] row-major (rows = tile rows, cols = the 64 units of the layer),  A: [128][LDA] layer input
template <int NT, int LDG, int LDA>
__device__ __forceinline__ void dw_gemm_3xtf32(float (&dacc)[NT][4], const float* __restrict__ G, int j0,
                                               const float* __restrict__ A, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll 2
  for (int kk = 0; kk < TILE / 8; ++kk) {
    const float* gp = G + (kk * 8 + t) * LDG + j0 + g;
    uint32_t ah[4], al[4];
    split_tf32(gp[0], ah[0], al[0]);            // (m = g    , k = t    )
    split_tf32(gp[8], ah[1], al[1]);            // (m = g + 8, k = t    )
    split_tf32(gp[4 * LDG], ah[2], al[2]);      // (m = g    , k = t + 4)
    split_tf32(gp[4 * LDG + 8], ah[3], al[3]);  // (m = g + 8, k = t + 4)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float* bp = A + (kk * 8 + t) * LDA + nt * 8 + g;
      uint32_t bh[2], bl[2];
      split_tf32(bp[0], bh[0], bl[0]);        // (k = t    , n = g)
      split_tf32(bp[4 * LDA], bh[1], bl[1]);  // (k = t + 4, n = g)
      mma_tf32(dacc[nt], al, bh);
      mma_tf32(dacc[nt], ah, bl);
      mma_tf32(dacc[nt], ah, bh);
    }
  }
}

// column sums of a 32 x 64 fragment set (rows of this warp) added to dst[0..63] in shared memory
__device__ __forceinline__ void frag_colsum_to_smem(const float (&acc)[2][8][4], float* dst, int lane) {
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float v = (acc[0][nt][e] + acc[0][nt][e + 2]) + (acc[1][nt][e] + acc[1][nt][e + 2]);
      v += __shfl_xor_sync(FULL, v, 4);
      v += __shfl_xor_sync(FULL, v, 8);
      v += __shfl_xor_sync(FULL, v, 16);
      if (lane < 4) atomicAdd(dst + nt * 8 + 2 * lane + e, v);
    }
}

// flush a register slab to the flat gradient vector: dW[j0 + m][i] for i < n_in
template <int NT>
__device__ __forceinline__ void flush_slab(const float (&dacc)[NT][4], float* __restrict__ gW, int j0, int n_in,
                                           int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = j0 + g + 8 * (c >> 1), i = nt * 8 + 2 * t + (c & 1);
      const float v = dacc[nt][c];
      if (i < n_in && v != 0.f) atomicAdd(gW + (size_t)j * n_in + i, v);
    }
}

// resident CTAs per SM the register allocation targets (shared memory allows 3 for the small decoders)
template <int FT, int LT>
constexpr int train_mma_min_ctas() {
  return (LT == 1 && FT <= 16) ? 3 : ((LT == 1 || FT <= 16) ? 2 : 1);
}

template <int FT, int LT>
__global__ void __launch_bounds__(TILE, train_mma_min_ctas<FT, LT>()) train_bwd_mma_kernel(const __grid_constant__ TrainParams p,
                                                                const TrainMmaLayout lay) {
  constexpr int H = 64;
  constexpr int F = FT, D = FT + 3;
  constexpr int KP0 = dec_in_pad(FT), KT0 = KP0 / 8, LDX = KP0 + 4;
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const pinb200_map_view& m = p.map;
  const int K = p.K, OC = p.dec.out_dim;
  const bool wf = p.wf != 0, leaky = p.dec.leaky_relu != 0;
  const float* __restrict__ feat = p.feat;

  float* s_x = smem + lay.x;   // [TILE][LDX]
  float* s_h = smem + lay.h;   // LT tiles of [TILE][LDH]
  float* s_dW = smem + lay.dW; // biases + output layer, flat-gradient offsets
  float* s_go = smem + lay.go; // [TILE][4]
  int* s_idx = reinterpret_cast<int*>(smem + lay.idx);
  float* s_w = smem + lay.w;

  stage_warp_decoder(p.dec, lay.dec, smem);
  for (int e = tid; e < p.n_acc; e += TILE) s_dW[e] = 0.f;
  __syncthreads();

  float dacc0[KT0][4];
  float dacc1[LT == 2 ? 8 : 1][4];
#pragma unroll
  for (int nt = 0; nt < KT0; ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) dacc0[nt][c] = 0.f;
#pragma unroll
  for (int nt = 0; nt < (LT == 2 ? 8 : 1); ++nt)
#pragma unroll
    for (int c = 0; c < 4; ++c) dacc1[nt][c] = 0.f;

  const bool vec_red = (reinterpret_cast<uintptr_t>(p.grad_feat) & 15) == 0;
  float* xrow = s_x + tid * LDX;            // this thread's tile row
  float* xw = s_x + warp * 32 * LDX;        // this warp's 32 rows
  const int QPT = p.qpt;
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const long long q0 = (long long)tile * QPT;
    // ---------------- A: rebuild decoder inputs (thread per tile row) ----------------
    {
      float go[4] = {0.f, 0.f, 0.f, 0.f};
      float nx = 0.f, ny = 0.f, nz = 0.f;
      if (!wf) {
        const int ql = tid / K, k = tid - ql * K;
        const long long qi = q0 + ql;
        int lk = -1;
        float w = 0.f;
        if (ql < QPT && qi < p.n) {
          lk = __ldg(p.knn_idx + qi * K + k);
          w = __ldg(p.knn_w + qi * K + k);
        }
        s_idx[tid] = lk;
        if (lk >= 0) {
          const float* pp = m.nb_points + 3 * (size_t)lk;
          nx = __fsub_rn(__ldg(p.query_xyz + 3 * qi), __ldg(pp));
          ny = __fsub_rn(__ldg(p.query_xyz + 3 * qi + 1), __ldg(pp + 1));
          nz = __fsub_rn(__ldg(p.query_xyz + 3 * qi + 2), __ldg(pp + 2));
          if (m.after_pgo) {
            const float* qq = m.nb_orient + 4 * (size_t)lk;
            quat_rotate_passive(__ldg(qq), __ldg(qq + 1), __ldg(qq + 2), __ldg(qq + 3), nx, ny, nz, nx, ny, nz);
          }
          const float4* fr = reinterpret_cast<const float4*>(feat + (size_t)lk * F);
#pragma unroll
          for (int j = 0; j < F / 4; ++j) *reinterpret_cast<float4*>(xrow + 4 * j) = __ldg(fr + j);
          for (int c = 0; c < OC; ++c) go[c] = __ldg(p.dl + qi * OC + c) * w;
        } else {
#pragma unroll
          for (int j = 0; j < F / 4; ++j) *reinterpret_cast<float4*>(xrow + 4 * j) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      } else {
        const long long qi = q0 + tid;
        const bool live = qi < p.n;
        int lks[PINB200_MAX_K];
        float ws[PINB200_MAX_K];
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
          for (int c = 0; c < OC; ++c) go[c] = __ldg(p.dl + qi * OC + c);
        }
#pragma unroll
        for (int k = 0; k < PINB200_MAX_K; ++k) {
          if (lks[k] < 0) continue;
          const float* pp = m.nb_points + 3 * (size_t)lks[k];
          float ux = __fsub_rn(qx, __ldg(pp)), uy = __fsub_rn(qy, __ldg(pp + 1)), uz = __fsub_rn(qz, __ldg(pp + 2));
          if (m.after_pgo) {
            const float* qq = m.nb_orient + 4 * (size_t)lks[k];
            quat_rotate_passive(__ldg(qq), __ldg(qq + 1), __ldg(qq + 2), __ldg(qq + 3), ux, uy, uz, ux, uy, uz);
          }
          nx = fmaf(ws[k], ux, nx);
          ny = fmaf(ws[k], uy, ny);
          nz = fmaf(ws[k], uz, nz);
        }
#pragma unroll
        for (int j = 0; j < F / 4; ++j) {
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int k = 0; k < PINB200_MAX_K; ++k) {
            if (lks[k] < 0) continue;
            const float4 v = __ldg(reinterpret_cast<const float4*>(feat + (size_t)lks[k] * F) + j);
            acc.x = fmaf(ws[k], v.x, acc.x);
            acc.y = fmaf(ws[k], v.y, acc.y);
            acc.z = fmaf(ws[k], v.z, acc.z);
            acc.w = fmaf(ws[k], v.w, acc.w);
          }
          *reinterpret_cast<float4*>(xrow + 4 * j) = acc;
        }
      }
      xrow[F + 0] = nx;
      xrow[F + 1] = ny;
      xrow[F + 2] = nz;
#pragma unroll
      for (int d = D; d < KP0; ++d) xrow[d] = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) s_go[tid * 4 + c] = go[c];
    }
    __syncwarp();

    // ---------------- B: forward on this warp's 32 rows ----------------
    float acc[2][8][4];
    uint64_t mk[LT];
    warp_gemm_3xtf32<KT0, 8, false, LDX>(acc, xw, smem + lay.dec.whi[0], smem + lay.dec.wlo[0], lay.dec.ldw[0], lane);
    mk[0] = bias_act_chain<8>(acc, smem + lay.dec.b[0], leaky, lane);
    if constexpr (LT == 2) {
      float* h0w = s_h + warp * 32 * LDH;
      store_frags<8, LDH>(h0w, acc, lane);  // h_0: input of layer 1 and of dW_1
      __syncwarp();
      warp_gemm_3xtf32<8, 8, false, LDH>(acc, h0w, smem + lay.dec.whi[1], smem + lay.dec.wlo[1], lay.dec.ldw[1], lane);
      mk[LT - 1] = bias_act_chain<8>(acc, smem + lay.dec.b[1], leaky, lane);
    }
    // d loss / d pre-output per row (sigmoid heads need the output value), output-layer gradients
    {
      const float* wo = smem + lay.dec.wout;
      float gor[2][2][4];  // [mt][hh][c]: this lane's 4 rows
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = warp * 32 + mt * 16 + (lane >> 2) + 8 * hh;
#pragma unroll
          for (int c = 0; c < 4; ++c) gor[mt][hh][c] = c < OC ? s_go[row * 4 + c] : 0.f;
        }
      if (p.dec.sigmoid_out) {
        for (int c = 0; c < OC; ++c) {
          float part[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
              for (int e = 0; e < 4; ++e)
                part[mt][e >> 1] = fmaf(acc[mt][nt][e], wo[c * H + frag_col(nt, e, lane)], part[mt][e >> 1]);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              float v = part[mt][hh];
              v += __shfl_xor_sync(FULL, v, 1);
              v += __shfl_xor_sync(FULL, v, 2);
              const float o = 1.f / (1.f + expf(-(v + smem[lay.dec.bout + c])));
#pragma unroll
              for (int cc = 0; cc < 4; ++cc)
                if (cc == c) gor[mt][hh][cc] *= o * (1.f - o);
            }
        }
      } else {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int c = 0; c < 4; ++c) gor[mt][hh][c] *= p.dec.out_scale;
      }
      // dW_out[c][j] += sum_r go[r][c] h[r][j],  db_out[c] += sum_r go[r][c]
      for (int c = 0; c < OC; ++c) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v = 0.f;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int cc = 0; cc < 4; ++cc)
                  if (cc == c) v = fmaf(gor[mt][hh][cc], acc[mt][nt][2 * hh + e], v);
            v += __shfl_xor_sync(FULL, v, 4);
            v += __shfl_xor_sync(FULL, v, 8);
            v += __shfl_xor_sync(FULL, v, 16);
            if (lane < 4) atomicAdd(s_dW + p.acc_wout + c * H + nt * 8 + 2 * lane + e, v);
          }
        float b = 0.f;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int cc = 0; cc < 4; ++cc)
              if (cc == c) b += gor[mt][hh][cc];
        if ((lane & 3) != 0) b = 0.f;  // the 4 lanes of a quad hold the same rows
        b = warp_sum(b);
        if (lane == 0) atomicAdd(s_dW + p.acc_bout + c, b);
      }
      // G_{L-1} = mask * (go w_out)
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float v = 0.f;
#pragma unroll
            for (int c = 0; c < 4; ++c)
              if (c < OC) v = fmaf(gor[mt][e >> 1][c], wo[c * H + frag_col(nt, e, lane)], v);
            acc[mt][nt][e] = v;
          }
      mask_chain<8>(acc, mk[LT - 1], leaky);
    }

    // ---------------- C: hidden layers, last to first ----------------
    if constexpr (LT == 2) {
      float* g1 = s_h + TILE * LDH;  // G_1 tile
      frag_colsum_to_smem(acc, s_dW + p.acc_b[1], lane);
      store_frags<8, LDH>(g1 + warp * 32 * LDH, acc, lane);
      __syncthreads();  // G_1 and h_0 of all 128 rows are in place
      dw_gemm_3xtf32<8, LDH, LDH>(dacc1, g1, warp * 16, s_h, lane);
      warp_gemm_3xtf32<8, 8, true, LDH>(acc, g1 + warp * 32 * LDH, smem + lay.dec.whi[1], smem + lay.dec.wlo[1],
                                        lay.dec.ldw[1], lane);
      mask_chain<8>(acc, mk[0], leaky);
      __syncthreads();  // everyone is done reading h_0
    }
    frag_colsum_to_smem(acc, s_dW + p.acc_b[0], lane);
    store_frags<8, LDH>(s_h + warp * 32 * LDH, acc, lane);  // G_0 over h_0
    __syncthreads();  // G_0 and x of all 128 rows are in place
    dw_gemm_3xtf32<KT0, LDH, LDX>(dacc0, s_h, warp * 16, s_x, lane);
    float gxa[2][KT0][4];
    warp_gemm_3xtf32<8, KT0, true, LDH>(gxa, s_h + warp * 32 * LDH, smem + lay.dec.whi[0], smem + lay.dec.wlo[0],
                                        lay.dec.ldw[0], lane);
    __syncthreads();  // everyone is done reading the x tile
    store_frags<KT0, LDX>(xw, gxa, lane);
    __syncwarp();

    // ---------------- D: scatter feature gradients (thread per tile row) ----------------
    if (!wf) {
      const int lk = s_idx[tid];
      if (lk >= 0) {
        float* gr = p.grad_feat + (size_t)lk * F;
        if (vec_red) {
#pragma unroll
          for (int j = 0; j < F / 4; ++j)
            atomicAdd(reinterpret_cast<float4*>(gr) + j, *reinterpret_cast<const float4*>(xrow + 4 * j));
        } else {
          for (int j = 0; j < F; ++j) atomicAdd(gr + j, xrow[j]);
        }
      }
    } else if (q0 + tid < p.n) {
      for (int k = 0; k < K; ++k) {
        const int lk = s_idx[tid * K + k];
        if (lk < 0) continue;
        const float w = s_w[tid * K + k];
        float* gr = p.grad_feat + (size_t)lk * F;
        if (vec_red) {
#pragma unroll
          for (int j = 0; j < F / 4; ++j) {
            const float4 v = *reinterpret_cast<const float4*>(xrow + 4 * j);
            atomicAdd(reinterpret_cast<float4*>(gr) + j, make_float4(w * v.x, w * v.y, w * v.z, w * v.w));
          }
        } else {
          for (int j = 0; j < F; ++j) atomicAdd(gr + j, w * xrow[j]);
        }
      }
    }
    __syncwarp();  // the next tile's gather overwrites this warp's x rows
  }

  // ---------------- flush the decoder gradients ----------------
  flush_slab<KT0>(dacc0, p.gd_w[0], warp * 16, D, lane);
  if constexpr (LT == 2) flush_slab<8>(dacc1, p.gd_w[1], warp * 16, H, lane);
  __syncthreads();
  flush_block(s_dW + p.acc_b[0], H, p.gd_b[0], tid);
  if constexpr (LT == 2) flush_block(s_dW + p.acc_b[1], H, p.gd_b[1], tid);
  flush_block(s_dW + p.acc_wout, OC * H, p.gd_wout, tid);
  flush_block(s_dW + p.acc_bout, OC, p.gd_bout, tid);
}

template <int FT, int LT>
static int launch_train_mma(TrainParams& p, cudaStream_t stream) {
  constexpr int LDX = dec_in_pad(FT) + 4;
  TrainMmaLayout l{};
  // leading dimensions == 4 (mod 32): conflict-free scalar fragment loads in warp_gemm_3xtf32
  l.dec = plan_warp_decoder_smem(p.dec, dec_in_pad(FT), 0, [](int k) { return k + 4; });
  int o = align4(l.dec.end);
  l.x = o;
  o += TILE * LDX;
  l.h = o;
  o += LT * TILE * LDH;
  l.dW = o;
  o += align4(p.n_acc);
  l.go = o;
  o += TILE * 4;
  l.idx = o;
  o += TILE * PINB200_MAX_K;
  l.w = o;
  o += TILE * PINB200_MAX_K;
  l.total = o;
  const size_t smem_bytes = (size_t)o * sizeof(float);
  if (smem_bytes > 227 * 1024) {
    set_error("train kernel needs %zu B shared memory (> 227 KB)", smem_bytes);
    return PINB200_ERR_UNSUPPORTED;
  }
  auto kern = train_bwd_mma_kernel<FT, LT>;
  int occ = 1;
  if (const int rc = prepare_kernel((const void*)kern, "train_bwd_mma_kernel", smem_bytes, TILE, &occ)) return rc;
  const int grid = (int)std::min<long long>(p.n_tiles, (long long)sm_count() * occ);
  kern<<<grid, TILE, smem_bytes, stream>>>(p, l);
  return check_launch("train_bwd_mma_kernel");
}

}  // namespace pinb
