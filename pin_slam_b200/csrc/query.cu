// K1: fused voxel-hash kNN + IDW interpolation + decoder MLP + analytic d/dq  (round-2 rewrite).
//
// Every WARP owns an independent tile of 32 queries (no block-wide barriers after the one-off weight staging: the
// 12 de-synchronised warps of the one CTA per SM overlap each other's memory and compute phases).  The phases of a
// tile and the thread mapping each one uses:
//   A1  thread per query   hash the query's cell; probe the C neighbour cells: ONE 16-byte load per probe from the
//                          probe index (probe_index.cu); branch-free top-8 selection with sorting
//                          networks (knn_select.cuh); the 8 winners' records are re-read (L1 hits) for positions and
//                          ids; IDW weights, certainty, training-mode scatters, kNN outputs; everything later phases
//                          need is stashed in [k][lane] shared-memory columns (conflict free)
//   A2  F/4 lanes per row  16-byte coalesced gathers of the K feature rows of 128/F queries at a time (a 128-byte row
//                          = 8 lanes x LDG.128: one L1 wavefront per row, 4 rows per instruction) and the IDW
//                          reduction in registers -> decoder input rows in the warp's row-major tile
//   B   warp MMA           decoder forward + backward to the decoder input on mma.sync 3xTF32 with register-chained
//                          fragments (mlp_chain.cuh): only layer 0's input and the input gradient touch shared memory
//   C1  F/4 lanes per row  a_k = <d sdf / d feature part of the input, f_k> (second coalesced pass over the K rows)
//   C2  thread per query   chain rule through the IDW weights and the neighbour vectors -> d sdf / d q, outputs
// weighted_first=0 decodes every (query, neighbour) pair: the 32 queries are processed in row tiles of floor(32/K)
// queries x K rows, and C combines the K per-neighbour values (IDW mean / std, utils/tracker.py:313-328).
//
// Replaces model/neural_points.py:530-746,950-1009, model/decoder.py:61-85,112,
// utils/tools.py:247-260, utils/tracker.py:313-328 of the reference.
#include "query_dev.cuh"

namespace pinb {

// K1a of the split pipeline: phase A1 alone, at high occupancy (no decoder weights in shared memory, <= 128
// registers): the probe rounds of ~16 resident warps per SM keep the load/store unit busy, which the fused kernel's
// 12 warps (most of them in compute phases at any time) cannot.  One warp = one 32-query tile.  COMPACT: the stash
// blocks are StashS blocks (the decode runs on wsq_decode_kernel); with p.perm the tiles are runs of p.perm
// (spatially sorted queries).
template <bool SEEDS, bool COMPACT>
__global__ void __launch_bounds__(128, 4) search_kernel(const __grid_constant__ QueryParams p) {
  extern __shared__ __align__(16) float smem[];
  uint32_t* s_delta = reinterpret_cast<uint32_t*>(smem);
  // programmatic dependent launch: the decode launch may start its prologue (mbarriers, weight staging) on the
  // SMs this grid's tail frees; it waits (griddepcontrol.wait) before it reads anything written here
  asm volatile("griddepcontrol.launch_dependents;");
  fill_probe_deltas(p.map, s_delta);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int st = blockIdx.x * nwarp + warp; st < p.n_tiles; st += gridDim.x * nwarp)
    a1_tile<SEEDS, COMPACT>(p, s_delta, (long long)st * WT, WT, lane,
                            p.stash + (size_t)st * (COMPACT ? StashS::floats : Stash::floats));
}

// ---------------------------------------------------------------------------
// the fused kernel
// ---------------------------------------------------------------------------
// SPLIT = false: fused (phase A1 runs here);  true: decode-only launch of the split pipeline (the stash of every tile
// was written by search_kernel)
template <int FT, bool WF, bool SPLIT>
__global__ void __launch_bounds__(WPB * 32, 1) query_kernel(const __grid_constant__ QueryParams p) {
  constexpr int H = 64;
  constexpr int KP0 = dec_in_pad(FT);  // decoder input width padded to the MMA k-step
  constexpr int KT0 = KP0 / 8;         // k-steps of layer 0 == n-tiles of the input gradient
  constexpr int LDX = ld8mod32(KP0);   // row-major tile leading dimension (== 8 mod 32)
  constexpr int F = FT, D = FT + 3;
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const pinb200_map_view& m = p.map;
  const int K = p.opts.nn_k, L = p.dec.n_hidden;
  const int OC = p.dec.out_dim;
  const bool need_grad = p.opts.need_grad != 0;
  const bool leaky = p.dec.leaky_relu != 0;
  const float* __restrict__ feat = p.feat;

  using WL = WarpLay<FT>;
  static_assert(WL::LDX == LDX && (WL::mask % 2) == 0 && (WL::stride % 4) == 0 && (WL::stash % 4) == 0 && Stash::floats == 1536, "per-warp layout");
  uint32_t* s_delta = reinterpret_cast<uint32_t*>(smem + p.lay.delta);
  float* wsm = smem + p.lay.warp0 + warp * WL::stride;  // this warp's private tile state
  float* s_x = wsm + WL::x;
  int* s_li = reinterpret_cast<int*>(wsm + WL::stash + Stash::li);
  float* s_w = wsm + WL::stash + Stash::w;
  float* s_dx = wsm + WL::stash + Stash::dx;
  float* s_dy = wsm + WL::stash + Stash::dy;
  float* s_dz = wsm + WL::stash + Stash::dz;
  float* s_q = wsm + WL::stash + Stash::q;
  float* s_usum = wsm + WL::stash + Stash::usum;
  int* s_nn = reinterpret_cast<int*>(wsm + WL::stash + Stash::nn);
  float* s_pos = wsm + WL::stash + Stash::pos;
  float* s_a = wsm + WL::a;
  float* s_out = wsm + WL::out;
  float* s_dv = wsm + WL::dv;
  uint64_t* s_mask = reinterpret_cast<uint64_t*>(wsm + WL::mask);

  stage_warp_decoder(p.dec, p.lay.dec, smem);
  if (!SPLIT && !p.use_saved_knn) fill_probe_deltas(m, s_delta);
  __syncthreads();

  const int QPT = WF ? WT : WT / K;                // queries per 32-row decoder tile
  const int WQ = p.qpt;                            // queries per warp tile (<= WT; small launches use fewer so
                                                   // that every resident warp gets work: latency, not issue, bound)
  const int n_rt = WF ? 1 : (WQ + QPT - 1) / QPT;  // row tiles per warp tile
  const int nwarp = blockDim.x >> 5;
  for (int st = blockIdx.x * nwarp + warp; st < p.n_tiles; st += gridDim.x * nwarp) {
    const long long q0s = (long long)st * WQ;

    // ============ phase A1: thread per query -- search, IDW weights, side effects, stash ============
    if (SPLIT) {  // the search launch did it: copy the tile's stash block (coalesced 16-byte accesses)
      const float4* __restrict__ src = reinterpret_cast<const float4*>(p.stash + (size_t)st * Stash::floats);
      float4* dst = reinterpret_cast<float4*>(wsm + WL::stash);
      float4 t[Stash::floats / 128];
#pragma unroll
      for (int i = 0; i < Stash::floats / 128; ++i) t[i] = __ldg(src + i * 32 + lane);
#pragma unroll
      for (int i = 0; i < Stash::floats / 128; ++i) dst[i * 32 + lane] = t[i];
      __syncwarp();
    } else {
      a1_tile(p, s_delta, q0s, WQ, lane, wsm + WL::stash);
    }
    if (WF) {  // the position part of the IDW-averaged decoder input (this thread's tile row) + zero padding
      s_x[lane * LDX + F + 0] = s_pos[0 * WT + lane];
      s_x[lane * LDX + F + 1] = s_pos[1 * WT + lane];
      s_x[lane * LDX + F + 2] = s_pos[2 * WT + lane];
#pragma unroll
      for (int d = D; d < KP0; ++d) s_x[lane * LDX + d] = 0.f;
    }
    __syncwarp();

    for (int rt = 0; rt < n_rt; ++rt) {
      const int sq0 = rt * QPT;            // first query of this row tile inside the warp tile
      const int qpt = min(QPT, WQ - sq0);  // queries in this row tile
      const int used_rows = WF ? WT : qpt * K;

      // ============ phase A2: F/4 lanes per row -- coalesced feature gathers into the tile ============
      if (WF) {
        gather_weighted<FT, LDX>(feat, K, WQ, s_li, s_w, lane, s_x);
      } else {
        gather_rows<FT, LDX>(feat, K, used_rows, sq0, s_li, lane, s_x);
        // neighbour vectors of the (query, k) rows: thread per row
        float nx = 0.f, ny = 0.f, nz = 0.f;
        if (lane < used_rows) {
          const int ql = lane / K, k = lane - ql * K, sq = sq0 + ql;
          const int lif = s_li[k * WT + sq];
          if (lif >= 0) {
            float4 quat;
            neighbour_vec(m, lif, s_dx[k * WT + sq], s_dy[k * WT + sq], s_dz[k * WT + sq], s_q[sq], s_q[WT + sq],
                          s_q[2 * WT + sq], nx, ny, nz, quat);
          }
        }
        s_x[lane * LDX + F + 0] = nx;
        s_x[lane * LDX + F + 1] = ny;
        s_x[lane * LDX + F + 2] = nz;
#pragma unroll
        for (int d = D; d < KP0; ++d) s_x[lane * LDX + d] = 0.f;
      }
      __syncwarp();

      // ============ phase B: decoder on the tensor cores (warp-level 3xTF32 MMA, register-chained) ============
      float acc[2][8][4];
      gemm_from_tile<KT0, LDX>(acc, s_x, smem + p.lay.dec.whi[0], smem + p.lay.dec.wlo[0], p.lay.dec.ldw[0], lane);
      s_mask[lane] = bias_act_chain<8>(acc, smem + p.lay.dec.b[0], leaky, lane);
      for (int l = 1; l < L; ++l) {
        float nxt[2][8][4];
        gemm_chain_fwd(nxt, acc, smem + p.lay.dec.whi[l], smem + p.lay.dec.wlo[l], p.lay.dec.ldw[l], lane);
        s_mask[l * WT + lane] = bias_act_chain<8>(nxt, smem + p.lay.dec.b[l], leaky, lane);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[mt][nt][e] = nxt[mt][nt][e];
      }
      // output head(s): dot with w_out over the 64 hidden units; 4 lanes share a row
      for (int c = 0; c < OC; ++c) {
        const float* wo = smem + p.lay.dec.wout + c * H;
        float part[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const float2 w2 = *reinterpret_cast<const float2*>(wo + frag_col(nt, 0, lane));
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int e = 0; e < 4; ++e) part[mt][e >> 1] = fmaf(acc[mt][nt][e], (e & 1) ? w2.y : w2.x, part[mt][e >> 1]);
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float v = part[mt][hh];
            v += __shfl_xor_sync(FULL, v, 1);
            v += __shfl_xor_sync(FULL, v, 2);
            if ((lane & 3) == 0) {
              const int row = mt * 16 + (lane >> 2) + 8 * hh;
              const float o = v + smem[p.lay.dec.bout + c];
              float val, dv;
              if (p.dec.sigmoid_out) {
                val = 1.f / (1.f + expf(-o));
                dv = val * (1.f - val);
              } else {
                val = o * p.dec.out_scale;
                dv = p.dec.out_scale;
              }
              s_out[row * 4 + c] = val;
              s_dv[row * 4 + c] = dv;
            }
          }
      }
      __syncwarp();

      // ======== per output channel: backward to the decoder input, then the IDW chain rule ========
      const int n_pass = need_grad ? OC : 1;
      for (int c = 0; c < n_pass; ++c) {
        if (need_grad) {
          const float* wo = smem + p.lay.dec.wout + c * H;
#pragma unroll
          for (int nt = 0; nt < 8; ++nt) {
            const float2 w2 = *reinterpret_cast<const float2*>(wo + frag_col(nt, 0, lane));
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int e = 0; e < 4; ++e) acc[mt][nt][e] = (e & 1) ? w2.y : w2.x;
          }
          mask_chain<8>(acc, s_mask[(L - 1) * WT + lane], leaky);
          for (int l = L - 1; l >= 1; --l) {
            float nxt[2][8][4];
            gemm_chain_bwd<8>(nxt, acc, smem + p.lay.dec.whi[l], smem + p.lay.dec.wlo[l], p.lay.dec.ldw[l], lane);
            mask_chain<8>(nxt, s_mask[(l - 1) * WT + lane], leaky);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[mt][nt][e] = nxt[mt][nt][e];
          }
          float gxa[2][KT0][4];
          gemm_chain_bwd<KT0>(gxa, acc, smem + p.lay.dec.whi[0], smem + p.lay.dec.wlo[0], p.lay.dec.ldw[0], lane);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const float dv = s_dv[(mt * 16 + (lane >> 2) + 8 * hh) * 4 + c];
#pragma unroll
              for (int nt = 0; nt < KT0; ++nt) {
                gxa[mt][nt][2 * hh] *= dv;
                gxa[mt][nt][2 * hh + 1] *= dv;
              }
            }
          __syncwarp();
          store_frags<KT0, LDX>(s_x, gxa, lane);
        }
        __syncwarp();

        if (WF) {
          // ---- C1: a_k = <g_xbar, f_k> (F/4 lanes per row, coalesced re-read of the K feature rows)
          if (need_grad) {
            feature_dots<FT, LDX>(feat, K, WQ, s_li, lane, s_x, s_a);
            __syncwarp();
          }
          // ---- C2: thread per query -- chain rule through the IDW weights, outputs
          const long long qi = q0s + lane;
          if (lane < WQ && qi < p.n) {
            const float val = s_out[lane * 4 + c];
            float gq0 = 0.f, gq1 = 0.f, gq2 = 0.f;
            if (need_grad) {
              const int nn = s_nn[lane];
              const float usum = s_usum[lane];
              const float qx = s_q[lane], qy = s_q[WT + lane], qz = s_q[2 * WT + lane];
              const float gn0 = s_x[lane * LDX + F + 0], gn1 = s_x[lane * LDX + F + 1], gn2 = s_x[lane * LDX + F + 2];
              float ak[KREG], wk[KREG], ck[KREG], dx[KREG], dy[KREG], dz[KREG];
#pragma unroll
              for (int k = 0; k < KREG; ++k) {
                ak[k] = wk[k] = ck[k] = dx[k] = dy[k] = dz[k] = 0.f;
                const int lif = k < K ? s_li[k * WT + lane] : -1;
                if (lif >= 0) {
                  dx[k] = s_dx[k * WT + lane];  // q - the point dist2 was measured to
                  dy[k] = s_dy[k * WT + lane];
                  dz[k] = s_dz[k * WT + lane];
                  float nx, ny, nz, r0 = gn0, r1 = gn1, r2 = gn2;
                  float4 quat;
                  neighbour_vec(m, lif, dx[k], dy[k], dz[k], qx, qy, qz, nx, ny, nz, quat);
                  if (m.after_pgo) quat_rotate_active(quat.x, quat.y, quat.z, quat.w, gn0, gn1, gn2, r0, r1, r2);
                  wk[k] = s_w[k * WT + lane];
                  ak[k] = s_a[k * WT + lane] + gn0 * nx + gn1 * ny + gn2 * nz;
                  ck[k] = nn > 0 ? -2.f * (wk[k] * usum) : 0.f;  // -2 u_k,  u_k = 1/(d2+eps) = w_k * sum_j u_j
                  gq0 = fmaf(wk[k], r0, gq0);
                  gq1 = fmaf(wk[k], r1, gq1);
                  gq2 = fmaf(wk[k], r2, gq2);
                }
              }
              // d w_k / d q = w_k (c_k - sum_j w_j c_j),  c_k = -2 u_k (q - p_k).
              // sum_k w_k (a_k - abar) c_k is invariant to a common shift of the a_k; shifting by the nearest
              // neighbour's a_0 first keeps (a_k - abar) exact when neighbours coincide (cancellation-free)
              float abar = 0.f;
              {
                const float a0 = ak[0];
#pragma unroll
                for (int k = 0; k < KREG; ++k) {
                  ak[k] = wk[k] != 0.f ? ak[k] - a0 : 0.f;
                  abar = fmaf(wk[k], ak[k], abar);
                }
              }
#pragma unroll
              for (int k = 0; k < KREG; ++k) {
                const float coef = wk[k] * (ak[k] - abar) * ck[k];
                gq0 = fmaf(coef, dx[k], gq0);
                gq1 = fmaf(coef, dy[k], gq1);
                gq2 = fmaf(coef, dz[k], gq2);
              }
            }
            if (!p.is_color) {
              if (p.out.sdf) p.out.sdf[qi] = val;
              if (p.out.sdf_std) p.out.sdf_std[qi] = 0.f;
              if (need_grad && p.out.grad) {
                p.out.grad[3 * qi + 0] = gq0;
                p.out.grad[3 * qi + 1] = gq1;
                p.out.grad[3 * qi + 2] = gq2;
              }
            } else {
              if (p.out.color) {
                if (need_grad) {
                  p.out.color[qi * OC + c] = val;
                } else {
                  for (int cc = 0; cc < OC; ++cc) p.out.color[qi * OC + cc] = s_out[lane * 4 + cc];
                }
              }
              if (need_grad && p.out.color_grad) {
                p.out.color_grad[(qi * OC + c) * 3 + 0] = gq0;
                p.out.color_grad[(qi * OC + c) * 3 + 1] = gq1;
                p.out.color_grad[(qi * OC + c) * 3 + 2] = gq2;
              }
            }
          }
        } else {
          // decode-every-neighbour: thread per query combines its K rows (tracker.py:317-323)
          if (lane < qpt && q0s + sq0 + lane < p.n) {
            const int ql = lane, sq = sq0 + ql;
            const long long qi = q0s + sq;
            const int nn = s_nn[sq];
            const float usum = s_usum[sq];
            const int n_ch = (need_grad || !p.is_color) ? 1 : OC;
            for (int ch = 0; ch < n_ch; ++ch) {
              const int cc = need_grad ? c : ch;
              float mean = 0.f, msh = 0.f;
              const float s0 = s_out[(ql * K) * 4 + cc];  // nearest neighbour's value: shift for exact differences
              for (int k = 0; k < K; ++k) {
                const float wk = s_w[k * WT + sq];
                mean = fmaf(wk, s_out[(ql * K + k) * 4 + cc], mean);
                msh = fmaf(wk, s_out[(ql * K + k) * 4 + cc] - s0, msh);
              }
              float var = 0.f, g0 = 0.f, g1 = 0.f, g2 = 0.f;
              for (int k = 0; k < K; ++k) {
                const int lif = s_li[k * WT + sq];
                if (lif < 0) continue;
                const float wk = s_w[k * WT + sq];
                const float dm = (s_out[(ql * K + k) * 4 + cc] - s0) - msh;  // == s_k - mean, cancellation-free
                var = fmaf(wk * dm, dm, var);
                if (need_grad) {
                  const int row = ql * K + k;
                  float r0 = s_x[row * LDX + F + 0], r1 = s_x[row * LDX + F + 1], r2 = s_x[row * LDX + F + 2];
                  if (m.after_pgo) {
                    const float4 qq = __ldg(reinterpret_cast<const float4*>(m.nb_orient) + (lif & ~REMAP));
                    quat_rotate_active(qq.x, qq.y, qq.z, qq.w, r0, r1, r2, r0, r1, r2);
                  }
                  const float uk = nn > 0 ? wk * usum : 0.f;
                  const float coef = wk * dm * (-2.f * uk);
                  g0 += fmaf(coef, s_dx[k * WT + sq], wk * r0);
                  g1 += fmaf(coef, s_dy[k * WT + sq], wk * r1);
                  g2 += fmaf(coef, s_dz[k * WT + sq], wk * r2);
                }
              }
              if (!p.is_color) {
                if (p.out.sdf) p.out.sdf[qi] = mean;
                if (p.out.sdf_std) p.out.sdf_std[qi] = sqrtf(var);
                if (need_grad && p.out.grad) {
                  p.out.grad[3 * qi + 0] = g0;
                  p.out.grad[3 * qi + 1] = g1;
                  p.out.grad[3 * qi + 2] = g2;
                }
              } else {
                if (p.out.color) p.out.color[qi * OC + cc] = mean;
                if (need_grad && p.out.color_grad) {
                  p.out.color_grad[(qi * OC + cc) * 3 + 0] = g0;
                  p.out.color_grad[(qi * OC + cc) * 3 + 1] = g1;
                  p.out.color_grad[(qi * OC + cc) * 3 + 2] = g2;
                }
              }
            }
          }
        }
        __syncwarp();
      }
    }
  }
}

// ---------------------------------------------------------------------------
// search-only kernels (warp per query, no decoder)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(TILE) knn_kernel(const __grid_constant__ pinb200_map_view m,
                                                   const float* __restrict__ query_xyz, long long n, int K,
                                                   int32_t* knn_idx, int32_t* knn_gidx, float* knn_d2, float* knn_w,
                                                   int32_t* nn_count) {
  extern __shared__ __align__(16) float smem[];
  uint32_t* s_delta = reinterpret_cast<uint32_t*>(smem);
  fill_probe_deltas(m, s_delta);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long wpb = blockDim.x >> 5;
  for (long long qi = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); qi < n; qi += (long long)gridDim.x * wpb) {
    const float qx = __ldg(query_xyz + 3 * qi), qy = __ldg(query_xyz + 3 * qi + 1), qz = __ldg(query_xyz + 3 * qi + 2);
    const Knn kn = knn_search_warp(m, s_delta, qx, qy, qz, K, lane);
    float u, inv_s;
    const float w = idw_weight(kn.d2, kn.idx >= 0, kn.count, K, lane, u, inv_s);
    if (lane < K) {
      if (knn_idx) knn_idx[qi * K + lane] = kn.idx;
      if (knn_gidx) knn_gidx[qi * K + lane] = kn.gidx;
      if (knn_d2) knn_d2[qi * K + lane] = kn.d2;
      if (knn_w) knn_w[qi * K + lane] = w;
    }
    if (lane == 0 && nn_count) nn_count[qi] = kn.count;
  }
}

// all-probe radius search: dist2 [N,C], global ids [N,C] (model/neural_points.py:950-1009)
__global__ void __launch_bounds__(TILE) radius_kernel(const __grid_constant__ pinb200_map_view m,
                                                      const float* __restrict__ query_xyz, long long n, float* dist2,
                                                      int32_t* idx, float* max_cert) {
  extern __shared__ __align__(16) float smem[];
  uint32_t* s_delta = reinterpret_cast<uint32_t*>(smem);
  fill_probe_deltas(m, s_delta);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long wpb = blockDim.x >> 5;
  const int C = m.n_probe;
  for (long long qi = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); qi < n; qi += (long long)gridDim.x * wpb) {
    const float qx = __ldg(query_xyz + 3 * qi), qy = __ldg(query_xyz + 3 * qi + 1), qz = __ldg(query_xyz + 3 * qi + 2);
    const uint32_t r0 = base_slot(m, qx, qy, qz);
    const float td_cur = m.time_filter ? __ldg(m.travel_dist + m.cur_ts) : 0.f;
    float best = 0.f;
    for (int c = lane; c < C; c += 32) {
      float d2;
      int li, gi;
      probe_cell(m, r0, s_delta[c], qx, qy, qz, td_cur, d2, li, gi);
      if (dist2) dist2[qi * C + c] = d2;
      if (idx) idx[qi * C + c] = gi;
      if (max_cert && gi >= 0) best = fmaxf(best, m.certainty[gi]);  // query_certainty (:1025-1028)
    }
    if (max_cert) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(FULL, best, o));
      if (lane == 0) max_cert[qi] = best;
    }
  }
}

// query_feature's materialised feature vectors from saved kNN (compat path)
__global__ void __launch_bounds__(256) gather_kernel(const __grid_constant__ pinb200_map_view m,
                                                      const float* __restrict__ feat,
                                                      const float* __restrict__ query_xyz,
                                                      const int32_t* __restrict__ knn_idx,
                                                      const float* __restrict__ knn_w, long long n, int K, int wf,
                                                      float* out) {
  const int F = m.feature_dim, D = F + 3;
  const long long total = wf ? n * D : n * K * D;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(e % D);
    const long long r = e / D;
    const long long qi = wf ? r : r / K;
    float acc = 0.f;
    const int k_lo = wf ? 0 : (int)(r % K), k_hi = wf ? K : k_lo + 1;
    for (int k = k_lo; k < k_hi; ++k) {
      const int lk = knn_idx[qi * K + k];
      if (lk < 0) continue;
      float v;
      if (d < F) {
        v = __ldg(feat + (size_t)lk * F + d);
      } else {
        float nx = query_xyz[3 * qi] - m.nb_points[3 * (size_t)lk];
        float ny = query_xyz[3 * qi + 1] - m.nb_points[3 * (size_t)lk + 1];
        float nz = query_xyz[3 * qi + 2] - m.nb_points[3 * (size_t)lk + 2];
        if (m.after_pgo) {
          const float* qq = m.nb_orient + 4 * (size_t)lk;
          quat_rotate_passive(qq[0], qq[1], qq[2], qq[3], nx, ny, nz, nx, ny, nz);
        }
        v = d == F ? nx : (d == F + 1 ? ny : nz);
      }
      acc = wf ? fmaf(knn_w[qi * K + k], v, acc) : v;
    }
    out[e] = acc;
  }
}

// run-time tunables (pinb200_set_option)
static long long g_split_min_queries = PINB200_SPLIT_MIN_QUERIES;        // decode-every-neighbour maps (mma.sync decode)
static long long g_split_min_queries_wf = PINB200_SPLIT_MIN_QUERIES_WF;  // weighted_first maps (tensor-core decode)
static long long g_sort_min_queries = PINB200_SORT_MIN_QUERIES;  // spatial sort before the search launch; 0: never
static long long g_sort_min_queries_color = 0;                    // the same for calls with a colour head

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
static int validate_map(const pinb200_map_view* m, bool need_feat) {
  if (!m || !m->slot_table || !m->points || !m->probe_dx || m->n_probe <= 0) {
    set_error("map view: null table/points/probe offsets");
    return PINB200_ERR_BAD_ARG;
  }
  if (m->buffer_size <= 0 || m->buffer_size >= (1LL << 31)) {
    set_error("map view: buffer_size %lld out of range (0, 2^31)", (long long)m->buffer_size);
    return PINB200_ERR_BAD_ARG;
  }
  if (m->time_filter && (!m->ts_create || !m->travel_dist)) {
    set_error("map view: time_filter needs ts_create and travel_dist");
    return PINB200_ERR_BAD_ARG;
  }
  if (need_feat) {
    if (!m->nb_points || !m->geo_feat || !m->certainty) {
      set_error("map view: null neighbour arrays");
      return PINB200_ERR_BAD_ARG;
    }
    const int F = m->feature_dim;
    const bool okF = F == 4 || F == 8 || F == 16 || F == 32 || F == 64;
    if (!okF) {
      set_error("feature_dim %d unsupported (4, 8, 16, 32, 64)", F);
      return PINB200_ERR_UNSUPPORTED;
    }
    if (m->after_pgo && !m->nb_orient) {
      set_error("map view: after_pgo needs nb_orient");
      return PINB200_ERR_BAD_ARG;
    }
    if (m->n_nb >= PINB200_REC_REMAP) {
      set_error("map view: n_nb %lld >= 2^30 (the id word of a probe record keeps bit 30 as a flag)", (long long)m->n_nb);
      return PINB200_ERR_UNSUPPORTED;
    }
  }
  return PINB200_OK;
}

template <int FT>
static QueryLayout plan_layout(const QueryParams& p) {
  QueryLayout l{};
  int o = 0;
  l.delta = o;
  o += align4(p.map.n_probe);
  l.dec = plan_warp_decoder_smem(p.dec, WarpLay<FT>::KP0, o, ld8mod32);
  l.warp0 = align4(l.dec.end);
  int nw = (227 * 1024 / 4 - l.warp0) / WarpLay<FT>::stride;
  l.n_warps = nw > WPB ? WPB : nw;
  l.total = l.warp0 + l.n_warps * WarpLay<FT>::stride;
  return l;
}

template <int FT, bool WF, bool SPLIT>
static int launch_query(QueryParams& p, cudaStream_t stream) {
  p.lay = plan_layout<FT>(p);
  const size_t smem_bytes = (size_t)p.lay.total * sizeof(float);
  if (p.lay.n_warps < 1 || smem_bytes > 227 * 1024) {
    set_error("query kernel needs %zu B shared memory (> 227 KB)", smem_bytes);
    return PINB200_ERR_UNSUPPORTED;
  }
  // small batches (tracker: a few thousand points, mapper: ~26k rows): spread the warp tiles over all SMs
  // instead of packing 10-12 warps into a few CTAs
  int nw = p.lay.n_warps;
  {
    // queries per warp tile: a full 32 when there is enough work to occupy every resident warp, fewer (whole
    // decoder row tiles in decode-every-neighbour mode) for the tracker / mapper sized launches
    const long long slots = (long long)sm_count() * nw;
    const long long per_warp = (p.n + slots - 1) / slots;
    int wq;
    if (SPLIT) {
      wq = WT;  // the stash is written per 32-query tile
    } else if (WF) {
      constexpr int G = RowMap<FT>::U * RowMap<FT>::RPP;  // queries per gather pass
      wq = (int)std::min<long long>(WT, std::max<long long>(G, (per_warp + G - 1) / G * G));
    } else {
      const int qpt_rows = WT / p.opts.nn_k;
      wq = (int)std::min<long long>(WT, (per_warp + qpt_rows - 1) / qpt_rows * qpt_rows);
    }
    p.qpt = wq;
    p.n_tiles = (int)((p.n + wq - 1) / wq);
    const long long per_sm = (p.n_tiles + sm_count() - 1) / sm_count();
    if (per_sm < nw) nw = (int)std::max<long long>(1, per_sm);
  }
  auto kern = query_kernel<FT, WF, SPLIT>;
  if (const int rc = prepare_kernel((const void*)kern, "query_kernel", smem_bytes)) return rc;
  const long long ctas_needed = (p.n_tiles + nw - 1) / nw;
  const int grid = (int)std::min<long long>(ctas_needed, (long long)sm_count());  // one CTA per SM (launch bounds)
  kern<<<grid, nw * 32, smem_bytes, stream>>>(p);
  return check_launch("query_kernel");
}

template <bool WF, bool SPLIT>
static int dispatch_query_wf(QueryParams& p, cudaStream_t stream) {
  switch (p.dec.in_dim - 3) {
    case 4: return launch_query<4, WF, SPLIT>(p, stream);
    case 8: return launch_query<8, WF, SPLIT>(p, stream);
    case 16: return launch_query<16, WF, SPLIT>(p, stream);
    case 32: return launch_query<32, WF, SPLIT>(p, stream);
    case 64: return launch_query<64, WF, SPLIT>(p, stream);
    default: break;
  }
  set_error("feature_dim %d unsupported (4, 8, 16, 32, 64)", p.dec.in_dim - 3);
  return PINB200_ERR_UNSUPPORTED;
}

static int dispatch_query(QueryParams& p, cudaStream_t stream, bool split) {
  if (p.dec.hidden_dim != 64) {
    set_error("decoder hidden_dim %d unsupported (64)", p.dec.hidden_dim);
    return PINB200_ERR_UNSUPPORTED;
  }
  if (split)
    return p.opts.weighted_first ? dispatch_query_wf<true, true>(p, stream) : dispatch_query_wf<false, true>(p, stream);
  return p.opts.weighted_first ? dispatch_query_wf<true, false>(p, stream) : dispatch_query_wf<false, false>(p, stream);
}

// K1a launch of the split pipeline; `compact`: write StashS blocks.  Only wsq_decode_kernel reads the forward-mode
// seeds, and it reads compact blocks, so p.seeds is set only with `compact`.
static int launch_search(QueryParams& p, bool compact, cudaStream_t stream) {
  p.qpt = WT;
  p.n_tiles = (int)((p.n + WT - 1) / WT);
  const long long ctas = (p.n_tiles + 3) / 4;
  const int grid = (int)std::min<long long>(ctas, (long long)sm_count() * 4);
  const size_t smem = align4(p.map.n_probe) * sizeof(float);
  if (!compact)
    search_kernel<false, false><<<grid, 128, smem, stream>>>(p);
  else if (p.seeds)
    search_kernel<true, true><<<grid, 128, smem, stream>>>(p);
  else
    search_kernel<false, true><<<grid, 128, smem, stream>>>(p);
  return check_launch("search_kernel");
}

static int validate_decoder(const pinb200_decoder_view* d, int F) {
  if (!d || !d->w_out || d->n_hidden < 1 || d->n_hidden > PINB200_MAX_HIDDEN_LAYERS) {
    set_error("decoder view: bad n_hidden / null w_out");
    return PINB200_ERR_BAD_ARG;
  }
  for (int l = 0; l < d->n_hidden; ++l)
    if (!d->w[l]) {
      set_error("decoder view: null weight of layer %d", l);
      return PINB200_ERR_BAD_ARG;
    }
  if (d->in_dim != F + 3) {
    set_error("decoder in_dim %d != feature_dim+3 = %d (positional encoding is not supported)", d->in_dim, F + 3);
    return PINB200_ERR_UNSUPPORTED;
  }
  if (d->out_dim < 1 || d->out_dim > 4) {
    set_error("decoder out_dim %d unsupported (1..4)", d->out_dim);
    return PINB200_ERR_UNSUPPORTED;
  }
  return PINB200_OK;
}

}  // namespace pinb

using namespace pinb;

extern "C" int pinb200_query_sdf(const pinb200_map_view* map, const pinb200_decoder_view* sdf_dec,
                                 const pinb200_decoder_view* color_dec, const float* query_xyz,
                                 const int32_t* query_ts, int64_t n, const pinb200_query_opts* opts,
                                 const pinb200_query_out* out, void* stream) {
  int rc = validate_map(map, true);
  if (rc) return rc;
  if (!opts || !out || (!query_xyz && n > 0)) {
    set_error("query_sdf: null opts/out/query");
    return PINB200_ERR_BAD_ARG;
  }
  rc = validate_decoder(sdf_dec, map->feature_dim);
  if (rc) return rc;
  if (!map->probe_words || !map->probe_rec || !map->probe_gid) {
    set_error("query_sdf: the map view has no probe index (pinb200_build_probe_index fills probe_words/rec/gid)");
    return PINB200_ERR_BAD_ARG;
  }
  const int K = opts->nn_k;
  if (K < 1 || K > KREG || K > map->n_probe) {
    set_error("nn_k %d out of range (1..%d, <= n_probe %d)", K, KREG, map->n_probe);
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  if (color_dec) {
    rc = validate_decoder(color_dec, map->feature_dim);
    if (rc) return rc;
    if (!map->color_feat || !out->knn_idx || !out->knn_gidx || !out->knn_dist2 || !out->nn_count) {
      set_error("colour head needs map->color_feat and out->knn_idx/knn_gidx/knn_dist2/nn_count as scratch");
      return PINB200_ERR_BAD_ARG;
    }
  }
  QueryParams p{};
  p.map = *map;
  p.dec = *sdf_dec;
  p.opts = *opts;
  p.out = *out;
  p.query_xyz = query_xyz;
  p.query_ts = query_ts;
  p.feat = map->geo_feat;
  p.n = n;
  p.qpt = WT;  // queries per warp tile
  p.n_tiles = (int)((n + WT - 1) / WT);
  // Large batches run as two launches (search at high occupancy, then decode) through the caller's workspace; small
  // ones (tracker / mapper sized, latency-bound) stay fused in one launch.
  const int64_t need = pinb200_query_workspace_bytes(n);
  // weighted_first maps with a wgmma-decodable configuration: the two-launch pipeline wins from ~1 k queries on
  // (8 k queries, F = 32: 48 us vs 72 us for the fused launch; scripts/exp_small_n.py)
  // (training-mode batches of the mapper are value-only and tile poorly at 16-26 k rows: they keep the general threshold)
  const long long split_min = (wsq_supported(*sdf_dec, *opts) && !opts->training_mode) ? g_split_min_queries_wf : g_split_min_queries;
  const bool split = opts->workspace && opts->workspace_bytes >= need && n >= split_min;
  // Split calls whose decodes all run on wsq_decode_kernel write compact stash blocks (StashS) and, with d/dq, the
  // forward-mode seeds after them; every decode of any other split call runs on query_kernel from full Stash blocks.
  const bool compact = split && wsq_supported(*sdf_dec, *opts) && (!color_dec || wsq_supported(*color_dec, *opts));
  if (split) {
    p.stash = reinterpret_cast<float*>(opts->workspace);
    const bool want_seeds = compact && opts->need_grad;
    // Large inference batches with compact stash blocks are searched in Morton order of their cells (2x the map
    // resolution): the lanes of a tile then probe the same or neighbouring cells.  The compact blocks leave room in
    // the workspace for the sort (query_sort.cu); if it does not fit, the batch runs unsorted.  Calls with a colour
    // head have their own threshold, off by default: the large one (the dense RGB-D query) comes in pixel order,
    // already coherent, and sorting it only adds the sort (0.420 -> 0.487 ms at 307 k pixels, H100 at 400 W).
    const long long sort_min = color_dec ? g_sort_min_queries_color : g_sort_min_queries;
    if (compact && !opts->training_mode && sort_min > 0 && n >= sort_min) {
      char* base = static_cast<char*>(opts->workspace);
      const size_t used = (size_t)p.n_tiles * (StashS::floats + (want_seeds ? Seeds::floats : 0)) * sizeof(float);
      rc = sort_queries(query_xyz, opts->transform, n, map->resolution, base + used,
                        (size_t)opts->workspace_bytes - used, &p.perm, (cudaStream_t)stream);
      if (rc) return rc;
    }
    p.seeds = want_seeds ? p.stash + (size_t)p.n_tiles * StashS::floats : nullptr;
    rc = launch_search(p, compact, (cudaStream_t)stream);
    if (rc) return rc;
  }
  // decode: wgmma tiles of 128 queries where every decoder of the call allows it, else the warp-level mma.sync kernel
  p.pdl = split ? 1 : 0;  // only the launch that directly follows the search launch
  auto decode = [&](QueryParams& qp) {
    return compact ? dispatch_wsq(qp, (cudaStream_t)stream) : dispatch_query(qp, (cudaStream_t)stream, split);
  };
  rc = decode(p);
  if (rc) return rc;
  if (color_dec) {  // second launch: decode the colour features with the kNN the first launch saved
    QueryParams c = p;
    c.pdl = 0;
    c.dec = *color_dec;
    c.feat = map->color_feat;
    c.use_saved_knn = split ? 0 : 1;  // the split pipeline re-uses the stash instead
    c.is_color = 1;
    c.opts.training_mode = 0;
    c.opts.need_grad = (opts->need_grad && out->color_grad) ? 1 : 0;
    rc = decode(c);
  }
  return rc;
}

extern "C" int pinb200_debug_read(const char* what, void* host_out, int64_t count) {
  if (what && std::string(what) == "ws_profile") return wsq_read_profile(reinterpret_cast<unsigned long long*>(host_out), count);
  set_error("debug_read: unknown item '%s'", what ? what : "(null)");
  return PINB200_ERR_BAD_ARG;
}

extern "C" int pinb200_set_option(const char* name, int64_t value) {
  if (!name) {
    set_error("set_option: null name");
    return PINB200_ERR_BAD_ARG;
  }
  const std::string key(name);
  if (key == "split_min_queries") {  // both thresholds; <= 0 restores the defaults
    g_split_min_queries = value > 0 ? value : PINB200_SPLIT_MIN_QUERIES;
    g_split_min_queries_wf = value > 0 ? value : PINB200_SPLIT_MIN_QUERIES_WF;
  } else if (key == "split_min_queries_wf") {
    g_split_min_queries_wf = value > 0 ? value : PINB200_SPLIT_MIN_QUERIES_WF;
  } else if (key == "sort_min_queries") {  // batches of at least this many queries are sorted; 0: never
    if (value < 0) {
      set_error("set_option: sort_min_queries %lld < 0", (long long)value);
      return PINB200_ERR_BAD_ARG;
    }
    g_sort_min_queries = value;
  } else if (key == "sort_min_queries_color") {  // the same for calls with a colour head; 0 (default): never
    if (value < 0) {
      set_error("set_option: sort_min_queries_color %lld < 0", (long long)value);
      return PINB200_ERR_BAD_ARG;
    }
    g_sort_min_queries_color = value;
  } else if (key == "ws_profile") {
    wsq_set_profile(value != 0);
  } else {
    set_error("set_option: unknown option '%s'", name);
    return PINB200_ERR_BAD_ARG;
  }
  return PINB200_OK;
}

extern "C" int64_t pinb200_query_workspace_bytes(int64_t n) {
  return n <= 0 ? 0 : ((n + WT - 1) / WT) * (int64_t)(Stash::floats + Seeds::floats) * (int64_t)sizeof(float);
}

extern "C" int pinb200_knn_search(const pinb200_map_view* map, const float* query_xyz, int64_t n, int32_t nn_k,
                                  int32_t* knn_idx, int32_t* knn_gidx, float* knn_dist2, float* knn_weight,
                                  int32_t* nn_count, void* stream) {
  int rc = validate_map(map, false);
  if (rc) return rc;
  if (nn_k < 1 || nn_k > PINB200_MAX_K || nn_k > map->n_probe) {
    set_error("nn_k %d out of range", nn_k);
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  const int grid = (int)std::min<long long>((n + 3) / 4, (long long)sm_count() * 8);
  knn_kernel<<<grid, TILE, align4(map->n_probe) * sizeof(float), (cudaStream_t)stream>>>(
      *map, query_xyz, n, nn_k, knn_idx, knn_gidx, knn_dist2, knn_weight, nn_count);
  return check_launch("knn_kernel");
}

extern "C" int pinb200_radius_search(const pinb200_map_view* map, const float* query_xyz, int64_t n, float* dist2,
                                     int32_t* idx, void* stream) {
  int rc = validate_map(map, false);
  if (rc) return rc;
  if (n <= 0) return PINB200_OK;
  const int grid = (int)std::min<long long>((n + 3) / 4, (long long)sm_count() * 8);
  radius_kernel<<<grid, TILE, align4(map->n_probe) * sizeof(float), (cudaStream_t)stream>>>(*map, query_xyz, n, dist2,
                                                                                            idx, nullptr);
  return check_launch("radius_kernel");
}

extern "C" int pinb200_query_certainty(const pinb200_map_view* map, const float* query_xyz, int64_t n,
                                       float* out_certainty, void* stream) {
  int rc = validate_map(map, false);
  if (rc) return rc;
  if (map->global2local || map->time_filter || !map->certainty) {
    set_error("query_certainty works on the global arrays: global2local must be NULL, time_filter 0");
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  const int grid = (int)std::min<long long>((n + 3) / 4, (long long)sm_count() * 8);
  radius_kernel<<<grid, TILE, align4(map->n_probe) * sizeof(float), (cudaStream_t)stream>>>(*map, query_xyz, n, nullptr,
                                                                                            nullptr, out_certainty);
  return check_launch("radius_kernel(certainty)");
}

extern "C" int pinb200_gather_features(const pinb200_map_view* map, const float* feat, const float* query_xyz,
                                       const int32_t* knn_idx, const float* knn_weight, int64_t n, int32_t nn_k,
                                       int32_t weighted_first, float* out, void* stream) {
  if (!map || !feat || !knn_idx || !knn_weight || !out || !map->nb_points) {
    set_error("gather_features: null argument");
    return PINB200_ERR_BAD_ARG;
  }
  if (n <= 0) return PINB200_OK;
  const long long total = (weighted_first ? n : n * nn_k) * (map->feature_dim + 3);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*map, feat, query_xyz, knn_idx, knn_weight, n, nn_k,
                                                        weighted_first, out);
  return check_launch("gather_kernel");
}
