// K1b on the Hopper warpgroup tensor cores: the phase-synchronous decode launch of the split pipeline for
// weighted_first maps (decode_variant 0; wsq.cu is the warp-specialised default).
//
// One CTA of 512 threads per SM works on tiles of 128 queries (warp w = row quadrant rq = w & 3, column block
// cb = w >> 2; thread <-> row 32 rq + lane of the tile; warp w owns the stash blocks of queries 32 rq .. 32 rq + 31).
// The decoder is a chain of [128 x K] x [K x 64] contractions: every layer is issued by the four warpgroups as
// wgmma.mma_async (kind tf32, M = 64, twice per tile) reading both operands from shared memory in the no-swizzle
// canonical K-major layout (8-row x 16-byte core matrices); warpgroup cb computes the 16 accumulator columns of its
// column block, so a thread's row/column block is produced inside its own warpgroup.  The 3xTF32 split
// (a_hi b_hi + a_lo b_hi + a_hi b_lo, see mlp_mma.cuh) becomes three MMAs per 8-wide k-step.  The accumulator
// fragments are handed to the row owners through the consumed A tile; the epilogue then applies bias / ReLU / mask in
// registers -> hi/lo split -> the next layer's A operand, written straight into the canonical layout with 16-byte
// stores.  The backward pass to the decoder input uses transposed copies of the weights staged once per CTA (tf32
// wgmma operands must be K-major).
#pragma once

#include "umma_common.cuh"

namespace pinb {

struct UmmaLayout {  // byte offsets from the 1024-byte aligned dynamic shared memory base
  int w0f_hi, w0f_lo, w1f_hi, w1f_lo;  // forward copies  W_l [64][K_l]   (B operand of h = x W^T)
  int w1b_hi, w1b_lo, w0b_hi, w0b_lo;  // backward copies W_l^T [K_l][64] (B operand of g_in = g_out W)
  int a_hi, a_lo;                      // A operand tiles [128][<=64] (the input-gradient tile for C1/C2 aliases a_hi)
  int b0, b1, wout, bout;              // fp32 vectors
  int warp0, warp_stride;              // per row-quadrant blocks: Stash | a[8][32]
  int part;                            // [4][4][128] partial output-head sums per column block
  int total;
};

// The CTA: 16 warps on ONE 128-row tile at a time.  Warp w = (row quadrant rq = w & 3, column block cb = w >> 2): the
// four warps of a quadrant split the 64 accumulator columns 16 each; the gather phases (A2 / C1) give every warp 8 of
// the 128 queries.  Four resident warps per scheduler hide the ALU / shared-memory / L2 latencies.
constexpr int UM_THREADS = 512;
constexpr int UM_CB = 4;        // column blocks (= warpgroups)
constexpr int UM_CW = 16;       // columns per block

// D[128 x 16] = A[128 x 8 ksteps] B^T (3xTF32) for the columns 16 cb .. 16 cb + 15 (rows of B) that warpgroup cb owns,
// skipped where 16 cb >= N.  The fragments pass through `xch` (the consumed a_lo tile) so that thread `row` of the
// warpgroup receives its row's 16 columns in v.  Starts after um_publish_and_sync(); ends with a block barrier, after
// which the A tiles may be rewritten.
__device__ __forceinline__ void um_gemm_rows(uint32_t a_hi, uint32_t a_lo, uint32_t a_sbo, uint32_t b_hi, uint32_t b_lo,
                                             uint32_t b_sbo, int ksteps, int N, int cb, float* xch, int row,
                                             uint32_t (&v)[UM_CW]) {
  const bool active = cb * UM_CW < N;
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  float acc[2][8];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[h][e] = 0.f;
  if (active) {
    const uint32_t bh = b_hi + 2 * cb * b_sbo, bl = b_lo + 2 * cb * b_sbo;  // two 8-row groups of B per column block
    wg_fence();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t ah = a_hi + h * 8 * a_sbo, al = a_lo + h * 8 * a_sbo;
      for (int s = 0; s < ksteps; ++s) {
        const uint64_t dah = um_desc(ah + s * 2 * UM_A_LBO, UM_A_LBO, a_sbo), dal = um_desc(al + s * 2 * UM_A_LBO, UM_A_LBO, a_sbo);
        const uint64_t dbh = um_desc(bh + s * 2 * UM_W_LBO, UM_W_LBO, b_sbo), dbl = um_desc(bl + s * 2 * UM_W_LBO, UM_W_LBO, b_sbo);
        wg_mma_n16(acc[h], dal, dbh, s > 0);  // small terms first
        wg_mma_n16(acc[h], dah, dbl, 1);
        wg_mma_n16(acc[h], dah, dbh, 1);
      }
    }
    wg_commit();
    wg_wait0();
  }
  __syncthreads();  // every warpgroup's MMAs have read the A tiles: a_lo becomes the exchange buffer
  float* x = xch + cb * (UM_ROWS * UM_CW);
  if (active) {
    const int g = lane >> 2, c = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int r0 = 64 * h + 16 * wq + g;
        *reinterpret_cast<float2*>(x + r0 * UM_CW + 8 * j + 2 * c) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
        *reinterpret_cast<float2*>(x + (r0 + 8) * UM_CW + 8 * j + 2 * c) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
      }
  }
  asm volatile("bar.sync %0, 128;" ::"r"(1 + cb) : "memory");  // the warpgroup's exchange block is complete
#pragma unroll
  for (int e4 = 0; e4 < UM_CW / 4; ++e4) {
    const float4 t = active ? *reinterpret_cast<const float4*>(x + row * UM_CW + 4 * e4) : make_float4(0.f, 0.f, 0.f, 0.f);
    v[4 * e4] = __float_as_uint(t.x);
    v[4 * e4 + 1] = __float_as_uint(t.y);
    v[4 * e4 + 2] = __float_as_uint(t.z);
    v[4 * e4 + 3] = __float_as_uint(t.w);
  }
  __syncthreads();  // the exchange buffer is read before the A tiles are rewritten
}

template <int FT>
__global__ void __launch_bounds__(UM_THREADS, 1) decode_umma_kernel(const __grid_constant__ QueryParams p, const UmmaLayout lay) {
  constexpr int H = 64;
  using DM = UmmaDims<FT>;
  constexpr int K0 = DM::K0, N0 = DM::N0, GLD = DM::GLD, F = FT, D = FT + 3;
  using M = RowMap<FT>;
  constexpr int QPW = UM_ROWS / (UM_THREADS / 32);  // queries gathered per warp (8)
  constexpr int GU = QPW / M::RPP > 0 ? QPW / M::RPP : 1;  // gather passes per warp
  constexpr bool NARROW = M::RPP > QPW;  // F < 16: a pass covers more queries than the warp owns, the upper lanes idle
  extern __shared__ __align__(1024) unsigned char um_smem[];
  unsigned char* sm = um_smem;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rq = warp & 3, cb = warp >> 2;
  const int row = rq * WT + lane;  // row of the 128-row tile
  const pinb200_map_view& m = p.map;
  const int K = p.opts.nn_k, L = p.dec.n_hidden, OC = p.dec.out_dim;
  const bool need_grad = p.opts.need_grad != 0, leaky = p.dec.leaky_relu != 0;
  const float* __restrict__ feat = p.feat;

  float* qsm = reinterpret_cast<float*>(sm + lay.warp0 + rq * lay.warp_stride);  // the quadrant's stash + a[8][32]
  const int* s_li = reinterpret_cast<const int*>(qsm + Stash::li);
  const float* s_w = qsm + Stash::w;
  const float* s_dx = qsm + Stash::dx;
  const float* s_dy = qsm + Stash::dy;
  const float* s_dz = qsm + Stash::dz;
  const float* s_q = qsm + Stash::q;
  const float* s_usum = qsm + Stash::usum;
  const int* s_nn = reinterpret_cast<const int*>(qsm + Stash::nn);
  const float* s_pos = qsm + Stash::pos;
  float* s_a = qsm + Stash::floats;  // [8][32]
  const float* s_b0 = reinterpret_cast<const float*>(sm + lay.b0);
  const float* s_b1 = reinterpret_cast<const float*>(sm + lay.b1);
  const float* s_wout = reinterpret_cast<const float*>(sm + lay.wout);
  const float* s_bout = reinterpret_cast<const float*>(sm + lay.bout);
  float* s_part = reinterpret_cast<float*>(sm + lay.part);  // [4 channels][UM_CB][128] partial output-head sums
  unsigned char* a_hi = sm + lay.a_hi;
  unsigned char* a_lo = sm + lay.a_lo;
  float* s_g = reinterpret_cast<float*>(sm + lay.a_hi);  // row-major [128][GLD] input gradient (aliases the A tile)
  float* xch = reinterpret_cast<float*>(sm + lay.a_lo);  // accumulator exchange (see um_gemm_rows)

  // ---- one-off: weights
  um_stage_weight(p.dec.w[0], D, H, D, H, K0, false, sm + lay.w0f_hi, sm + lay.w0f_lo);
  if (need_grad) um_stage_weight(p.dec.w[0], D, D, H, N0, H, true, sm + lay.w0b_hi, sm + lay.w0b_lo);
  if (L > 1) {
    um_stage_weight(p.dec.w[1], H, H, H, H, H, false, sm + lay.w1f_hi, sm + lay.w1f_lo);
    if (need_grad) um_stage_weight(p.dec.w[1], H, H, H, H, H, true, sm + lay.w1b_hi, sm + lay.w1b_lo);
  }
  for (int e = tid; e < H; e += UM_THREADS) {
    reinterpret_cast<float*>(sm + lay.b0)[e] = p.dec.b[0] ? __ldg(p.dec.b[0] + e) : 0.f;
    reinterpret_cast<float*>(sm + lay.b1)[e] = (L > 1 && p.dec.b[1]) ? __ldg(p.dec.b[1] + e) : 0.f;
  }
  for (int e = tid; e < OC * H; e += UM_THREADS) reinterpret_cast<float*>(sm + lay.wout)[e] = __ldg(p.dec.w_out + e);
  if (tid < 4) reinterpret_cast<float*>(sm + lay.bout)[tid] = (p.dec.b_out && tid < OC) ? __ldg(p.dec.b_out + tid) : 0.f;
  um_publish_and_sync();

  const uint32_t a_hi_u = um_smem_u32(a_hi), a_lo_u = um_smem_u32(a_lo);
  const uint32_t w0f_hi = um_smem_u32(sm + lay.w0f_hi), w0f_lo = um_smem_u32(sm + lay.w0f_lo);
  const uint32_t w1f_hi = um_smem_u32(sm + lay.w1f_hi), w1f_lo = um_smem_u32(sm + lay.w1f_lo);
  const uint32_t w1b_hi = um_smem_u32(sm + lay.w1b_hi), w1b_lo = um_smem_u32(sm + lay.w1b_lo);
  const uint32_t w0b_hi = um_smem_u32(sm + lay.w0b_hi), w0b_lo = um_smem_u32(sm + lay.w0b_lo);
  constexpr uint32_t A_SBO0 = (K0 / 4) * UM_A_LBO, A_SBO1 = (H / 4) * UM_A_LBO;
  constexpr uint32_t W_SBO0 = (K0 / 4) * UM_W_LBO, W_SBO1 = (H / 4) * UM_W_LBO;
  const int n_tiles32 = p.n_tiles;  // 32-query stash tiles
  const int n_tiles128 = (n_tiles32 + 3) / 4;
  // gather mapping of this warp: queries qb .. qb + QPW - 1 of its quadrant, F/4 lanes per feature row
  const int sub = lane / M::LPR, c4 = lane % M::LPR;
  const int qb = cb * QPW;
  const float4* __restrict__ f4 = reinterpret_cast<const float4*>(feat) + c4;

  for (int T = blockIdx.x; T < n_tiles128; T += gridDim.x) {
    const int st = 4 * T + rq;  // the quadrant's stash tile
    const bool qlive = st < n_tiles32;
    const long long qi = (long long)st * WT + lane;  // this thread's query (threads of the four column blocks share it)
    const bool live = qlive && qi < p.n;

    // ---- stash block of the quadrant's 32 queries (written by search_kernel): 4 warps x 3 coalesced 16-byte copies
    __syncthreads();  // every reader of the previous tile's stash / gradient tile is done
    {
      float4* dst = reinterpret_cast<float4*>(qsm);
      constexpr int PER = Stash::floats / 4 / (UM_CB * 32);  // float4 per thread (3)
      if (qlive) {
        const float4* __restrict__ src = reinterpret_cast<const float4*>(p.stash + (size_t)st * Stash::floats);
        float4 t[PER];
#pragma unroll
        for (int i = 0; i < PER; ++i) t[i] = __ldg(src + (i * UM_CB + cb) * 32 + lane);
#pragma unroll
        for (int i = 0; i < PER; ++i) dst[(i * UM_CB + cb) * 32 + lane] = t[i];
      } else {  // tail tile: no neighbours (ids -1, everything else 0)
#pragma unroll
        for (int i = 0; i < PER; ++i) {
          const int e4 = (i * UM_CB + cb) * 32 + lane;
          dst[e4] = e4 * 4 < Stash::w ? make_float4(__int_as_float(-1), __int_as_float(-1), __int_as_float(-1), __int_as_float(-1))
                                      : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
    __syncthreads();  // stash visible to the quadrant's four warps

    // ============ A2: F/4 lanes per row -- IDW-weighted feature rows -> A tile (hi / lo) ============
    {
      float4 fv[GU][KREG];
#pragma unroll
      for (int u = 0; u < GU; ++u) {
        const int ql = qb + u * M::RPP + sub;
#pragma unroll
        for (int k = 0; k < KREG; ++k) {
          fv[u][k] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (k < K && (!NARROW || sub < QPW)) {
            const int lif = s_li[k * WT + ql];
            if (lif >= 0) fv[u][k] = __ldg(f4 + (size_t)(lif & ~REMAP) * M::LPR);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < GU; ++u) {
        const int ql = qb + u * M::RPP + sub;
        if (NARROW && sub >= QPW) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < KREG; ++k)
          if (k < K) {
            const float w = s_w[k * WT + ql];
            acc.x = fmaf(w, fv[u][k].x, acc.x);
            acc.y = fmaf(w, fv[u][k].y, acc.y);
            acc.z = fmaf(w, fv[u][k].z, acc.z);
            acc.w = fmaf(w, fv[u][k].w, acc.w);
          }
        float4 hi, lo;
        um_split4(acc, hi, lo);
        const int off = um_a_off(rq * WT + ql, c4, K0);
        *reinterpret_cast<float4*>(a_hi + off) = hi;
        *reinterpret_cast<float4*>(a_lo + off) = lo;
      }
      // position part + zero padding of the rows: columns F .. K0-1 (two 16-byte chunks), column blocks 0 and 1
      if (cb < (K0 - F) / 4) {
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (cb == 0) t = make_float4(s_pos[lane], s_pos[WT + lane], s_pos[2 * WT + lane], 0.f);
        float4 hi, lo;
        um_split4(t, hi, lo);
        const int off = um_a_off(row, F / 4 + cb, K0);
        *reinterpret_cast<float4*>(a_hi + off) = hi;
        *reinterpret_cast<float4*>(a_lo + off) = lo;
      }
    }

    // ============ B: decoder forward on wgmma ============
    uint32_t v[UM_CW];
    uint32_t mk0 = 0u, mkL = 0u;  // ReLU masks (this thread's 16 columns) of layer 0 and of the last hidden layer
    um_publish_and_sync();
    um_gemm_rows(a_hi_u, a_lo_u, A_SBO0, w0f_hi, w0f_lo, W_SBO0, K0 / 8, H, cb, xch, row, v);
    if (L > 1) {
      // layer-0 epilogue: bias, ReLU (mask kept), split, next A operand
#pragma unroll
      for (int c = 0; c < UM_CW / 4; ++c) {
        const float4 b = *reinterpret_cast<const float4*>(s_b0 + cb * UM_CW + 4 * c);
        float z[4] = {__uint_as_float(v[4 * c]) + b.x, __uint_as_float(v[4 * c + 1]) + b.y, __uint_as_float(v[4 * c + 2]) + b.z,
                      __uint_as_float(v[4 * c + 3]) + b.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (z[e] > 0.f)
            mk0 |= 1u << (4 * c + e);
          else
            z[e] = leaky ? 0.01f * z[e] : 0.f;
        }
        float4 hi, lo;
        um_split4(make_float4(z[0], z[1], z[2], z[3]), hi, lo);
        const int off = um_a_off(row, cb * (UM_CW / 4) + c, H);
        *reinterpret_cast<float4*>(a_hi + off) = hi;
        *reinterpret_cast<float4*>(a_lo + off) = lo;
      }
      um_publish_and_sync();
      um_gemm_rows(a_hi_u, a_lo_u, A_SBO1, w1f_hi, w1f_lo, W_SBO1, H / 8, H, cb, xch, row, v);
    }
    // last hidden layer: bias, ReLU (mask kept), this column block's part of the output head(s)
    {
      const float* bl = L > 1 ? s_b1 : s_b0;
      float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < UM_CW / 4; ++c) {
        const float4 b = *reinterpret_cast<const float4*>(bl + cb * UM_CW + 4 * c);
        float z[4] = {__uint_as_float(v[4 * c]) + b.x, __uint_as_float(v[4 * c + 1]) + b.y, __uint_as_float(v[4 * c + 2]) + b.z,
                      __uint_as_float(v[4 * c + 3]) + b.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (z[e] > 0.f)
            mkL |= 1u << (4 * c + e);
          else
            z[e] = leaky ? 0.01f * z[e] : 0.f;
        }
#pragma unroll
        for (int ch = 0; ch < 4; ++ch)
          if (ch < OC) {
            const float4 wo = *reinterpret_cast<const float4*>(s_wout + ch * H + cb * UM_CW + 4 * c);
            o[ch] = fmaf(z[3], wo.w, fmaf(z[2], wo.z, fmaf(z[1], wo.y, fmaf(z[0], wo.x, o[ch]))));
          }
      }
#pragma unroll
      for (int ch = 0; ch < 4; ++ch)
        if (ch < OC) s_part[(ch * UM_CB + cb) * UM_ROWS + row] = o[ch];
    }

    // ======== per output channel: backward to the decoder input, then the IDW chain rule ========
    float val[4] = {0.f, 0.f, 0.f, 0.f}, dvv[4] = {0.f, 0.f, 0.f, 0.f};
    const int n_pass = need_grad ? OC : 1;
#pragma unroll 1
    for (int c = 0; c < n_pass; ++c) {
      float gq0 = 0.f, gq1 = 0.f, gq2 = 0.f;
      if (need_grad) {
        // G_last = mask_last (.) w_out[c]  -> A operand (this thread's 16 columns)
#pragma unroll
        for (int cc = 0; cc < UM_CW / 4; ++cc) {
          const float4 wo = *reinterpret_cast<const float4*>(s_wout + c * H + cb * UM_CW + 4 * cc);
          float g[4] = {wo.x, wo.y, wo.z, wo.w};
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (!((mkL >> (4 * cc + e)) & 1u)) g[e] = leaky ? 0.01f * g[e] : 0.f;
          float4 hi, lo;
          um_split4(make_float4(g[0], g[1], g[2], g[3]), hi, lo);
          const int off = um_a_off(row, cb * (UM_CW / 4) + cc, H);
          *reinterpret_cast<float4*>(a_hi + off) = hi;
          *reinterpret_cast<float4*>(a_lo + off) = lo;
        }
        if (L > 1) {
          um_publish_and_sync();
          um_gemm_rows(a_hi_u, a_lo_u, A_SBO1, w1b_hi, w1b_lo, W_SBO1, H / 8, H, cb, xch, row, v);
#pragma unroll
          for (int cc = 0; cc < UM_CW / 4; ++cc) {
            float g[4] = {__uint_as_float(v[4 * cc]), __uint_as_float(v[4 * cc + 1]), __uint_as_float(v[4 * cc + 2]),
                          __uint_as_float(v[4 * cc + 3])};
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (!((mk0 >> (4 * cc + e)) & 1u)) g[e] = leaky ? 0.01f * g[e] : 0.f;
            float4 hi, lo;
            um_split4(make_float4(g[0], g[1], g[2], g[3]), hi, lo);
            const int off = um_a_off(row, cb * (UM_CW / 4) + cc, H);
            *reinterpret_cast<float4*>(a_hi + off) = hi;
            *reinterpret_cast<float4*>(a_lo + off) = lo;
          }
        }
        um_publish_and_sync();
        um_gemm_rows(a_hi_u, a_lo_u, A_SBO1, w0b_hi, w0b_lo, W_SBO1, H / 8, N0, cb, xch, row, v);
      } else {
        __syncthreads();  // output-head partial sums of the other column blocks
      }
      // decoder outputs of this row (the barriers above ordered the partial sums)
      if (c == 0) {
#pragma unroll
        for (int ch = 0; ch < 4; ++ch)
          if (ch < OC) {
            float oo = s_bout[ch];
#pragma unroll
            for (int b = 0; b < UM_CB; ++b) oo += s_part[(ch * UM_CB + b) * UM_ROWS + row];
            if (p.dec.sigmoid_out) {
              val[ch] = 1.f / (1.f + expf(-oo));
              dvv[ch] = val[ch] * (1.f - val[ch]);
            } else {
              val[ch] = oo * p.dec.out_scale;
              dvv[ch] = p.dec.out_scale;
            }
          }
      }
      const float val_c = c == 0 ? val[0] : (c == 1 ? val[1] : (c == 2 ? val[2] : val[3]));
      const float dv_c = c == 0 ? dvv[0] : (c == 1 ? dvv[1] : (c == 2 ? dvv[2] : dvv[3]));
      if (need_grad) {
        // every row of the A tile has been consumed by the MMA: the tile becomes the row-major input gradient
        if (cb * UM_CW < K0) {
#pragma unroll
          for (int cc = 0; cc < UM_CW / 4; ++cc)
            if (cb * UM_CW + 4 * cc < K0)
              *reinterpret_cast<float4*>(s_g + row * GLD + cb * UM_CW + 4 * cc) =
                  make_float4(__uint_as_float(v[4 * cc]) * dv_c, __uint_as_float(v[4 * cc + 1]) * dv_c,
                              __uint_as_float(v[4 * cc + 2]) * dv_c, __uint_as_float(v[4 * cc + 3]) * dv_c);
        }
        __syncthreads();

        // ---- C1: a_k = <g_xbar, f_k> for the warp's 8 queries (F/4 lanes per row, coalesced re-read of the K rows)
        {
          float4 fv[GU][KREG];
#pragma unroll
          for (int u = 0; u < GU; ++u) {
            const int ql = qb + u * M::RPP + sub;
#pragma unroll
            for (int k = 0; k < KREG; ++k) {
              fv[u][k] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (k < K && (!NARROW || sub < QPW)) {
                const int lif = s_li[k * WT + ql];
                if (lif >= 0) fv[u][k] = __ldg(f4 + (size_t)(lif & ~REMAP) * M::LPR);
              }
            }
          }
#pragma unroll
          for (int u = 0; u < GU; ++u) {
            const int ql = (NARROW && sub >= QPW) ? qb : qb + u * M::RPP + sub;  // idle lanes still take part in the shuffles
            const float4 g4 = *reinterpret_cast<const float4*>(s_g + (rq * WT + ql) * GLD + 4 * c4);
            float part[KREG];
#pragma unroll
            for (int k = 0; k < KREG; ++k)
              part[k] = fmaf(g4.w, fv[u][k].w, fmaf(g4.z, fv[u][k].z, fmaf(g4.y, fv[u][k].y, g4.x * fv[u][k].x)));
            int first, n_out;
            group_reduce8<M::LPR>(part, lane, first, n_out);
            const bool writer = M::LPR <= KREG ? true : (lane % (M::LPR / KREG)) == 0;
            if (writer && (!NARROW || sub < QPW))
#pragma unroll
              for (int i = 0; i < KREG; ++i)
                if (i < n_out && first + i < K) s_a[(first + i) * WT + ql] = part[i];
          }
        }
        __syncthreads();

        // ---- C2: thread per query (column block 0) -- chain rule through the IDW weights
        if (cb == 0 && live) {
          const int nn = s_nn[lane];
          const float usum = s_usum[lane];
          const float qx = s_q[lane], qy = s_q[WT + lane], qz = s_q[2 * WT + lane];
          const float gn0 = s_g[row * GLD + F + 0], gn1 = s_g[row * GLD + F + 1], gn2 = s_g[row * GLD + F + 2];
          float ak[KREG], wk[KREG], ck[KREG], dx[KREG], dy[KREG], dz[KREG];
#pragma unroll
          for (int k = 0; k < KREG; ++k) {
            ak[k] = wk[k] = ck[k] = dx[k] = dy[k] = dz[k] = 0.f;
            const int lif = k < K ? s_li[k * WT + lane] : -1;
            if (lif >= 0) {
              dx[k] = s_dx[k * WT + lane];
              dy[k] = s_dy[k * WT + lane];
              dz[k] = s_dz[k * WT + lane];
              float nx, ny, nz, r0 = gn0, r1 = gn1, r2 = gn2;
              float4 quat;
              neighbour_vec(m, lif, dx[k], dy[k], dz[k], qx, qy, qz, nx, ny, nz, quat);
              if (m.after_pgo) quat_rotate_active(quat.x, quat.y, quat.z, quat.w, gn0, gn1, gn2, r0, r1, r2);
              wk[k] = s_w[k * WT + lane];
              ak[k] = s_a[k * WT + lane] + gn0 * nx + gn1 * ny + gn2 * nz;
              ck[k] = nn > 0 ? -2.f * (wk[k] * usum) : 0.f;
              gq0 = fmaf(wk[k], r0, gq0);
              gq1 = fmaf(wk[k], r1, gq1);
              gq2 = fmaf(wk[k], r2, gq2);
            }
          }
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
      }
      // ---- outputs of this pass
      if (cb == 0 && live) {
        if (!p.is_color) {
          if (p.out.sdf) p.out.sdf[qi] = val_c;
          if (p.out.sdf_std) p.out.sdf_std[qi] = 0.f;
          if (need_grad && p.out.grad) {
            p.out.grad[3 * qi + 0] = gq0;
            p.out.grad[3 * qi + 1] = gq1;
            p.out.grad[3 * qi + 2] = gq2;
          }
        } else {
          if (p.out.color) {
            if (need_grad) {
              p.out.color[qi * OC + c] = val_c;
            } else {
#pragma unroll
              for (int cc = 0; cc < 4; ++cc)
                if (cc < OC) p.out.color[qi * OC + cc] = val[cc];
            }
          }
          if (need_grad && p.out.color_grad) {
            p.out.color_grad[(qi * OC + c) * 3 + 0] = gq0;
            p.out.color_grad[(qi * OC + c) * 3 + 1] = gq1;
            p.out.color_grad[(qi * OC + c) * 3 + 2] = gq2;
          }
        }
      }
      // the gradient tile aliases the A tile the next pass writes (the next TILE is ordered by its stash barrier)
      if (need_grad && c + 1 < n_pass) __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
template <int FT>
static UmmaLayout plan_umma_layout(const pinb200_decoder_view& d, bool need_grad) {
  using DM = UmmaDims<FT>;
  UmmaLayout l{};
  int o = 0;
  auto take = [&](int bytes) {
    const int at = o;
    o += (bytes + 127) & ~127;
    return at;
  };
  const int w0 = 64 * DM::K0 * 4, w1 = 64 * 64 * 4, w0b = DM::N0 * 64 * 4;
  l.w0f_hi = take(w0);
  l.w0f_lo = take(w0);
  if (d.n_hidden > 1) {
    l.w1f_hi = take(w1);
    l.w1f_lo = take(w1);
    if (need_grad) {
      l.w1b_hi = take(w1);
      l.w1b_lo = take(w1);
    }
  }
  if (need_grad) {
    l.w0b_hi = take(w0b);
    l.w0b_lo = take(w0b);
  }
  const int a_bytes = (UM_ROWS / 8) * (64 / 4) * UM_A_LBO;  // K = 64
  static_assert(UM_ROWS * UmmaDims<FT>::GLD * 4 <= (UM_ROWS / 8) * (64 / 4) * UM_A_LBO, "gradient tile must fit the A tile");
  static_assert(UM_CB * UM_ROWS * UM_CW * 4 <= (UM_ROWS / 8) * (64 / 4) * UM_A_LBO, "accumulator exchange must fit the A tile");
  l.a_hi = take(a_bytes);
  l.a_lo = take(a_bytes);
  l.b0 = take(64 * 4);
  l.b1 = take(64 * 4);
  l.wout = take(4 * 64 * 4);
  l.bout = take(16);
  l.warp_stride = (Stash::floats + WT * 8) * 4;
  l.warp0 = take(4 * l.warp_stride);
  l.part = take(4 * 4 * UM_ROWS * 4);
  l.total = o;
  return l;
}

template <int FT>
static int launch_decode_umma(QueryParams& p, cudaStream_t stream) {
  const UmmaLayout lay = plan_umma_layout<FT>(p.dec, p.opts.need_grad != 0);
  const size_t smem_bytes = (size_t)lay.total;  // no-swizzle descriptors need 16-byte alignment only
  if (smem_bytes > 227 * 1024) {
    set_error("decode_umma kernel needs %zu B shared memory (> 227 KB)", smem_bytes);
    return PINB200_ERR_UNSUPPORTED;
  }
  auto kern = decode_umma_kernel<FT>;
  static std::mutex mu;
  static std::vector<int> done;
  int dev = 0;
  cudaGetDevice(&dev);
  {
    std::lock_guard<std::mutex> lk(mu);
    if (std::find(done.begin(), done.end(), dev) == done.end()) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
      if (e != cudaSuccess) {
        set_error("cudaFuncSetAttribute(decode_umma): %s", cudaGetErrorString(e));
        return PINB200_ERR_CUDA;
      }
      done.push_back(dev);
    }
  }
  p.qpt = WT;
  p.n_tiles = (int)((p.n + WT - 1) / WT);
  const int n128 = (p.n_tiles + 3) / 4;
  const int grid = std::min(n128, sm_count());
  kern<<<grid, UM_THREADS, smem_bytes, stream>>>(p, lay);
  return check_launch("decode_umma_kernel");
}

// the tensor-core decode covers weighted_first maps with a 1- or 2-layer 64-wide decoder and F in {8, 16, 32}
static bool umma_decode_supported(const QueryParams& p) {
  const int F = p.dec.in_dim - 3;
  return p.opts.weighted_first && p.dec.hidden_dim == 64 && p.dec.n_hidden >= 1 && p.dec.n_hidden <= 2 &&
         (F == 8 || F == 16 || F == 32) && p.opts.nn_k <= KREG;
}

static int dispatch_decode_umma(QueryParams& p, cudaStream_t stream) {
  switch (p.dec.in_dim - 3) {
    case 8: return launch_decode_umma<8>(p, stream);
    case 16: return launch_decode_umma<16>(p, stream);
    case 32: return launch_decode_umma<32>(p, stream);
    default: break;
  }
  set_error("decode_umma: feature_dim %d unsupported", p.dec.in_dim - 3);
  return PINB200_ERR_UNSUPPORTED;
}

}  // namespace pinb
