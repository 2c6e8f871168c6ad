// K1b, warp-specialised: gather + decoder + d/dq of the split pipeline for weighted_first maps, as ONE persistent CTA
// per SM whose warps have different jobs and only meet through mbarriers (no block-wide barrier after the prologue):
//
//   G  gather teams   (2 x 4 warps, 120 registers) TMA bulk copies (cp.async.bulk, completion counted in bytes on an
//                     mbarrier) of what search_kernel wrote for a 32-query block -- neighbour ids, IDW weights, position
//                     part of the decoder input and, when d/dq is wanted, the forward-mode seeds  omega_kj = d w_k / d q_j
//                     and d(position part)/dq -- into a ring of "meta" blocks in shared memory, issued by one lane a few
//                     blocks ahead; then F/4 lanes per feature row (a 128-byte row = 8 lanes x LDG.128): ONE pass over the
//                     K rows gives the IDW-interpolated feature  xbar = sum_k w_k f_k  AND its three directional
//                     derivatives  T_j = sum_k omega_kj (f_k - f_0)  -> rows of an A tile (canonical K-major, hi / lo TF32)
//   C  consumers      (2 warpgroups, 136 registers; warpgroup h owns the 64-row half h of every tile) layer 0 as
//                     wgmma.mma_async with the A tile from shared memory (accumulators in registers), then releases the A
//                     tile to its gather team; ReLU gate, hi / lo split in registers, layer 1 with the A operand IN
//                     REGISTERS (the accumulator fragment is the A fragment once the k order inside a k-step is permuted,
//                     see um_kperm: the layer-1 weights are staged in that order); last layer: output head in registers
//                     (quad shuffles), results to global memory.  The two warpgroups drift apart, so one's MMA waits run
//                     under the other's epilogue.
//
// d sdf / d q is computed in FORWARD mode: a tile row is either a value row (decoder input x) or one of the three
// tangent rows (dx / dq_j) of the same query; tangent rows go through the same weights, without bias, and are gated
// by the value row's ReLU pattern.  Rows 4i .. 4i+3 of a tile belong to query i, so in the accumulator fragment the
// gate comes from the lane four rows up (one shuffle of a 32-bit mask per 64-row half).  This needs no transposed weight
// copies, no backward MMAs, no second pass over the feature rows (a backward decode needs one for <d/d xbar, f_k>) and
// no input-gradient tile, which is what makes room for a ring of A tiles: the gathers of later tiles run under the MMA
// chain of tile t.  Without d/dq (mesher, dense RGB-D queries) a tile is 128 value rows.
//
// With a single output channel (the SDF head) d/dq takes the ADJOINT schedule instead: for a 2-layer head,
// d out / d q_j = s v' . u_j with u_j = W0 (dx/dq_j) (the layer-0 tangent), ONE adjoint vector per query
// v' = D0 W1^T (w_out . D1) (D = the (leaky-)ReLU derivative masks of the value row; L = 1: v' = D0 w_out) and s the
// output scale or sigmoid derivative, so the tangent rows stop at layer 0: 108 instead of 156 wgmma per 64 queries.
// Gather team h fills 64-query groups that consumer warpgroup h alone decodes: four fp32 blocks V, T1, T2, T3 of 64
// rows each, row r of every block = query r, so a thread holds the same accumulator elements of the value rows, of v'
// and of every u_j (no mask shuffle).  Layer 0 takes its A fragments from these blocks through registers (split into
// hi / lo there: fp32 blocks are half the size of hi / lo tiles, which is what leaves room for the staged W1^T).
// A colour Jacobian (3 channels) would need three adjoint vectors and save no MMA work, so it stays in forward mode.
//
// Replaces model/neural_points.py:598-731 (gathers, IDW, weighted_first), model/decoder.py:61-85,112 and the autograd
// call of utils/tools.py:247-260 for batches of >= PINB200_SPLIT_MIN_QUERIES_WF queries (inference mode).
#include "query_dev.cuh"
#include "umma_common.cuh"

namespace pinb {

constexpr int WS_CG = 2;       // consumer warpgroups: warpgroup h owns rows 64 h .. 64 h + 63 (half h) of every tile
constexpr int WS_CW = 4 * WS_CG;  // consumer warps
constexpr int WS_GT = 2;       // gather teams of 4 warps: team t fills the A tiles of the CTA's tiles i = t (mod WS_GT)
constexpr int WS_GW = 4;       // warps per gather team
constexpr int WS_THREADS = (WS_CW + WS_GT * WS_GW) * 32;
// register budget per thread (setmaxnreg, one value per 4-warp group).  The pool is what the CTA was launched with
// (512 threads x 128 registers)
constexpr int WS_REG_C = 136, WS_REG_G = 120;
static_assert((WS_CW * WS_REG_C + WS_GT * WS_GW * WS_REG_G) * 32 <= WS_THREADS * 128, "setmaxnreg pool");
constexpr int WS_A0 = 2;       // A-tile ring slots, one per gather team
// ring of the original query indices of a tile: tile i in slot i % WS_QX.  Slot i % WS_QX is
// rewritten for tile i + WS_QX only after the A tile of tile i + WS_A0 was released, i.e. after every consumer warp
// stored tile i
constexpr int WS_QX = 2 * WS_A0;
// adjoint schedule (d/dq of a single-output head): a group of 64 queries is four 64-row fp32 blocks V, T1, T2, T3 of
// WS_LDA floats per row; WS_LDA == 4 (mod 32) keeps the consumers' scalar A-fragment loads free of bank conflicts.
// Columns >= WS_LDA (the last four of K0 = 40) are zero and never stored
constexpr int WS_QG = 64;
constexpr int WS_LDA = 36;
constexpr int WS_GBLK = WS_QG * WS_LDA;  // floats per block of a group

struct WsMeta {  // float offsets inside a meta block of 32 queries, [field][k][lane]
  static constexpr int li = 0;                   // [8][32] neighbour id | REMAP, -1 invalid
  static constexpr int w = li + WT * 8;          // [8][32] IDW weight
  static constexpr int xn = w + WT * 8;          // [3][32] sum_k w_k n_k
  static constexpr int perm = xn + WT * 3;       // [32] original query index, -1 past the end of the batch
  static constexpr int floats_ng = perm + WT;
  static constexpr int om = floats_ng;           // [3][8][32] d w_k / d q_j
  static constexpr int P = om + WT * 24;         // [3 j][3 i][32] d (sum_k w_k n_k)_i / d q_j
  static constexpr int floats_g = P + WT * 9;
};

struct WsLayout {  // byte offsets from the dynamic shared memory base
  int adj;                     // 1: adjoint schedule (d/dq with one output channel), A slots are fp32 groups
  int w0_hi, w0_lo, w1_hi, w1_lo, w1t_hi, w1t_lo, b0, b1, wout, bout;
  int a0, a0_half, a0_stride;  // ring of A tiles: slot s = [a0 + s*stride: hi | + half: lo] (adjoint: one fp32 group)
  int qidx;                    // [WS_QX][128] original query index of every tile row's query
  int meta, meta_stride, n_meta;
  int bars, total;
};
// mbarrier indices
constexpr int WS_MB_MAX = 16;
constexpr int WSB_A0_FULL = 0, WSB_A0_EMPTY = WSB_A0_FULL + WS_A0, WSB_META_FULL = WSB_A0_EMPTY + WS_A0,
              WSB_META_EMPTY = WSB_META_FULL + WS_MB_MAX, WSB_COUNT = WSB_META_EMPTY + WS_MB_MAX;

// Optional cycle accounting (pinb200_set_option("ws_profile", 1)): per warp, clock deltas of up to 7 phases,
// summed over the tiles of the launch, for the first WS_PROF_CTAS CTAs; read back with
// pinb200_debug_read("ws_profile", ...).  The last slot of every warp holds its role code (WS_ROLE_*), so that a
// reader of the counters (scripts/exp_decode.py) follows the kernel's role layout.
constexpr int WS_PROF_SLOTS = 8;
// C consumer warps (CA: of the adjoint schedule), G gather warps that also fill the meta ring
constexpr int WS_ROLE_C = 1, WS_ROLE_CA = 2, WS_ROLE_G = 4;
constexpr int WS_PROF_CTAS = 132;  // one CTA per SM of an H100 SXM
__device__ unsigned long long g_ws_prof[WS_PROF_CTAS * (WS_THREADS / 32) * WS_PROF_SLOTS];
static int g_ws_profile = 0;

template <bool PROF>
struct WsClock {  // PROF = false: no code at all (64-bit counters in the production kernel spilled to local memory)
  unsigned int acc[WS_PROF_SLOTS];
  unsigned int last;
  __device__ __forceinline__ void start() {
    if (PROF) {
#pragma unroll
      for (int i = 0; i < WS_PROF_SLOTS; ++i) acc[i] = 0u;
      last = (unsigned int)clock();
    }
  }
  __device__ __forceinline__ void lap(int slot) {
    if (PROF) {
      const unsigned int now = (unsigned int)clock();
      acc[slot] += now - last;
      last = now;
    }
  }
  __device__ __forceinline__ void flush(int warp, int role) {
    if (PROF) {
      if ((threadIdx.x & 31) == 0 && blockIdx.x < WS_PROF_CTAS) {
        unsigned long long* dst = g_ws_prof + (blockIdx.x * (WS_THREADS / 32) + warp) * WS_PROF_SLOTS;
#pragma unroll
        for (int i = 0; i < WS_PROF_SLOTS - 1; ++i) dst[i] = acc[i];
        dst[WS_PROF_SLOTS - 1] = (unsigned long long)role;
      }
    }
  }
};

// mbarrier wait, executed by every lane of a converged warp (ONE warp instruction per attempt).  The suspend-time hint
// parks the warp in hardware until the phase completes, instead of a software poll loop that steals issue slots from
// the working warps.  Bounded: a mis-programmed pipeline must trap, not hang the GPU.
__device__ __forceinline__ void ws_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
#pragma unroll 1
  for (int it = 0; it < 2048 && !done; ++it) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(1000000)  // <= 1 ms per attempt
        : "memory");
  }
  if (!done) __trap();
}
// ring waits of the producer roles (not latency critical): back off between attempts instead of re-polling
__device__ __forceinline__ void ws_wait_relaxed(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
#pragma unroll 1
  for (int it = 0; it < (1 << 22) && !done; ++it) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(1000000)
        : "memory");
    if (!done) __nanosleep(128);
  }
  if (!done) __trap();
}
__device__ __forceinline__ void ws_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

static_assert(WsMeta::P - WsMeta::om == Seeds::P - Seeds::om && WsMeta::floats_g - WsMeta::om == Seeds::floats,
              "the seed block of the search launch is copied verbatim into the meta block");
static_assert(WsMeta::xn == StashS::pos && WsMeta::perm == StashS::perm && WsMeta::floats_ng == StashS::floats,
              "the stash block is the head of the meta block (one bulk copy)");

// fn(std::integral_constant<int, s>) for s = 0 .. N-1: a k-step loop whose step is a compile-time constant
template <typename Fn, int... S>
__device__ __forceinline__ void ws_unroll_seq(Fn&& fn, std::integer_sequence<int, S...>) {
  (fn(std::integral_constant<int, S>{}), ...);
}
template <int N, typename Fn>
__device__ __forceinline__ void ws_unroll(Fn&& fn) {
  ws_unroll_seq(fn, std::make_integer_sequence<int, N>{});
}

__device__ __forceinline__ bool ws_elect() {  // one lane of the (converged) warp; keeps the code warp-uniform for the compiler
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}
// TMA bulk copy global -> shared, completion counted in bytes on an mbarrier
__device__ __forceinline__ void ws_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(um_smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void ws_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

template <int FT, bool GRAD, bool PROF>
__global__ void __launch_bounds__(WS_THREADS, 1) wsq_decode_kernel(const __grid_constant__ QueryParams p, const WsLayout lay) {
  constexpr int H = 64;
  using DM = UmmaDims<FT>;
  constexpr int K0 = DM::K0, F = FT, D = FT + 3;
  using M = RowMap<FT>;
  const bool adj = GRAD && lay.adj;     // adjoint schedule: tiles are 64-query groups, one per consumer warpgroup
  const int QT = adj ? WS_QG : (GRAD ? 32 : 128);  // queries per tile
  const int BPT = QT / WT;              // meta blocks per tile
  constexpr int MB = GRAD ? 8 : 16;     // meta ring slots (blocks of 32 queries; a value-only tile has 4)
  constexpr int MSTRIDE = GRAD ? WsMeta::floats_g : WsMeta::floats_ng;
  constexpr int NPASS = WT / M::RPP;    // gather passes per meta block (F = 32: 8 passes of 4 queries)
  extern __shared__ __align__(1024) unsigned char ws_smem[];
  unsigned char* sm = ws_smem;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const pinb200_map_view& m = p.map;
  const int K = p.opts.nn_k, L = p.dec.n_hidden, OC = p.dec.out_dim;
  const float slope = p.dec.leaky_relu ? 0.01f : 0.f;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + lay.bars);
  float* meta = reinterpret_cast<float*>(sm + lay.meta);
  WsClock<PROF> clk;

  // ---- prologue (the only block-wide barrier): mbarriers, decoder weights
  if (tid == 0) {
    auto init = [&](int i, int count) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(um_smem_u32(bars + i)), "r"(count));
    };
    for (int s = 0; s < WS_A0; ++s) {
      init(WSB_A0_FULL + s, WS_GW);
      init(WSB_A0_EMPTY + s, adj ? 4 : WS_CW);  // adjoint: one warpgroup consumes a group
    }
    for (int s = 0; s < WS_MB_MAX; ++s) {
      init(WSB_META_FULL + s, 1);
      init(WSB_META_EMPTY + s, WS_GW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;");
  }
  um_stage_weight(p.dec.w[0], D, H, D, H, K0, sm + lay.w0_hi, sm + lay.w0_lo);
  if (L > 1) um_stage_weight(p.dec.w[1], H, H, H, H, H, sm + lay.w1_hi, sm + lay.w1_lo, true);
  if (adj && L > 1) um_stage_weight(p.dec.w[1], H, H, H, H, H, sm + lay.w1t_hi, sm + lay.w1t_lo, true, true);
  __syncthreads();
  // the layer-0 bias rides on the MMA: input column D is 1 for value rows (0 for tangent rows), weight column D = b0
  static_assert(D < K0, "a spare (padding) input column carries the bias");
  if (tid < H) {
    const float bv = p.dec.b[0] ? __ldg(p.dec.b[0] + tid) : 0.f;
    const float bh = __uint_as_float(__float_as_uint(bv) & TF32_MASK);
    const int off = (tid >> 3) * ((K0 >> 2) * UM_W_LBO) + (D >> 2) * UM_W_LBO + (tid & 7) * 16 + (D & 3) * 4;
    *reinterpret_cast<float*>(sm + lay.w0_hi + off) = bh;
    *reinterpret_cast<float*>(sm + lay.w0_lo + off) = bv - bh;
  }
  for (int e = tid; e < H; e += WS_THREADS) {
    reinterpret_cast<float*>(sm + lay.b0)[e] = 0.f;  // layer-0 bias: see the weight staging above
    reinterpret_cast<float*>(sm + lay.b1)[e] = (L > 1 && p.dec.b[1]) ? __ldg(p.dec.b[1] + e) : 0.f;
  }
  for (int e = tid; e < 4 * H; e += WS_THREADS) reinterpret_cast<float*>(sm + lay.wout)[e] = e < OC * H ? __ldg(p.dec.w_out + e) : 0.f;
  if (tid < 4) reinterpret_cast<float*>(sm + lay.bout)[tid] = (p.dec.b_out && tid < OC) ? __ldg(p.dec.b_out + tid) : 0.f;
  um_publish_and_sync();
  clk.start();

  const long long n_tiles = (p.n + QT - 1) / QT;
  const int n_blocks = p.n_tiles;  // 32-query stash blocks

  if (warp < WS_CW) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WS_REG_C));
    // =====================================================================================================
    // C: both consumer warpgroups work through every tile of this CTA; warpgroup h takes rows 64 h .. 64 h + 63 of a
    // tile (half h), so one warpgroup's MMA waits run under the other's epilogue.  The four rows of a query lie in
    // the same half.  In the accumulator fragment this thread holds rows 64 h + 16 wq + g8 (+ 8) and columns
    // 8 j + 2 c (+ 1).
    // profile slots: 0 wait A tile, 1 layer 0, 2 layer 1, 3 last-layer epilogue + outputs
    // =====================================================================================================
    const int h = warp / 4, wq = warp % 4;
    const int g8 = lane >> 2, c = lane & 3;
    const int t = GRAD ? (g8 & 3) : 0;  // row type: 0 value, 1..3 tangent d/dq_{t-1}
    const float bsel = t == 0 ? 1.f : 0.f;
    const int src = lane & ~12;  // the lane holding the same columns of this row's value row
    const float* s_b1 = reinterpret_cast<const float*>(sm + lay.b1);
    const float* s_wout = reinterpret_cast<const float*>(sm + lay.wout);
    const float* s_bout = reinterpret_cast<const float*>(sm + lay.bout);
    constexpr uint32_t A_SBO0 = (K0 / 4) * UM_A_LBO, W_SBO0 = (K0 / 4) * UM_W_LBO, W_SBO1 = (H / 4) * UM_W_LBO;
    // a k-step (8 columns = two 16-byte chunks) advances the start-address field of a descriptor by 2 * LBO / 16
    constexpr uint64_t A_STEP = (2 * UM_A_LBO) >> 4, W_STEP = (2 * UM_W_LBO) >> 4, A_HALF = (8 * A_SBO0) >> 4;
    const uint64_t w0h_d = um_desc(um_smem_u32(sm + lay.w0_hi), UM_W_LBO, W_SBO0), w0l_d = um_desc(um_smem_u32(sm + lay.w0_lo), UM_W_LBO, W_SBO0);
    const uint64_t w1h_d = um_desc(um_smem_u32(sm + lay.w1_hi), UM_W_LBO, W_SBO1), w1l_d = um_desc(um_smem_u32(sm + lay.w1_lo), UM_W_LBO, W_SBO1);

    // bias (times bs: 1 for value rows, 0 for tangent rows; `bias` may be null) + ReLU gate of the 32 accumulator
    // values of a half; returns the sign pattern.  In a forward-mode tile (`interleaved`) the gate of a tangent row is
    // the sign pattern of its query's value row: the 32 sign bits travel in ONE shuffle.
    auto gate = [&](float (&z)[32], const float* bias, float bs, bool interleaved) {
      if (bias) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * c);
          z[4 * j] = fmaf(bs, b.x, z[4 * j]);
          z[4 * j + 1] = fmaf(bs, b.y, z[4 * j + 1]);
          z[4 * j + 2] = fmaf(bs, b.x, z[4 * j + 2]);
          z[4 * j + 3] = fmaf(bs, b.y, z[4 * j + 3]);
        }
      }
      uint32_t mk = 0u;
#pragma unroll
      for (int e = 0; e < 32; ++e) mk |= z[e] > 0.f ? (1u << e) : 0u;
      if (GRAD && interleaved) mk = __shfl_sync(FULL, mk, src);
#pragma unroll
      for (int e = 0; e < 32; ++e) z[e] = ((mk >> e) & 1u) ? z[e] : slope * z[e];
      return mk;
    };
    // D = A W^T (64 x 64 x 64, 3xTF32) with A the accumulator fragment `a` of a 64 x 64 activation (overwritten with
    // its hi part) and W a weight staged with kperm: the accumulator fragment is the A fragment once the k order inside
    // a k-step is permuted
    auto mma_rs64 = [&](float (&a)[32], float (&d)[32], uint64_t wh_d, uint64_t wl_d) {
      uint32_t lo[32];
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        d[e] = 0.f;
        const float hi = __uint_as_float(__float_as_uint(a[e]) & TF32_MASK);
        lo[e] = __float_as_uint(a[e] - hi);
        a[e] = hi;
      }
      wg_fence();
      ws_unroll<H / 8>([&](auto S) {
        constexpr int s = decltype(S)::value, WO = s * W_STEP;
        const uint32_t h0 = __float_as_uint(a[4 * s]), h1 = __float_as_uint(a[4 * s + 2]), h2 = __float_as_uint(a[4 * s + 1]),
                       h3 = __float_as_uint(a[4 * s + 3]);
        wg_mma_n64_rs_at<WO>(d, lo[4 * s], lo[4 * s + 2], lo[4 * s + 1], lo[4 * s + 3], wh_d, s > 0);  // small terms first
        wg_mma_n64_rs_at<WO>(d, h0, h1, h2, h3, wl_d, 1);
        wg_mma_n64_rs_at<WO>(d, h0, h1, h2, h3, wh_d, 1);
      });
      wg_commit();
      wg_wait0();
    };
    // output head of the two rows of this thread (quad-reduced: every lane of the quad holds the sums)
    auto head = [&](const float (&z)[32], float (&o)[2][4]) {
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        o[0][ch] = o[1][ch] = 0.f;
        if (ch < OC) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 w = *reinterpret_cast<const float2*>(s_wout + ch * H + 8 * j + 2 * c);
            o[0][ch] = fmaf(z[4 * j + 1], w.y, fmaf(z[4 * j], w.x, o[0][ch]));
            o[1][ch] = fmaf(z[4 * j + 3], w.y, fmaf(z[4 * j + 2], w.x, o[1][ch]));
          }
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            o[r][ch] += __shfl_xor_sync(FULL, o[r][ch], 1);
            o[r][ch] += __shfl_xor_sync(FULL, o[r][ch], 2);
          }
        }
      }
    };
    // where this row's results go: element (query qi, channel ch) at out_base[qi * out_qstride + ch * out_chstride]
    float* out_base;
    float* out_std = nullptr;
    int out_qstride, out_chstride, out_nch = p.is_color ? OC : 1;
    if (t == 0) {
      out_base = p.is_color ? p.out.color : p.out.sdf;
      out_qstride = p.is_color ? OC : 1;
      out_chstride = 1;
      if (!p.is_color) out_std = p.out.sdf_std;
    } else {
      out_base = p.is_color ? p.out.color_grad : p.out.grad;
      if (out_base) out_base += t - 1;
      out_qstride = p.is_color ? 3 * OC : 3;
      out_chstride = 3;
    }
    // value rows write the prediction, tangent rows one component of its gradient; lane c == r of the quad writes row r.
    // Tile i holds queries T * QT .. in search order, mapped to their original index through the index ring the
    // gather team filled (shared memory: no global load on this path)
    const int* s_qidx = reinterpret_cast<const int*>(sm + lay.qidx);
    auto store = [&](long long T, int i, float (&o)[2][4]) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (p.dec.sigmoid_out) {
#pragma unroll
          for (int ch = 0; ch < 4; ++ch)
            if (ch < OC) {
              const float oo = fmaf(bsel, s_bout[ch], o[r][ch]);
              const float val = 1.f / (1.f + expf(-oo));
              const float dv = val * (1.f - val);
              const float dvq = GRAD ? __shfl_sync(FULL, dv, src) : dv;
              o[r][ch] = t == 0 ? val : dvq * oo;
            }
        } else {
#pragma unroll
          for (int ch = 0; ch < 4; ++ch) o[r][ch] = fmaf(bsel, s_bout[ch], o[r][ch]) * p.dec.out_scale;
        }
        const int row = 64 * h + 16 * wq + g8 + 8 * r, qrow = GRAD ? (row >> 2) : row;
        if (c == r && T * QT + qrow < p.n) {  // the tail of the last tile carries no valid index
          const long long qi = s_qidx[(i % WS_QX) * QT + qrow];
          if (out_base) {
            float* dst = out_base + qi * out_qstride;
#pragma unroll
            for (int ch = 0; ch < 4; ++ch)
              if (ch < out_nch) dst[ch * out_chstride] = o[r][ch];
          }
          if (out_std) out_std[qi] = 0.f;
        }
      }
    };

    if (adj) {
      // ---------------------------------------------------------------------------------------------------
      // Adjoint schedule (d/dq of a single-output head): warpgroup h consumes the groups i = h (mod 2) of this CTA,
      // which gather team h fills into A slot h.  Row r of each block V, T1, T2, T3 of a group is query r, so the
      // thread that holds element (r, col) of u_j = W0 T_j also holds it for the value rows and for
      //   v' = D0 W1^T (w_out . D1)   (L = 1: D0 w_out),   and   d out / d q_j = v' . u_j:
      // the tangents stop at layer 0 and need neither the value row's mask shuffle nor a second layer.
      // profile slots: 0 wait A group, 1 value rows (layers, head, sdf), 2 adjoint, 3 tangents + gradient stores
      // ---------------------------------------------------------------------------------------------------
      const uint64_t w1th_d = um_desc(um_smem_u32(sm + lay.w1t_hi), UM_W_LBO, W_SBO1),
                     w1tl_d = um_desc(um_smem_u32(sm + lay.w1t_lo), UM_W_LBO, W_SBO1);
      const int row0 = 16 * wq + g8;  // this thread's rows of every block: row0, row0 + 8
      float* out_v = p.is_color ? p.out.color : p.out.sdf;
      float* out_g = p.is_color ? p.out.color_grad : p.out.grad;
      float* out_s = p.is_color ? nullptr : p.out.sdf_std;
      // layer 0 of one 64-row block: the A fragments come from the fp32 group and are split into hi / lo in registers
      // (same 3xTF32 terms and order as an A tile stored hi / lo).  `release` frees the A slot once they are loaded
      auto layer0 = [&](const float* blk, float (&d)[32], int slot, bool release) {
        const float* r = blk + row0 * WS_LDA + c;
        float a[K0 / 8][4];
        ws_unroll<K0 / 8>([&](auto S) {
          constexpr int s = decltype(S)::value;
          a[s][0] = r[8 * s];
          a[s][1] = r[8 * WS_LDA + 8 * s];
          if constexpr (8 * s + 4 < WS_LDA) {
            a[s][2] = r[8 * s + 4];
            a[s][3] = r[8 * WS_LDA + 8 * s + 4];
          } else {
            a[s][2] = a[s][3] = 0.f;
          }
        });
        if (release) {
          __syncwarp();
          if (lane == 0) ws_arrive(um_smem_u32(bars + WSB_A0_EMPTY + slot));  // the gather team may refill the slot
        }
#pragma unroll
        for (int e = 0; e < 32; ++e) d[e] = 0.f;
        ws_unroll<K0 / 8>([&](auto S) {
          constexpr int s = decltype(S)::value, WO = s * W_STEP;
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            hi[k] = __float_as_uint(a[s][k]) & TF32_MASK;
            lo[k] = __float_as_uint(a[s][k] - __uint_as_float(hi[k]));
          }
          wg_fence();
          wg_mma_n64_rs_at<WO>(d, lo[0], lo[1], lo[2], lo[3], w0h_d, s > 0);  // small terms first
          wg_mma_n64_rs_at<WO>(d, hi[0], hi[1], hi[2], hi[3], w0l_d, 1);
          wg_mma_n64_rs_at<WO>(d, hi[0], hi[1], hi[2], hi[3], w0h_d, 1);
        });
        wg_commit();
        wg_wait0();
      };

      int i = h;
      for (long long G = blockIdx.x + (long long)h * gridDim.x; G < n_tiles; G += (long long)WS_GT * gridDim.x, i += WS_GT) {
        const int slot = i % WS_A0;
        ws_wait(um_smem_u32(bars + WSB_A0_FULL + slot), (uint32_t)(i / WS_A0) & 1u);
        clk.lap(0);
        const float* grp = reinterpret_cast<const float*>(sm + lay.a0 + slot * lay.a0_stride);
        // ---- value rows: layer 0 (bias through the MMA), gate, layer 1, head, sdf
        float d0[32], v[32], o[2][4];
        layer0(grp, d0, slot, false);
        const uint32_t m0 = gate(d0, nullptr, 1.f, false);
        if (L > 1) {
          mma_rs64(d0, v, w1h_d, w1l_d);
          const uint32_t m1 = gate(v, s_b1, 1.f, false);
          head(v, o);
          // g1 = w_out . D1, the A operand of the adjoint layer
#pragma unroll
          for (int e = 0; e < 32; ++e)
            v[e] = s_wout[8 * (e >> 2) + 2 * c + (e & 1)] * (((m1 >> e) & 1u) ? 1.f : slope);
        } else {
          head(d0, o);
#pragma unroll
          for (int e = 0; e < 32; ++e) v[e] = s_wout[8 * (e >> 2) + 2 * c + (e & 1)];
        }
        // lane c = r of a quad stores the results of row r (r = 0, 1)
        const bool st = c < 2 && G * QT + row0 + 8 * c < p.n;  // the tail of the last group carries no valid index
        const long long qi = st ? s_qidx[(i % WS_QX) * QT + row0 + 8 * c] : 0;
        float sc[2];  // d out / d (head sum) of the two rows
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float oo = o[r][0] + s_bout[0];
          float val;
          if (p.dec.sigmoid_out) {
            val = 1.f / (1.f + expf(-oo));
            sc[r] = val * (1.f - val);
          } else {
            val = oo * p.dec.out_scale;
            sc[r] = p.dec.out_scale;
          }
          if (st && c == r) {
            if (out_v) out_v[qi] = val;
            if (out_s) out_s[qi] = 0.f;
          }
        }
        clk.lap(1);
        // ---- adjoint: v' = D0 (W1^T g1), scaled by d out / d (head sum)
        if (L > 1) {
          mma_rs64(v, d0, w1th_d, w1tl_d);
#pragma unroll
          for (int e = 0; e < 32; ++e) v[e] = d0[e];
        }
#pragma unroll
        for (int e = 0; e < 32; ++e) v[e] = (((m0 >> e) & 1u) ? v[e] : slope * v[e]) * sc[(e >> 1) & 1];
        clk.lap(2);
        // ---- tangent rows: u_j = W0 T_j (T rows carry 0 in the bias column), d out / d q_j = v' . u_j
        float* const gdst = st && out_g ? out_g + 3 * qi : nullptr;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          layer0(grp + (j + 1) * WS_GBLK, d0, slot, j == 2);
          float g[2];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float acc = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              acc = fmaf(v[4 * jj + 2 * r], d0[4 * jj + 2 * r], acc);
              acc = fmaf(v[4 * jj + 2 * r + 1], d0[4 * jj + 2 * r + 1], acc);
            }
            acc += __shfl_xor_sync(FULL, acc, 1);
            g[r] = acc + __shfl_xor_sync(FULL, acc, 2);
          }
          if (gdst) gdst[j] = c == 0 ? g[0] : g[1];
        }
        clk.lap(3);
      }
    } else {
      int i = 0;
      for (long long T = blockIdx.x; T < n_tiles; T += gridDim.x, ++i) {
        const int slot = i % WS_A0;
        ws_wait(um_smem_u32(bars + WSB_A0_FULL + slot), (uint32_t)(i / WS_A0) & 1u);
        clk.lap(0);
        // ---- layer 0 of this warpgroup's half, A tile from shared memory
        float d0[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) d0[e] = 0.f;
        {
          const uint32_t a_hi = um_smem_u32(sm + lay.a0 + slot * lay.a0_stride);
          const uint64_t ah = um_desc(a_hi, UM_A_LBO, A_SBO0) + h * A_HALF, al = um_desc(a_hi + lay.a0_half, UM_A_LBO, A_SBO0) + h * A_HALF;
          wg_fence();
          ws_unroll<K0 / 8>([&](auto S) {
            constexpr int s = decltype(S)::value, AO = s * A_STEP, WO = s * W_STEP;
            wg_mma_n64_at<AO, WO>(d0, al, w0h_d, s > 0);  // small terms first
            wg_mma_n64_at<AO, WO>(d0, ah, w0l_d, 1);
            wg_mma_n64_at<AO, WO>(d0, ah, w0h_d, 1);
          });
          wg_commit();
          wg_wait0();
        }
        __syncwarp();
        if (lane == 0) ws_arrive(um_smem_u32(bars + WSB_A0_EMPTY + slot));  // the gather team may refill the A tile
        clk.lap(1);
        float o[2][4];
        if (L > 1) {
          // ---- layer-0 epilogue (the bias came through the MMA): gated activations -> layer 1 with the A operand
          // from registers
          float d1[32];
          gate(d0, nullptr, bsel, true);
          mma_rs64(d0, d1, w1h_d, w1l_d);
          clk.lap(2);
          // ---- last hidden layer: bias, gate, output head(s), results
          gate(d1, s_b1, bsel, true);
          head(d1, o);
          store(T, i, o);
        } else {
          // single hidden layer: its bias came through the MMA
          gate(d0, nullptr, bsel, true);
          head(d0, o);
          store(T, i, o);
        }
        clk.lap(3);
      }
    }
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WS_REG_G));
    // =====================================================================================================
    // G: gather teams -- the 4 warps of a team work on the same tile, each on its share of the queries: per round a
    // lane has GU passes x K feature-row loads (16 x LDG.128 for F = 32) in flight; the two teams (and the ring of A
    // tiles) overlap one team's load latency with the other team's reduction.  (A register double buffer over the
    // passes of ONE warp was tried: it spills inside the loop at 120 registers and lost 5 %.)
    //
    // The teams also fill the meta ring: TMA bulk copies (cp.async.bulk, completion counted in bytes on the block's
    // "full" mbarrier; no thread touches the data) of what search_kernel wrote for a 32-query block -- the StashS block
    // (2.5 KB: neighbour ids, IDW weights, position part, original query indices) and, with d/dq, the forward-mode
    // seeds (4.1 KB).  Block blk + MB of the
    // ring belongs to the same team as block blk, so a team refills its own slots: position j of the team's stream of
    // meta blocks takes the slot of position j - MD, and before it works on position j one warp of the team (in
    // turn) issues position j + PF, whose slot the team left two positions ago.
    // profile slots: 0 wait free A tile, 1 wait meta block, 2 feature-row loads issued, 3 reduce + A-tile stores,
    //                4 position rows + fence + arrive, 5 meta refill (wait free slot + copies), 6 wait for the search grid
    // =====================================================================================================
    const int team = (warp - WS_CW) / WS_GW, gw = (warp - WS_CW) % WS_GW;
    const int sub = lane / M::LPR, c4 = lane % M::LPR;
    const float4* __restrict__ f4 = reinterpret_cast<const float4*>(p.feat) + c4;
    constexpr int GU = NPASS / WS_GW >= 2 ? 2 : 1;  // passes in flight per gather warp
    static_assert(MB % (WS_GT * (GRAD ? WS_QG / WT : 128 / WT)) == 0, "the slots of a team's meta blocks repeat every MB blocks");
    constexpr int MD = MB / WS_GT;  // meta slots per team
    constexpr int PF = MD - 2;      // meta blocks in flight ahead of the one being gathered
    static_assert(PF >= 1, "meta ring too small to refill ahead");
    // position jj of this team's stream: block b = jj % BPT of its tile i = team + WS_GT * (jj / BPT)
    auto refill = [&](int jj) {
      if (jj % WS_GW != gw) return;
      const int ri = team + WS_GT * (jj / BPT), b = jj % BPT;
      const long long T = blockIdx.x + (long long)ri * gridDim.x;
      if (T >= n_tiles) return;
      const int blk = ri * BPT + b, ms = blk % MB;
      ws_wait_relaxed(um_smem_u32(bars + WSB_META_EMPTY + ms), ((uint32_t)(blk / MB) & 1u) ^ 1u);
      float* mt = meta + ms * MSTRIDE;
      const uint32_t full = um_smem_u32(bars + WSB_META_FULL + ms);
      const long long st = T * BPT + b;  // stash block
      if (st < n_blocks) {
        if (ws_elect()) {
          constexpr uint32_t B_S = StashS::floats * 4, B_SD = Seeds::floats * 4;
          ws_arrive_expect_tx(full, B_S + (GRAD ? B_SD : 0u));
          ws_bulk_g2s(mt, p.stash + (size_t)st * StashS::floats, B_S, full);  // li | w | pos | perm: one copy
          if (GRAD) ws_bulk_g2s(mt + WsMeta::om, p.seeds + (size_t)st * Seeds::floats, B_SD, full);
        }
      } else {  // tail of the last value-only tile or adjoint group: a block without neighbours
        for (int e = lane; e < MSTRIDE; e += 32) mt[e] = e < WsMeta::w ? __int_as_float(-1) : 0.f;
        __syncwarp();
        if (lane == 0) ws_arrive(full);
      }
      __syncwarp();
    };
    // the meta copies read what the search launch wrote: with programmatic dependent launch this grid may have
    // started before that one finished
    asm volatile("griddepcontrol.wait;" ::: "memory");
    clk.lap(6);
    for (int jj = 0; jj < PF; ++jj) refill(jj);
    clk.lap(5);
    int i = team, j = 0;
    for (long long T = blockIdx.x + (long long)team * gridDim.x; T < n_tiles; T += (long long)WS_GT * gridDim.x, i += WS_GT) {
      const int slot = i % WS_A0;
      unsigned char* a_hi = sm + lay.a0 + slot * lay.a0_stride;
      unsigned char* a_lo = a_hi + lay.a0_half;
      // chunk ch (columns 4 ch .. 4 ch + 3) of the row of type tt (0 value, 1..3 d/dq_{tt-1}) of query ql of meta
      // block b: a forward-mode tile interleaves the four rows of a query and stores hi / lo TF32 parts, an adjoint
      // group keeps fp32 blocks V, T1, T2, T3
      auto put = [&](int b, int ql, int tt, int ch, float4 v) {
        if (adj) {
          *reinterpret_cast<float4*>(a_hi + ((tt * WS_QG + b * WT + ql) * WS_LDA + 4 * ch) * 4) = v;
        } else {
          float4 hi, lo;
          um_split4(v, hi, lo);
          const int off = um_a_off(GRAD ? 4 * ql + tt : b * WT + ql, ch, K0);
          *reinterpret_cast<float4*>(a_hi + off) = hi;
          *reinterpret_cast<float4*>(a_lo + off) = lo;
        }
      };
      bool slot_free = false;
#pragma unroll 1
      for (int b = 0; b < BPT; ++b, ++j) {
        refill(j + PF);
        clk.lap(5);
        const int blk = i * BPT + b, ms = blk % MB;
        ws_wait_relaxed(um_smem_u32(bars + WSB_META_FULL + ms), (uint32_t)(blk / MB) & 1u);
        clk.lap(1);
        const float* mt = meta + ms * MSTRIDE;
        const int* m_li = reinterpret_cast<const int*>(mt + WsMeta::li);
        const float* m_w = mt + WsMeta::w;
#pragma unroll 1
        for (int p0 = gw * GU; p0 < NPASS; p0 += WS_GW * GU) {
          float4 fv[GU][KREG];
#pragma unroll
          for (int u = 0; u < GU; ++u) {
            const int ql = (p0 + u) * M::RPP + sub;
#pragma unroll
            for (int k = 0; k < KREG; ++k) {
              fv[u][k] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (k < K) {
                const int lif = m_li[k * WT + ql];
                if (lif >= 0) fv[u][k] = __ldg(f4 + (size_t)(lif & ~REMAP) * M::LPR);
              }
            }
          }
          clk.lap(2);
          if (!slot_free) {  // the loads are in flight while the previous tile in this slot is consumed by layer 0
            ws_wait_relaxed(um_smem_u32(bars + WSB_A0_EMPTY + slot), ((uint32_t)(i / WS_A0) & 1u) ^ 1u);
            slot_free = true;
            clk.lap(0);
          }
#pragma unroll
          for (int u = 0; u < GU; ++u) {
            const int ql = (p0 + u) * M::RPP + sub;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 tq[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) tq[j] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < KREG; ++k)
              if (k < K) {
                const float w = m_w[k * WT + ql];
                acc.x = fmaf(w, fv[u][k].x, acc.x);
                acc.y = fmaf(w, fv[u][k].y, acc.y);
                acc.z = fmaf(w, fv[u][k].z, acc.z);
                acc.w = fmaf(w, fv[u][k].w, acc.w);
                if (GRAD && k >= 1) {
                  const float4 d = make_float4(fv[u][k].x - fv[u][0].x, fv[u][k].y - fv[u][0].y, fv[u][k].z - fv[u][0].z,
                                               fv[u][k].w - fv[u][0].w);
#pragma unroll
                  for (int j = 0; j < 3; ++j) {
                    const float om = mt[WsMeta::om + (j * KREG + k) * WT + ql];  // 0 for invalid neighbours
                    tq[j].x = fmaf(om, d.x, tq[j].x);
                    tq[j].y = fmaf(om, d.y, tq[j].y);
                    tq[j].z = fmaf(om, d.z, tq[j].z);
                    tq[j].w = fmaf(om, d.w, tq[j].w);
                  }
                }
              }
            put(b, ql, 0, c4, acc);
            if (GRAD) {
#pragma unroll
              for (int j = 0; j < 3; ++j) put(b, ql, 1 + j, c4, tq[j]);
            }
          }
          clk.lap(3);
        }
        if (!slot_free) {  // warps without a pass in this block (F = 8) still write position rows
          ws_wait_relaxed(um_smem_u32(bars + WSB_A0_EMPTY + slot), ((uint32_t)(i / WS_A0) & 1u) ^ 1u);
          slot_free = true;
        }
        // the tile's original query indices, for the consumers' stores (the meta slot is refilled before they store)
        if ((b % WS_GW) == gw)
          reinterpret_cast<int*>(sm + lay.qidx)[(i % WS_QX) * QT + b * WT + lane] = reinterpret_cast<const int*>(mt + WsMeta::perm)[lane];
        // position part (columns F .. F+2) and zero padding of the rows: thread per row
        if (GRAD || (b % WS_GW) == gw) {
          const int row = gw * WT + lane;  // forward mode: row of the tile
          const int ql = adj ? lane : (GRAD ? row >> 2 : lane), tt = adj ? gw : (GRAD ? row & 3 : 0);
          const float* src3 = tt == 0 ? mt + WsMeta::xn : mt + WsMeta::P + (tt - 1) * 3 * WT;
          put(b, ql, tt, F / 4, make_float4(src3[ql], src3[WT + ql], src3[2 * WT + ql], tt == 0 ? 1.f : 0.f));  // column D: bias input
          // columns an adjoint group does not store (>= WS_LDA) are zero in the consumers' registers
          const int n_ch = adj ? (K0 < WS_LDA ? K0 : WS_LDA) / 4 : K0 / 4;
#pragma unroll
          for (int cz = F / 4 + 1; cz < K0 / 4; ++cz)
            if (cz < n_ch) put(b, ql, tt, cz, make_float4(0.f, 0.f, 0.f, 0.f));
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // A-tile writes -> visible to wgmma
        __syncwarp();
        if (lane == 0) ws_arrive(um_smem_u32(bars + WSB_META_EMPTY + ms));
        clk.lap(4);
      }
      if (lane == 0) ws_arrive(um_smem_u32(bars + WSB_A0_FULL + slot));
    }
  }
  clk.flush(warp, warp < WS_CW ? (adj ? WS_ROLE_CA : WS_ROLE_C) : WS_ROLE_G);
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
template <int FT>
static WsLayout plan_ws_layout(const pinb200_decoder_view& d, bool grad) {
  using DM = UmmaDims<FT>;
  WsLayout l{};
  int o = 0;
  auto take = [&](int bytes) {
    const int at = o;
    o += (bytes + 127) & ~127;
    return at;
  };
  const int w0 = 64 * DM::K0 * 4, w1 = 64 * 64 * 4;
  // d/dq of a single output channel takes the adjoint schedule; a colour Jacobian (out_dim 3) would need one adjoint
  // vector per channel and saves no MMA work, so it stays in forward mode
  l.adj = grad && d.out_dim == 1;
  l.w0_hi = take(w0);
  l.w0_lo = take(w0);
  if (d.n_hidden > 1) {
    l.w1_hi = take(w1);
    l.w1_lo = take(w1);
    if (l.adj) {
      l.w1t_hi = take(w1);
      l.w1t_lo = take(w1);
    }
  }
  l.b0 = take(64 * 4);
  l.b1 = take(64 * 4);
  l.wout = take(4 * 64 * 4);
  l.bout = take(16);
  l.a0_half = ((UM_ROWS / 8) * (DM::K0 / 4) * UM_A_LBO + 127) & ~127;
  l.a0_stride = l.adj ? 4 * WS_GBLK * 4 : 2 * l.a0_half;
  l.a0 = take(WS_A0 * l.a0_stride);
  l.qidx = take(WS_QX * 128 * 4);
  l.meta_stride = (grad ? WsMeta::floats_g : WsMeta::floats_ng) * 4;
  l.n_meta = grad ? 8 : 16;
  l.meta = take(l.n_meta * l.meta_stride);
  l.bars = take(WSB_COUNT * 8);
  l.total = o;
  return l;
}

template <int FT, bool GRAD, bool PROF>
static int launch_wsq(QueryParams& p, cudaStream_t stream) {
  const WsLayout lay = plan_ws_layout<FT>(p.dec, GRAD);
  const size_t smem_bytes = (size_t)lay.total;
  if (smem_bytes > 227 * 1024) {
    set_error("wsq_decode kernel needs %zu B shared memory (> 227 KB)", smem_bytes);
    return PINB200_ERR_UNSUPPORTED;
  }
  auto kern = wsq_decode_kernel<FT, GRAD, PROF>;
  if (const int rc = prepare_kernel((const void*)kern, "wsq_decode_kernel", smem_bytes)) return rc;
  p.qpt = WT;
  p.n_tiles = (int)((p.n + WT - 1) / WT);
  const int QT = lay.adj ? WS_QG : (GRAD ? 32 : 128);
  const long long n_tiles = (p.n + QT - 1) / QT;
  const int grid = (int)std::min<long long>(n_tiles, (long long)sm_count());
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(WS_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = p.pdl ? 1 : 0;
  const QueryParams pk = p;
  const cudaError_t le = cudaLaunchKernelEx(&cfg, kern, pk, lay);
  if (le != cudaSuccess) {
    set_error("wsq_decode_kernel launch: %s", cudaGetErrorString(le));
    return PINB200_ERR_CUDA;
  }
  return check_launch("wsq_decode_kernel");
}

bool wsq_supported(const pinb200_decoder_view& d, const pinb200_query_opts& o) {
  const int F = d.in_dim - 3;
  return o.weighted_first && d.hidden_dim == 64 && d.n_hidden >= 1 && d.n_hidden <= 2 && (F == 8 || F == 16 || F == 32) &&
         o.nn_k <= KREG;
}

int dispatch_wsq(QueryParams& p, cudaStream_t stream) {
  const bool grad = p.opts.need_grad != 0;
  switch (p.dec.in_dim - 3) {
    case 8: return grad ? launch_wsq<8, true, false>(p, stream) : launch_wsq<8, false, false>(p, stream);
    case 16: return grad ? launch_wsq<16, true, false>(p, stream) : launch_wsq<16, false, false>(p, stream);
    case 32:
      if (g_ws_profile) return grad ? launch_wsq<32, true, true>(p, stream) : launch_wsq<32, false, true>(p, stream);
      return grad ? launch_wsq<32, true, false>(p, stream) : launch_wsq<32, false, false>(p, stream);
    default: break;
  }
  set_error("wsq_decode: feature_dim %d unsupported", p.dec.in_dim - 3);
  return PINB200_ERR_UNSUPPORTED;
}

void wsq_set_profile(int on) { g_ws_profile = on; }

// copies the cycle counters of the last profiled launch: [WS_PROF_CTAS CTAs][16 warps][8 slots] uint64
int wsq_read_profile(unsigned long long* host_out, int64_t count) {
  const int64_t have = (int64_t)(sizeof(g_ws_prof) / sizeof(unsigned long long));
  if (count < have) {
    set_error("ws_profile: buffer of %lld < %lld counters", (long long)count, (long long)have);
    return PINB200_ERR_BAD_ARG;
  }
  const cudaError_t e = cudaMemcpyFromSymbol(host_out, g_ws_prof, sizeof(g_ws_prof));
  if (e != cudaSuccess) {
    set_error("ws_profile: %s", cudaGetErrorString(e));
    return PINB200_ERR_CUDA;
  }
  return PINB200_OK;
}

}  // namespace pinb
