// Device-side pieces of K1 shared by the translation units of the query path (query.cu, wsq.cu): launch parameters,
// the thread-per-query neighbour search over the probe index, feature-row movement, phase A1 of a 32-query tile.
#pragma once
#include <algorithm>
#include <string>

#include "mlp_chain.cuh"

namespace pinb {

constexpr int WT = 32;   // queries (= threads) per warp tile
constexpr int WPB = 12;  // warps per CTA (one CTA per SM): 12 x 32 threads x 168 registers fill the register file
constexpr int REMAP = PINB200_REC_REMAP;

struct QueryLayout {  // float offsets into dynamic smem
  WarpDecSmem dec;
  int delta, warp0, n_warps, total;  // CTA-shared part, then n_warps per-warp blocks (WarpLay<FT>)
};

// Per-warp tile state, compile-time offsets (floats) so that every access is base + immediate.
template <int FT>
struct WarpLay {
  static constexpr int KP0 = dec_in_pad(FT);
  static constexpr int LDX = ld8mod32(KP0);
  static constexpr int x = 0;                      // [32][LDX] decoder input rows / input gradient
  static constexpr int stash = x + WT * LDX;       // Stash block (see a1_tile)
  static constexpr int a = stash + 1536;           // [K][32] <g_xbar, f_k>
  static constexpr int out = a + WT * 8;           // [32][<=4] decoder outputs
  static constexpr int dv = out + WT * 4;          // [32][4] d out / d pre-activation
  static constexpr int mask = dv + WT * 4;         // [<=4 layers][32] 64-bit ReLU masks
  static constexpr int stride = mask + 2 * WT * PINB200_MAX_HIDDEN_LAYERS;
};

struct QueryParams {
  pinb200_map_view map;
  pinb200_decoder_view dec;
  pinb200_query_opts opts;
  pinb200_query_out out;
  const float* query_xyz;
  const int32_t* query_ts;
  const float* feat;  // feature table decoded by `dec` (geo or colour)
  long long n;
  int use_saved_knn;  // 1: take kNN from out.knn_idx / knn_gidx / knn_dist2 (decode-only launch, e.g. colour head)
  int is_color;       // outputs go to out.color / out.color_grad instead of sdf / grad
  int n_tiles;
  int qpt;  // queries per warp tile
  // split pipeline: [n_tiles][Stash::floats] (decode on query_kernel) or [n_tiles][StashS::floats] (decode on
  // wsq_decode_kernel) workspace written by search_kernel, read by the decode launch
  float* stash;
  float* seeds;  // split pipeline with d/dq on the warp-specialised decode: [n_tiles][Seeds::floats] forward-mode seeds
  int pdl;       // host only: this decode launch directly follows its search launch (programmatic dependent launch)
  QueryLayout lay;
  // search launch with spatially sorted queries (StashS blocks only): sorted[i] = {x, y, z, original index} of the
  // i-th query in sorted order (the query untransformed); the search launch works on sorted[32 st + lane].  nullptr:
  // queries in the caller's order.
  const float4* sorted;
};

// squared distance with the reference's arithmetic: sum((p - q)^2) in fp32, no contraction (:990-994)
__device__ __forceinline__ float dist2_rn(float px, float py, float pz, float qx, float qy, float qz) {
  const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy), dz = __fsub_rn(pz, qz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ uint32_t probe_slot(uint32_t r0, uint32_t delta, uint32_t B) {
  uint32_t s = r0 + delta;
  if (s >= B) s -= B;
  return s;
}

// ---------------------------------------------------------------------------
// A1: thread-per-query search over the probe index (pinb200_map_view.probe_words / probe_rec).  Returns nn_count;
// T holds the 8 best (distance, record rank) pairs, ascending.  Per SUPER probes: one round of 8-byte word loads
// (occupancy + rank), then the records of the occupied slots 16 at a time (two sorting-network batches per round
// trip).  The odd last probe of an 8n+1 neighbourhood (33, 57, 81) is issued with the first round and inserted last.
// ---------------------------------------------------------------------------
constexpr int PROBE_SUPER = 32;
constexpr int PROBE_ROUND = 16;

// Optional cycle accounting of the search launch (a library built with -DPINB200_SEARCH_PROFILE=1): per warp, clock deltas of
// the phases of a1_tile summed over the warp's tiles, for the first SEARCH_PROF_WARPS warps of the grid; read back with
// pinb200_debug_read("search_profile", ...).  A stamp is taken when the warp issues the phase's last instruction, so
// a load's latency counts in the phase that first uses its result.  Slots: the phases SP_HASH .. SP_OUT, the number of
// distinct base slots (map voxels, up to hash collisions) of each tile summed over the warp's tiles, its tiles.
enum SearchPhase { SP_HASH = 0, SP_WORDS, SP_SELECT, SP_WINNERS, SP_STASH, SP_OUT, SP_VOXELS, SP_TILES };
constexpr int SEARCH_PROF_SLOTS = 8;
constexpr int SEARCH_PROF_WARPS = 132 * 4 * 4;  // every warp of a full-size search grid on an H100 SXM
template <bool PROF>
struct SearchClock {  // PROF = false: no code at all
  unsigned int acc[SEARCH_PROF_SLOTS];
  unsigned int last;
  __device__ __forceinline__ void start() {
    if (PROF) {
#pragma unroll
      for (int i = 0; i < SEARCH_PROF_SLOTS; ++i) acc[i] = 0u;
    }
  }
  __device__ __forceinline__ void tile() {
    if (PROF) last = (unsigned int)clock();
  }
  __device__ __forceinline__ void lap(int slot) {
    if (PROF) {
      const unsigned int now = (unsigned int)clock();
      acc[slot] += now - last;
      last = now;
    }
  }
  __device__ __forceinline__ void add(int slot, unsigned int v) {
    if (PROF) acc[slot] += v;
  }
  __device__ __forceinline__ void flush(unsigned long long* dst) {
    if (PROF) {
#pragma unroll
      for (int i = 0; i < SEARCH_PROF_SLOTS; ++i) dst[i] = acc[i];
    }
  }
};

__device__ __forceinline__ int probe_rank(uint2 w, uint32_t slot) {
  const uint32_t b = slot & 31u;
  return ((w.x >> b) & 1u) ? (int)(w.y + __popc(w.x & ((1u << b) - 1u))) : -1;
}

// SUPER: probes per word round (a multiple of PROBE_ROUND).  The batches of 8 and the order they are merged in do not
// depend on it, so neither does the result: a smaller SUPER only holds fewer word results in registers at a time.
template <int SUPER, bool PROF>
__device__ __forceinline__ int knn_search_lane(const pinb200_map_view& m, const uint32_t* s_delta, bool live, uint32_t r0,
                                               float qx, float qy, float qz, KnnTop& T, SearchClock<PROF>& clk) {
  knn_top_init(T);
  int count = 0;
  const uint32_t B = (uint32_t)m.buffer_size;
  const int C = m.n_probe;
  const uint2* __restrict__ words = reinterpret_cast<const uint2*>(m.probe_words);
  const float4* __restrict__ rec4 = reinterpret_cast<const float4*>(m.probe_rec);
  const float inf = __int_as_float(0x7f800000);
  const float maxd2 = m.max_valid_dist2;
  const bool odd = C > KREG && (C & (KREG - 1)) == 1;
  const int Cb = odd ? C - 1 : C;
  int rk_last = -1;
  if (odd && live) {
    const uint32_t slot = probe_slot(r0, s_delta[C - 1], B);
    rk_last = probe_rank(__ldg(words + (slot >> 5)), slot);
  }
#pragma unroll 1
  for (int c0 = 0; c0 < Cb; c0 += SUPER) {
    const int nb = Cb - c0;
    int rk[SUPER];
    {
      uint32_t slot[SUPER];
      uint2 wv[SUPER];
#pragma unroll
      for (int j = 0; j < SUPER; ++j) {
        slot[j] = 0u;
        wv[j] = make_uint2(0u, 0u);
        if (live && j < nb) {
          slot[j] = probe_slot(r0, s_delta[c0 + j], B);
          wv[j] = __ldg(words + (slot[j] >> 5));
        }
      }
#pragma unroll
      for (int j = 0; j < SUPER; ++j) rk[j] = probe_rank(wv[j], slot[j]);
    }
    clk.lap(SP_WORDS);
#pragma unroll
    for (int h = 0; h < SUPER / PROBE_ROUND; ++h) {
      if (h * PROBE_ROUND < nb) {
        float4 r[PROBE_ROUND];
#pragma unroll
        for (int j = 0; j < PROBE_ROUND; ++j) {
          r[j] = make_float4(inf, inf, inf, 0.f);
          if (rk[h * PROBE_ROUND + j] >= 0) r[j] = __ldg(rec4 + rk[h * PROBE_ROUND + j]);
        }
#pragma unroll
        for (int b = 0; b < PROBE_ROUND / KREG; ++b) {
          if (h * PROBE_ROUND + b * KREG < nb) {
            float d[KREG];
            int pc[KREG];
#pragma unroll
            for (int j = 0; j < KREG; ++j) {
              const float4 rr = r[b * KREG + j];
              const float dd = dist2_rn(rr.x, rr.y, rr.z, qx, qy, qz);
              const bool ok = dd <= maxd2;  // unoccupied probes carry +inf; dist2 > max is a hash collision (:999)
              d[j] = ok ? dd : SEL_INVALID_D2;
              pc[j] = ok ? rk[h * PROBE_ROUND + b * KREG + j] : -1;
              count += ok ? 1 : 0;
            }
            if (c0 == 0 && h == 0 && b == 0)
              knn_top_first8(T, d, pc);
            else
              knn_top_merge8(T, d, pc);
          }
        }
      }
    }
  }
  if (odd) {
    float4 rl = make_float4(inf, inf, inf, 0.f);
    if (rk_last >= 0) rl = __ldg(rec4 + rk_last);
    const float dd = dist2_rn(rl.x, rl.y, rl.z, qx, qy, qz);
    const bool ok = dd <= maxd2;
    count += ok ? 1 : 0;
    knn_top_insert1(T, ok ? dd : SEL_INVALID_D2, ok ? rk_last : -1);
  }
  clk.lap(SP_SELECT);
  return count;
}

// neighbour vector n_k = q - p_k in the frame of the neural point (model/neural_points.py:632-651) from the stashed
// global difference; `lif` = local id | REMAP flag.  Also returns the point quaternion when after_pgo.
__device__ __forceinline__ void neighbour_vec(const pinb200_map_view& m, int lif, float dx, float dy, float dz, float qx,
                                              float qy, float qz, float& nx, float& ny, float& nz, float4& quat) {
  nx = dx;
  ny = dy;
  nz = dz;
  const int li = lif & ~REMAP;
  if (lif & REMAP) {  // the local id does not name the point the distance was measured to (reference quirk Q1)
    const float* pp = m.nb_points + 3 * (size_t)li;
    nx = __fsub_rn(qx, __ldg(pp));
    ny = __fsub_rn(qy, __ldg(pp + 1));
    nz = __fsub_rn(qz, __ldg(pp + 2));
  }
  quat = make_float4(1.f, 0.f, 0.f, 0.f);
  if (m.after_pgo) {
    quat = __ldg(reinterpret_cast<const float4*>(m.nb_orient) + li);
    quat_rotate_passive(quat.x, quat.y, quat.z, quat.w, nx, ny, nz, nx, ny, nz);
  }
}

// ---------------------------------------------------------------------------
// A2 / C1: feature-row movement, FT/4 lanes per row (a lane owns 4 consecutive columns of its row)
// ---------------------------------------------------------------------------
template <int FT>
struct RowMap {
  static constexpr int LPR = FT / 4;    // lanes per feature row
  static constexpr int RPP = 32 / LPR;  // rows (or queries) per pass
  static constexpr int U = RPP >= 32 ? 1 : (RPP >= 16 ? 2 : 4);  // passes in flight (<= 32 rows of 16-byte loads per lane)
};

// weighted_first: x[ql][0..F) = sum_k w_k f_k[.]  for the queries of the warp tile
template <int FT, int LDX>
__device__ __forceinline__ void gather_weighted(const float* __restrict__ feat, int K, int WQ, const int* s_li,
                                                const float* s_w, int lane, float* s_x) {
  using M = RowMap<FT>;
  const int sub = lane / M::LPR, c4 = lane % M::LPR;
  const float4* __restrict__ f4 = reinterpret_cast<const float4*>(feat) + c4;
#pragma unroll 1
  for (int q0 = 0; q0 < WQ; q0 += M::U * M::RPP) {
    float4 v[M::U][KREG];
#pragma unroll
    for (int u = 0; u < M::U; ++u) {
      const int ql = q0 + u * M::RPP + sub;  // < WT: WQ <= WT and U*RPP divides WT
#pragma unroll
      for (int k = 0; k < KREG; ++k) {
        v[u][k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < K) {
          const int lif = s_li[k * WT + ql];
          if (lif >= 0) v[u][k] = __ldg(f4 + (size_t)(lif & ~REMAP) * M::LPR);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < M::U; ++u) {
      const int ql = q0 + u * M::RPP + sub;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < KREG; ++k)
        if (k < K) {
          const float w = s_w[k * WT + ql];  // 0 for invalid neighbours
          acc.x = fmaf(w, v[u][k].x, acc.x);
          acc.y = fmaf(w, v[u][k].y, acc.y);
          acc.z = fmaf(w, v[u][k].z, acc.z);
          acc.w = fmaf(w, v[u][k].w, acc.w);
        }
      *reinterpret_cast<float4*>(s_x + ql * LDX + 4 * c4) = acc;
    }
  }
}

// decode-every-neighbour: x[ql*K + k][0..F) = f_k (0 if invalid) for the `qpt` queries of the row tile starting at sq0
template <int FT, int LDX>
__device__ __forceinline__ void gather_rows(const float* __restrict__ feat, int K, int used_rows, int sq0, const int* s_li,
                                            int lane, float* s_x) {
  using M = RowMap<FT>;
  const int sub = lane / M::LPR, c4 = lane % M::LPR;
#pragma unroll 1
  for (int r0 = 0; r0 < WT; r0 += M::U * M::RPP) {
    float4 v[M::U];
#pragma unroll
    for (int u = 0; u < M::U; ++u) {
      const int row = r0 + u * M::RPP + sub;
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < used_rows) {
        const int ql = row / K, k = row - ql * K;
        const int lif = s_li[k * WT + sq0 + ql];
        if (lif >= 0) v[u] = __ldg(reinterpret_cast<const float4*>(feat + (size_t)(lif & ~REMAP) * FT) + c4);
      }
    }
#pragma unroll
    for (int u = 0; u < M::U; ++u) {
      const int row = r0 + u * M::RPP + sub;
      if (row < WT) *reinterpret_cast<float4*>(s_x + row * LDX + 4 * c4) = v[u];  // unused rows stay finite (zero)
    }
  }
}

// Sum 8 per-lane values over groups of LPR consecutive lanes.  Halving exchange: every step a lane keeps half of its
// values and adds the partner's partial of those (7 shuffles for LPR = 8 instead of 24).  On return v[0..n_out) are
// group totals; `first` is the neighbour index k of v[0] (the lane's values are k = first .. first + n_out - 1).
template <int LPR>
__device__ __forceinline__ void group_reduce8(float (&v)[KREG], int lane, int& first, int& n_out) {
  first = 0;
  int n = KREG;
#pragma unroll
  for (int o = LPR / 2; o >= 1; o >>= 1) {
    if (n > 1) {
      const bool hi = (lane & o) != 0;
      const int h = n / 2;
#pragma unroll
      for (int i = 0; i < KREG / 2; ++i)
        if (i < h) {
          const float send = hi ? v[i] : v[i + h];
          const float keep = hi ? v[i + h] : v[i];
          v[i] = keep + __shfl_xor_sync(FULL, send, o);
        }
      if (hi) first += h;
      n = h;
    } else {
      v[0] += __shfl_xor_sync(FULL, v[0], o);
    }
  }
  n_out = n;
}

// C1: a[k][ql] = <g_xbar[ql][0..F), f_k>
template <int FT, int LDX>
__device__ __forceinline__ void feature_dots(const float* __restrict__ feat, int K, int WQ, const int* s_li, int lane,
                                             const float* s_x, float* s_a) {
  using M = RowMap<FT>;
  const int sub = lane / M::LPR, c4 = lane % M::LPR;
  const float4* __restrict__ f4 = reinterpret_cast<const float4*>(feat) + c4;
#pragma unroll 1
  for (int q0 = 0; q0 < WQ; q0 += M::U * M::RPP) {
    float4 v[M::U][KREG];
#pragma unroll
    for (int u = 0; u < M::U; ++u) {
      const int ql = q0 + u * M::RPP + sub;
#pragma unroll
      for (int k = 0; k < KREG; ++k) {
        v[u][k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < K) {
          const int lif = s_li[k * WT + ql];
          if (lif >= 0) v[u][k] = __ldg(f4 + (size_t)(lif & ~REMAP) * M::LPR);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < M::U; ++u) {
      const int ql = q0 + u * M::RPP + sub;
      const float4 g4 = *reinterpret_cast<const float4*>(s_x + ql * LDX + 4 * c4);
      float part[KREG];
#pragma unroll
      for (int k = 0; k < KREG; ++k)
        part[k] = fmaf(g4.w, v[u][k].w, fmaf(g4.z, v[u][k].z, fmaf(g4.y, v[u][k].y, g4.x * v[u][k].x)));
      int first, n_out;
      group_reduce8<M::LPR>(part, lane, first, n_out);
      // after the exchange steps the lanes of a group hold disjoint k ranges; lanes that only took part in plain
      // butterfly steps (LPR > 8) hold duplicates: the lowest lane of each duplicate set writes
      const bool writer = M::LPR <= KREG ? true : (lane % (M::LPR / KREG)) == 0;
      if (writer)
#pragma unroll
        for (int i = 0; i < KREG; ++i)
          if (i < n_out && first + i < K) s_a[(first + i) * WT + ql] = part[i];
    }
  }
}

// ---------------------------------------------------------------------------
// Phase A1 of one 32-query tile: search, IDW weights, certainty, training-mode scatters, kNN outputs, and the "stash"
// every later phase works from.  The stash is one block of STASH_FLOATS floats in [field][k][lane] order (conflict
// free columns in shared memory, fully coalesced rows in global memory): the fused kernel keeps it in the warp's
// shared memory, the split pipeline (search_kernel -> decode) writes it to the workspace.
// ---------------------------------------------------------------------------
struct Stash {
  static constexpr int li = 0;              // [K][32] neighbour id | REMAP (-1 invalid)
  static constexpr int w = li + WT * 8;     // [K][32] IDW weight
  static constexpr int dx = w + WT * 8;     // [K][32] q - p_k (the point dist2 was measured to)
  static constexpr int dy = dx + WT * 8;
  static constexpr int dz = dy + WT * 8;
  static constexpr int q = dz + WT * 8;     // [3][32] query
  static constexpr int usum = q + WT * 3;   // [32] sum of the unnormalised weights
  static constexpr int nn = usum + WT;      // [32] nn_count
  static constexpr int pos = nn + WT;       // [3][32] sum_k w_k n_k
  static constexpr int floats = pos + WT * 3;
};
static_assert(Stash::floats % 4 == 0, "stash block is copied with 16-byte accesses");
// The block read by the warp-specialised decode (wsq.cu) holds only what that decode reads, in the order of its meta
// block (one bulk copy): neighbour ids, IDW weights, position part, and the original index of every query of the
// tile (-1 past the end of the batch).
struct StashS {
  static constexpr int li = 0;
  static constexpr int w = li + WT * 8;
  static constexpr int pos = w + WT * 8;
  static constexpr int perm = pos + WT * 3;
  static constexpr int floats = perm + WT;
};
static_assert(StashS::li == Stash::li && StashS::w == Stash::w && StashS::floats % 4 == 0, "li | w lead both layouts");

// Forward-mode seeds of d sdf / d q for one query (wsq.cu pushes them through the decoder as tangent rows):
//   w_k = u_k / sum u,  u_k = 1 / (d_k^2 + eps)  =>  omega_kj = d w_k / d q_j = w_k (c_k d_kj - sum_m w_m c_m d_mj),
//   c_k = -2 u_k,  d_k = q - p_k (the point the distance was measured to);   x_n = sum_k w_k n_k  =>
//   P_ji = d (x_n)_i / d q_j = sum_k omega_kj (n_k - n_0)_i + sum_k w_k (R_k e_j)_i
// (sum_k omega_kj = 0: the shift by the nearest neighbour keeps the sums cancellation-free when neighbours coincide;
// R_k = I before loop closure).  Block layout [field][k][lane]: omega [3 j][8 k][32], P [3 j][3 i][32].
// The closed forms are restated in oracle/pin_oracle.py: idw_tangent_seeds and pinned against autograd on the CPU
// (tests/test_oracle_golden.py::test_forward_mode_seeds_equal_autograd).
struct Seeds {
  static constexpr int om = 0;
  static constexpr int P = om + WT * 24;
  static constexpr int floats = P + WT * 9;
};
__device__ __forceinline__ void tangent_seeds(const pinb200_map_view& m, int K, const int (&lif)[KREG], const float (&w)[KREG],
                                              const float (&px)[KREG], const float (&py)[KREG], const float (&pz)[KREG], float qx,
                                              float qy, float qz, float usum, int nn, float* sd, int lane) {
  float c[KREG], S0 = 0.f, S1 = 0.f, S2 = 0.f;
#pragma unroll
  for (int k = 0; k < KREG; ++k) {
    const bool v = k < K && lif[k] >= 0;
    c[k] = (v && nn > 0) ? -2.f * (w[k] * usum) : 0.f;
    const float wc = v ? w[k] * c[k] : 0.f;
    S0 = fmaf(wc, __fsub_rn(qx, px[k]), S0);
    S1 = fmaf(wc, __fsub_rn(qy, py[k]), S1);
    S2 = fmaf(wc, __fsub_rn(qz, pz[k]), S2);
  }
  float P[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  float n0x = 0.f, n0y = 0.f, n0z = 0.f;
#pragma unroll
  for (int k = 0; k < KREG; ++k) {
    const bool v = k < K && lif[k] >= 0;
    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
    if (v) {
      const float dx = __fsub_rn(qx, px[k]), dy = __fsub_rn(qy, py[k]), dz = __fsub_rn(qz, pz[k]);
      o0 = w[k] * (c[k] * dx - S0);
      o1 = w[k] * (c[k] * dy - S1);
      o2 = w[k] * (c[k] * dz - S2);
      float nx, ny, nz;
      float4 quat;
      neighbour_vec(m, lif[k], dx, dy, dz, qx, qy, qz, nx, ny, nz, quat);
      if (k == 0) {
        n0x = nx;
        n0y = ny;
        n0z = nz;
      }
      const float ex = nx - n0x, ey = ny - n0y, ez = nz - n0z;
      P[0][0] = fmaf(o0, ex, P[0][0]);
      P[0][1] = fmaf(o0, ey, P[0][1]);
      P[0][2] = fmaf(o0, ez, P[0][2]);
      P[1][0] = fmaf(o1, ex, P[1][0]);
      P[1][1] = fmaf(o1, ey, P[1][1]);
      P[1][2] = fmaf(o1, ez, P[1][2]);
      P[2][0] = fmaf(o2, ex, P[2][0]);
      P[2][1] = fmaf(o2, ey, P[2][1]);
      P[2][2] = fmaf(o2, ez, P[2][2]);
      if (m.after_pgo) {  // column j of the point's (passive) rotation
        float r0, r1, r2;
        quat_rotate_passive(quat.x, quat.y, quat.z, quat.w, 1.f, 0.f, 0.f, r0, r1, r2);
        P[0][0] = fmaf(w[k], r0, P[0][0]);
        P[0][1] = fmaf(w[k], r1, P[0][1]);
        P[0][2] = fmaf(w[k], r2, P[0][2]);
        quat_rotate_passive(quat.x, quat.y, quat.z, quat.w, 0.f, 1.f, 0.f, r0, r1, r2);
        P[1][0] = fmaf(w[k], r0, P[1][0]);
        P[1][1] = fmaf(w[k], r1, P[1][1]);
        P[1][2] = fmaf(w[k], r2, P[1][2]);
        quat_rotate_passive(quat.x, quat.y, quat.z, quat.w, 0.f, 0.f, 1.f, r0, r1, r2);
        P[2][0] = fmaf(w[k], r0, P[2][0]);
        P[2][1] = fmaf(w[k], r1, P[2][1]);
        P[2][2] = fmaf(w[k], r2, P[2][2]);
      } else {
        P[0][0] += w[k];
        P[1][1] += w[k];
        P[2][2] += w[k];
      }
    }
    sd[Seeds::om + (0 * KREG + k) * WT + lane] = o0;
    sd[Seeds::om + (1 * KREG + k) * WT + lane] = o1;
    sd[Seeds::om + (2 * KREG + k) * WT + lane] = o2;
  }
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 3; ++i) sd[Seeds::P + (j * 3 + i) * WT + lane] = P[j][i];
}

// COMPACT: `stash` is a StashS block; with p.sorted, lane `lane` works on the query of record p.sorted[q0s + lane]
// (per-query outputs go to its index).  The seeds stay in tile order.
template <bool SEEDS = false, bool COMPACT = false, bool PROF = false, int SUPER = PROBE_SUPER>
__device__ __forceinline__ void a1_tile(const QueryParams& p, const uint32_t* s_delta, long long q0s, int WQ, int lane,
                                        float* stash, SearchClock<PROF>& clk) {
  const pinb200_map_view& m = p.map;
  const int K = p.opts.nn_k;
  int* s_li = reinterpret_cast<int*>(stash + Stash::li);
  float* s_w = stash + Stash::w;
  float* s_dx = stash + Stash::dx;
  float* s_dy = stash + Stash::dy;
  float* s_dz = stash + Stash::dz;
  float* s_q = stash + Stash::q;
  float* s_usum = stash + Stash::usum;
  int* s_nn = reinterpret_cast<int*>(stash + Stash::nn);
  float* s_pos = stash + (COMPACT ? StashS::pos : Stash::pos);
  const bool live = lane < WQ && q0s + lane < p.n;
  long long qi = q0s + lane;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (COMPACT) {
    if (!live) {
      qi = -1;
    } else if (p.sorted) {  // one coalesced 16-byte load: the query and its index
      const float4 r = __ldg(p.sorted + q0s + lane);
      qx = r.x;
      qy = r.y;
      qz = r.z;
      qi = __float_as_int(r.w);
    }
    reinterpret_cast<int*>(stash + StashS::perm)[lane] = (int)qi;
  }
  if (live) {
    if (!COMPACT || !p.sorted) {
      qx = __ldg(p.query_xyz + 3 * qi + 0);
      qy = __ldg(p.query_xyz + 3 * qi + 1);
      qz = __ldg(p.query_xyz + 3 * qi + 2);
    }
    if (p.opts.transform) {  // q = T p in fp32 (utils/tools.py:534-553)
      const double* T = p.opts.transform;
      const float x = fmaf(qz, (float)T[2], fmaf(qy, (float)T[1], qx * (float)T[0])) + (float)T[3];
      const float y = fmaf(qz, (float)T[6], fmaf(qy, (float)T[5], qx * (float)T[4])) + (float)T[7];
      const float z = fmaf(qz, (float)T[10], fmaf(qy, (float)T[9], qx * (float)T[8])) + (float)T[11];
      qx = x;
      qy = y;
      qz = z;
    }
  }
  // the K nearest: squared distance, position of the (global) point it was measured to, id | REMAP, global id
  float d2[KREG], px[KREG], py[KREG], pz[KREG];
  int lif[KREG], gid[KREG];
  int cnt = 0;
#pragma unroll
  for (int k = 0; k < KREG; ++k) {
    d2[k] = INVALID_D2;
    px[k] = py[k] = pz[k] = 0.f;
    lif[k] = gid[k] = -1;
  }
  if (p.use_saved_knn) {
    if (live) {
      cnt = __ldg(p.out.nn_count + qi);
#pragma unroll
      for (int k = 0; k < KREG; ++k)
        if (k < K) {
          const int li = __ldg(p.out.knn_idx + qi * K + k);
          if (li >= 0) {
            gid[k] = __ldg(p.out.knn_gidx + qi * K + k);
            d2[k] = __ldg(p.out.knn_dist2 + qi * K + k);
            const float* pg = m.points + 3 * (size_t)gid[k];
            const float* pl = m.nb_points + 3 * (size_t)li;
            px[k] = __ldg(pg);
            py[k] = __ldg(pg + 1);
            pz[k] = __ldg(pg + 2);
            const bool same = __ldg(pl) == px[k] && __ldg(pl + 1) == py[k] && __ldg(pl + 2) == pz[k];
            lif[k] = same ? li : (li | REMAP);
          }
        }
    }
  } else {
    const uint32_t r0 = base_slot(m, qx, qy, qz);
    if (PROF) {  // lanes of a voxel share r0 (base slots are < 2^31)
      const uint32_t same = __match_any_sync(FULL, live ? r0 : 0xffffffffu);
      clk.add(SP_VOXELS, __popc(__ballot_sync(FULL, live && __ffs(same) - 1 == lane)));
    }
    clk.lap(SP_HASH);
    KnnTop T;
    cnt = knn_search_lane<SUPER>(m, s_delta, live, r0, qx, qy, qz, T, clk);
    // re-read the winners (the probe loop kept only distance + record rank through the sorting networks)
    const float4* __restrict__ rec4 = reinterpret_cast<const float4*>(m.probe_rec);
    float4 r[KREG];
#pragma unroll
    for (int k = 0; k < KREG; ++k) {
      r[k] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
      if (k < K && T.p[k] >= 0) {
        r[k] = __ldg(rec4 + T.p[k]);
        if (p.out.knn_gidx) gid[k] = __ldg(m.probe_gid + T.p[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < KREG; ++k)
      if (k < K && T.p[k] >= 0) {
        d2[k] = T.d[k];
        px[k] = r[k].x;
        py[k] = r[k].y;
        pz[k] = r[k].z;
        lif[k] = __float_as_int(r[k].w);
      }
  }
  // normalised inverse-distance weights, summed in neighbour order (model/neural_points.py:665-683)
  float u[KREG], w[KREG], usum = 0.f;
#pragma unroll
  for (int k = 0; k < KREG; ++k) {
    const bool v = k < K && lif[k] >= 0;
    u[k] = k < K ? (cnt == 0 ? IDW_EPS : (v ? __frcp_rn(d2[k] + IDW_EPS) : 0.f)) : 0.f;
    usum += u[k];
  }
#pragma unroll
  for (int k = 0; k < KREG; ++k) w[k] = (k < K && lif[k] >= 0) ? __fdiv_rn(u[k], usum) : 0.f;
  // neighbour vectors n_k = q - p_k (rotated into the point frame after PGO), certainty (:631-651)
  float sx = 0.f, sy = 0.f, sz = 0.f, qc = 0.f;
  const bool want_cert = !p.is_color && (p.out.certainty != nullptr);
#pragma unroll
  for (int k = 0; k < KREG; ++k) {
    float dx = 0.f, dy = 0.f, dz = 0.f;
    if (k < K && lif[k] >= 0) {
      dx = __fsub_rn(qx, px[k]);
      dy = __fsub_rn(qy, py[k]);
      dz = __fsub_rn(qz, pz[k]);
      {
        float nx, ny, nz;
        float4 quat;
        neighbour_vec(m, lif[k], dx, dy, dz, qx, qy, qz, nx, ny, nz, quat);
        sx = fmaf(w[k], nx, sx);
        sy = fmaf(w[k], ny, sy);
        sz = fmaf(w[k], nz, sz);
        if (want_cert) qc = fmaf(w[k], m.certainty[lif[k] & ~REMAP], qc);
      }
    }
    if (k < K) {
      s_li[k * WT + lane] = lif[k];
      s_w[k * WT + lane] = w[k];
      if (!COMPACT) {
        s_dx[k * WT + lane] = dx;
        s_dy[k * WT + lane] = dy;
        s_dz[k * WT + lane] = dz;
      }
    }
  }
  if (!COMPACT) {
    s_nn[lane] = cnt;
    s_usum[lane] = usum;
    s_q[0 * WT + lane] = qx;
    s_q[1 * WT + lane] = qy;
    s_q[2 * WT + lane] = qz;
  }
  clk.lap(SP_WINNERS);
  s_pos[0 * WT + lane] = sx;  // position part of the IDW-averaged decoder input (weighted_first)
  s_pos[1 * WT + lane] = sy;
  s_pos[2 * WT + lane] = sz;
  if (SEEDS) tangent_seeds(m, K, lif, w, px, py, pz, qx, qy, qz, usum, cnt, p.seeds + (size_t)(q0s / WT) * Seeds::floats, lane);
  clk.lap(SP_STASH);
  if (live && !p.is_color) {
    if (p.opts.training_mode && (p.opts.training_rows <= 0 || qi < p.opts.training_rows)) {
      // certainty scatter_add / ts amax (:685-710); invalid entries add 0 / max with 0 in the reference
      const int ts = (m.ts_update && p.query_ts) ? __ldg(p.query_ts + qi) : 0;
#pragma unroll
      for (int k = 0; k < KREG; ++k)
        if (k < K && lif[k] >= 0) {
          atomicAdd(m.certainty + (lif[k] & ~REMAP), w[k]);
          if (m.ts_update && p.query_ts) atomicMax(m.ts_update + (lif[k] & ~REMAP), ts);
        }
    }
    if (p.out.certainty) p.out.certainty[qi] = qc;
    if (!p.use_saved_knn) {
      if (p.out.nn_count) p.out.nn_count[qi] = cnt;
#pragma unroll
      for (int k = 0; k < KREG; ++k)
        if (k < K) {
          if (p.out.knn_idx) p.out.knn_idx[qi * K + k] = lif[k] < 0 ? -1 : (lif[k] & ~REMAP);
          if (p.out.knn_gidx) p.out.knn_gidx[qi * K + k] = gid[k];
          if (p.out.knn_dist2) p.out.knn_dist2[qi * K + k] = d2[k];
          if (p.out.knn_weight) p.out.knn_weight[qi * K + k] = w[k];
        }
    }
    if (p.out.xyz) {
      p.out.xyz[3 * qi + 0] = qx;
      p.out.xyz[3 * qi + 1] = qy;
      p.out.xyz[3 * qi + 2] = qz;
    }
  }
  clk.lap(SP_OUT);
}


struct QueryParams;
// wsq.cu: the warp-specialised decode covers weighted_first maps with a 1- or 2-layer 64-wide decoder and F in {8, 16, 32}
bool wsq_supported(const pinb200_decoder_view& d, const pinb200_query_opts& o);
int dispatch_wsq(QueryParams& p, cudaStream_t stream);
void wsq_set_profile(int on);
int wsq_read_profile(unsigned long long* host_out, int64_t count);
int sort_queries(const float* xyz, const double* transform, long long n, float resolution, void* scratch,
                 size_t scratch_bytes, const float4** sorted, cudaStream_t stream);  // query_sort.cu

}  // namespace pinb
