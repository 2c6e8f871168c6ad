// Thread-per-row tiny-MLP building blocks shared by the query (K1) and the
// training-backward (K2) kernels.
//
// A CTA works on a tile of TILE=128 rows.  Activations live in shared memory
// TRANSPOSED: act[feature][row] with leading dimension ACT_LD=129, so that
//   * a thread reading/writing its own row (column `tid` of the tile) is
//     bank-conflict free, and
//   * a warp writing one row's features across lanes is conflict free too.
// Each thread owns one row: it streams the layer input from its smem column and
// keeps the H (=64) outputs in registers; weights are read from shared memory
// as warp-uniform (broadcast) 128-bit loads, 4 FMAs per load.
#pragma once
#include "common.cuh"

namespace pinb {

struct DecSmem {  // offsets in floats from the dynamic-smem base (all multiples of 4)
  int wt[PINB200_MAX_HIDDEN_LAYERS];  // forward layout  [in_l][H]
  int w[PINB200_MAX_HIDDEN_LAYERS];   // backward layout [H][in_pad_l] (torch layout, layer 0 padded to DP)
  int b[PINB200_MAX_HIDDEN_LAYERS];   // [H]
  int wout;                           // [out_dim][H]
  int bout;                           // [out_dim] padded to 4
  int end;                            // first free float
};

inline DecSmem plan_decoder_smem(const pinb200_decoder_view& d, int DP, bool with_bwd_layout, int start) {
  DecSmem s{};
  int o = align4(start);
  const int H = d.hidden_dim;
  for (int l = 0; l < d.n_hidden; ++l) {
    const int in = l == 0 ? d.in_dim : H;
    s.wt[l] = o;
    o += align4(in * H);
    s.b[l] = o;
    o += H;
    if (with_bwd_layout) {
      s.w[l] = o;
      o += H * (l == 0 ? DP : H);
    }
  }
  s.wout = o;
  o += d.out_dim * H;
  s.bout = o;
  o += align4(d.out_dim);
  s.end = o;
  return s;
}

// Copy the decoder weights into shared memory (both layouts). All threads call.
__device__ __forceinline__ void stage_decoder(const pinb200_decoder_view& d, const DecSmem& s, float* smem, int DP,
                                              bool with_bwd_layout) {
  const int H = d.hidden_dim;
  const int nt = blockDim.x, tid = threadIdx.x;
  for (int l = 0; l < d.n_hidden; ++l) {
    const int in = l == 0 ? d.in_dim : H;
    const float* W = d.w[l];
    float* wt = smem + s.wt[l];
    for (int e = tid; e < in * H; e += nt) {  // wt[i][j] = W[j][i]
      const int i = e / H, j = e - i * H;
      wt[e] = __ldg(W + (size_t)j * in + i);
    }
    float* bb = smem + s.b[l];
    for (int e = tid; e < H; e += nt) bb[e] = d.b[l] ? __ldg(d.b[l] + e) : 0.f;
    if (with_bwd_layout) {
      const int ip = l == 0 ? DP : H;
      float* w = smem + s.w[l];
      for (int e = tid; e < H * ip; e += nt) {
        const int j = e / ip, i = e - j * ip;
        w[e] = i < in ? __ldg(W + (size_t)j * in + i) : 0.f;
      }
    }
  }
  float* wo = smem + s.wout;
  for (int e = tid; e < d.out_dim * H; e += nt) wo[e] = __ldg(d.w_out + e);
  float* bo = smem + s.bout;
  for (int e = tid; e < align4(d.out_dim); e += nt) bo[e] = (d.b_out && e < d.out_dim) ? __ldg(d.b_out + e) : 0.f;
}

// {d0,d1} += {a0,a1} * b, two round-to-nearest fp32 FMAs (Hopper has no packed fp32 FMA)
__device__ __forceinline__ void ffma2(float& d0, float& d1, float a0, float a1, float b) {
  d0 = fmaf(a0, b, d0);
  d1 = fmaf(a1, b, d1);
}

// out[o] = bias[o] + sum_i w[i][o] * col[i*ACT_LD]   (w: [n_in][NOUT] in smem, warp-uniform float4 reads)
template <int NOUT, int LD = ACT_LD>
__device__ __forceinline__ void matvec_col(const float* __restrict__ w, const float* __restrict__ bias,
                                           const float* __restrict__ col, int n_in, float (&out)[NOUT]) {
  static_assert(NOUT % 4 == 0, "NOUT must be a multiple of 4");
  if (bias) {
#pragma unroll
    for (int o = 0; o < NOUT; o += 4) {
      const float4 b = *reinterpret_cast<const float4*>(bias + o);
      out[o] = b.x;
      out[o + 1] = b.y;
      out[o + 2] = b.z;
      out[o + 3] = b.w;
    }
  } else {
#pragma unroll
    for (int o = 0; o < NOUT; ++o) out[o] = 0.f;
  }
#pragma unroll 2
  for (int i = 0; i < n_in; ++i) {
    const float a = col[i * LD];
    const float4* w4 = reinterpret_cast<const float4*>(w + i * NOUT);
#pragma unroll
    for (int o = 0; o < NOUT / 4; ++o) {
      const float4 ww = w4[o];
      ffma2(out[4 * o + 0], out[4 * o + 1], ww.x, ww.y, a);
      ffma2(out[4 * o + 2], out[4 * o + 3], ww.z, ww.w, a);
    }
  }
}

// ReLU / leaky-ReLU in place; returns the bit mask of positive pre-activations
// (threshold_backward passes the gradient where the input is > 0).
template <int H>
__device__ __forceinline__ uint64_t activate(float (&h)[H], bool leaky) {
  uint64_t mk = 0;
#pragma unroll
  for (int j = 0; j < H; ++j) {
    if (h[j] > 0.f)
      mk |= (1ull << j);
    else
      h[j] = leaky ? 0.01f * h[j] : 0.f;
  }
  return mk;
}

template <int H>
__device__ __forceinline__ void apply_mask(float (&g)[H], uint64_t mk, bool leaky) {
#pragma unroll
  for (int j = 0; j < H; ++j)
    if (!((mk >> j) & 1ull)) g[j] = leaky ? 0.01f * g[j] : 0.f;
}

template <int N, int LD = ACT_LD>
__device__ __forceinline__ void store_col(float* col, const float (&v)[N], int n) {
#pragma unroll
  for (int j = 0; j < N; ++j)
    if (j < n) col[j * LD] = v[j];
}

}  // namespace pinb
