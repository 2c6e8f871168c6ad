// Warp-level tensor-core decoder for the per-warp 32-row tiles of K1.
//
// The decoder is a chain of [32 x K] x [K x 64] contractions per warp tile.  On fp32 SIMT it was ~47 % of K1's
// instructions; here each contraction is issued as mma.sync.m16n8k8 TF32 tensor-core instructions with the
// 3xTF32 split  a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo  (a_hi = a with the low 13 mantissa bits cleared,
// a_lo = a - a_hi exactly), which keeps ~21 mantissa bits: the SDF stays within the 1e-5 parity bound of the
// fp32 reference.  Weights are split once per CTA when they are staged into shared memory.
//
// Tile layout: ROW-major x[row][col], leading dimension LDX = 68 (== 4 mod 32: the A-fragment pattern
// (row = lane/4, col = lane%4) is bank-conflict free); weights in the torch nn.Linear layout [out][in] with
// leading dimension in_pad + 4 for the same reason.
//
// (wgmma needs 64-row warpgroup tiles and a warpgroup-wide issue / wait choreography; with independent 32-row warp
// tiles the warp-synchronous mma.sync form is the natural fit.  DESIGN.md section 7 discusses the trade-off.)
#pragma once
#include "common.cuh"

namespace pinb {

constexpr uint32_t TF32_MASK = 0xffffe000u;

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void split_tf32(float v, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(v) & TF32_MASK;
  lo = __float_as_uint(v - __uint_as_float(hi)) & TF32_MASK;
}

struct MmaDecSmem {  // float offsets from the dynamic-smem base
  int whi[PINB200_MAX_HIDDEN_LAYERS];  // [H][ldw_l]  tf32 "hi" part, torch layout, zero padded
  int wlo[PINB200_MAX_HIDDEN_LAYERS];  // [H][ldw_l]  tf32 "lo" part
  int b[PINB200_MAX_HIDDEN_LAYERS];    // [H]
  int ldw[PINB200_MAX_HIDDEN_LAYERS];  // in_pad_l + 4
  int wout, bout, end;
};

__host__ __device__ inline int align4i(int x) { return (x + 3) & ~3; }

inline MmaDecSmem plan_mma_decoder_smem(const pinb200_decoder_view& d, int KP0, int start) {
  MmaDecSmem s{};
  int o = align4i(start);
  const int H = d.hidden_dim;
  for (int l = 0; l < d.n_hidden; ++l) {
    s.ldw[l] = (l == 0 ? KP0 : H) + 4;
    s.whi[l] = o;
    o += H * s.ldw[l];
    s.wlo[l] = o;
    o += H * s.ldw[l];
    s.b[l] = o;
    o += H;
  }
  s.wout = o;
  o += d.out_dim * H;
  s.bout = o;
  o += align4i(d.out_dim);
  s.end = o;
  return s;
}

__device__ __forceinline__ void stage_mma_decoder(const pinb200_decoder_view& d, const MmaDecSmem& s, float* smem) {
  const int H = d.hidden_dim, nt = blockDim.x, tid = threadIdx.x;
  for (int l = 0; l < d.n_hidden; ++l) {
    const int in = l == 0 ? d.in_dim : H, ldw = s.ldw[l];
    float* hi = smem + s.whi[l];
    float* lo = smem + s.wlo[l];
    for (int e = tid; e < H * ldw; e += nt) {
      const int j = e / ldw, i = e - j * ldw;
      const float w = i < in ? __ldg(d.w[l] + (size_t)j * in + i) : 0.f;
      uint32_t h, lw;
      split_tf32(w, h, lw);
      hi[e] = __uint_as_float(h);
      lo[e] = __uint_as_float(lw);
    }
    float* bb = smem + s.b[l];
    for (int e = tid; e < H; e += nt) bb[e] = d.b[l] ? __ldg(d.b[l] + e) : 0.f;
  }
  float* wo = smem + s.wout;
  for (int e = tid; e < d.out_dim * H; e += nt) wo[e] = __ldg(d.w_out + e);
  float* bo = smem + s.bout;
  for (int e = tid; e < align4i(d.out_dim); e += nt) bo[e] = (d.b_out && e < d.out_dim) ? __ldg(d.b_out + e) : 0.f;
}

// acc[mt][nt] (16x8 C fragments, mt < 2 row blocks, nt < NT column blocks) = X[32 x 8*KT] * B
//   BWD == false: B[k][n] = W[n][k]   (forward layer:  h = x W^T)
//   BWD == true : B[k][n] = W[k][n]   (backward layer: g_in = g_out W)
template <int KT, int NT, bool BWD, int LDX>
__device__ __forceinline__ void warp_gemm_3xtf32(float (&acc)[2][NT][4], const float* __restrict__ x,
                                                 const float* __restrict__ whi, const float* __restrict__ wlo, int ldw,
                                                 int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[mt][nt][c] = 0.f;
#pragma unroll 1
  for (int kk = 0; kk < KT; ++kk) {
    uint32_t ah[2][4], al[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const float* xr = x + (mt * 16 + g) * LDX + kk * 8 + t;
      split_tf32(xr[0], ah[mt][0], al[mt][0]);
      split_tf32(xr[8 * LDX], ah[mt][1], al[mt][1]);
      split_tf32(xr[4], ah[mt][2], al[mt][2]);
      split_tf32(xr[8 * LDX + 4], ah[mt][3], al[mt][3]);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      int o0, o1;
      if (!BWD) {
        o0 = (nt * 8 + g) * ldw + kk * 8 + t;
        o1 = o0 + 4;
      } else {
        o0 = (kk * 8 + t) * ldw + nt * 8 + g;
        o1 = o0 + 4 * ldw;
      }
      uint32_t bh[2], bl[2];
      bh[0] = __float_as_uint(whi[o0]);
      bh[1] = __float_as_uint(whi[o1]);
      bl[0] = __float_as_uint(wlo[o0]);
      bl[1] = __float_as_uint(wlo[o1]);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma_tf32(acc[mt][nt], al[mt], bh);  // small terms first
        mma_tf32(acc[mt][nt], ah[mt], bl);
        mma_tf32(acc[mt][nt], ah[mt], bh);
      }
    }
  }
}

// C-fragment coordinates of element c of block (mt, nt) for this lane
__device__ __forceinline__ int frag_row(int mt, int c, int lane) { return mt * 16 + (lane >> 2) + 8 * (c >> 1); }
__device__ __forceinline__ int frag_col(int nt, int c, int lane) { return nt * 8 + 2 * (lane & 3) + (c & 1); }

// x[row][col] = acc (float2 stores); caller brackets with __syncwarp()
template <int NT, int LDX>
__device__ __forceinline__ void store_frags(float* __restrict__ x, const float (&acc)[2][NT][4], int lane) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2 v = make_float2(acc[mt][nt][2 * h], acc[mt][nt][2 * h + 1]);
        *reinterpret_cast<float2*>(x + frag_row(mt, 2 * h, lane) * LDX + frag_col(nt, 0, lane)) = v;
      }
    }
}

// bias + (leaky) ReLU in place; returns the 64-bit mask of positive pre-activations in fragment order
template <int NT>
__device__ __forceinline__ uint64_t bias_act_frags(float (&acc)[2][NT][4], const float* __restrict__ bias, bool leaky,
                                                   int lane) {
  uint64_t mk = 0;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float v = acc[mt][nt][c] + bias[frag_col(nt, c, lane)];
        if (v > 0.f)
          mk |= 1ull << (mt * 32 + nt * 4 + c);
        else
          v = leaky ? 0.01f * v : 0.f;
        acc[mt][nt][c] = v;
      }
  return mk;
}

template <int NT>
__device__ __forceinline__ void mask_frags(float (&acc)[2][NT][4], uint64_t mk, bool leaky) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (!((mk >> (mt * 32 + nt * 4 + c)) & 1ull)) acc[mt][nt][c] = leaky ? 0.01f * acc[mt][nt][c] : 0.f;
}

}  // namespace pinb
