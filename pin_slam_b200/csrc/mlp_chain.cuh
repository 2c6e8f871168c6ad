// Warp-level tensor-core decoder building blocks of the query kernel (K1, query_kernel) and the tensor-core training
// backward (K2, train_bwd_mma_kernel).
//
// The decoder is a chain of [32 x K] x [K x 64] contractions per warp tile, issued as mma.sync.m16n8k8 TF32
// tensor-core instructions with the 3xTF32 split  a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo  (a_hi = a with the low
// 13 mantissa bits cleared, a_lo = a - a_hi exactly), which keeps ~21 mantissa bits: the SDF stays within the 1e-5
// parity bound of the fp32 reference.  Weights are split once per CTA when they are staged into shared memory.
//
// Register chaining (K1): the k index of a contraction may be permuted freely as long as A and B agree.  With
// the permutation  slot t <-> unit 8kk+2t,  slot t+4 <-> unit 8kk+2t+1  of every k-step the C fragments of one layer
// ARE the A fragments of the next one (c0,c2,c1,c3 -> a0,a1,a2,a3), so the activations never leave the register
// file between layers, and the two B values of a lane become adjacent in the nn.Linear row: one LDS.64 per (hi | lo)
// fragment instead of two LDS.32.  Leading dimensions == 8 (mod 32) make those 64-bit fragment loads bank-conflict
// free.  K2 keeps its activations in row-major shared-memory tiles (it needs them again for the weight gradients)
// and multiplies them with warp_gemm_3xtf32, whose scalar fragment loads are conflict free with leading dimensions
// == 4 (mod 32).
//
// (wgmma needs 64-row warpgroup tiles and a warpgroup-wide issue / wait choreography; with independent 32-row warp
// tiles the warp-synchronous mma.sync form is the natural fit.  DESIGN.md section 7 discusses the trade-off.)
#pragma once
#include "common.cuh"

namespace pinb {

constexpr uint32_t TF32_MASK = 0xffffe000u;

// decoder input width (FT features + 3 position components) padded to the MMA k-step
__host__ __device__ constexpr int dec_in_pad(int FT) { return (FT + 3 + 7) / 8 * 8; }

// smallest leading dimension >= x that is == 8 (mod 32): conflict-free 64-bit fragment loads
__host__ __device__ constexpr int ld8mod32(int x) { return x <= 8 ? 8 : ((x - 8 + 31) / 32) * 32 + 8; }

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

struct WarpDecSmem {  // float offsets from the dynamic-smem base
  int whi[PINB200_MAX_HIDDEN_LAYERS];  // [H][ldw_l]  tf32 "hi" part, torch layout, zero padded
  int wlo[PINB200_MAX_HIDDEN_LAYERS];  // [H][ldw_l]  tf32 "lo" part
  int b[PINB200_MAX_HIDDEN_LAYERS];    // [H]
  int ldw[PINB200_MAX_HIDDEN_LAYERS];  // ld(padded fan-in of layer l)
  int wout, bout, end;
};

// KP0: padded fan-in of layer 0; ld(fan_in) -> leading dimension of a weight matrix (the kernel's fragment loads
// decide which one is bank-conflict free)
template <class Ld>
inline WarpDecSmem plan_warp_decoder_smem(const pinb200_decoder_view& d, int KP0, int start, Ld ld) {
  WarpDecSmem s{};
  int o = align4(start);
  const int H = d.hidden_dim;
  for (int l = 0; l < d.n_hidden; ++l) {
    s.ldw[l] = ld(l == 0 ? KP0 : H);
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
  o += align4(d.out_dim);
  s.end = o;
  return s;
}

__device__ __forceinline__ void stage_warp_decoder(const pinb200_decoder_view& d, const WarpDecSmem& s, float* smem) {
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
  for (int e = tid; e < align4(d.out_dim); e += nt) bo[e] = (d.b_out && e < d.out_dim) ? __ldg(d.b_out + e) : 0.f;
}

template <int NT>
__device__ __forceinline__ void zero_frags(float (&acc)[2][NT][4]) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[mt][nt][c] = 0.f;
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

// K2: acc[mt][nt] (16x8 C fragments, mt < 2 row blocks, nt < NT column blocks) = X[32 x 8*KT] * B, X row-major in
// shared memory (leading dimension LDX == 4 mod 32), k in natural order
//   BWD == false: B[k][n] = W[n][k]   (forward layer:  h = x W^T)
//   BWD == true : B[k][n] = W[k][n]   (backward layer: g_in = g_out W)
template <int KT, int NT, bool BWD, int LDX>
__device__ __forceinline__ void warp_gemm_3xtf32(float (&acc)[2][NT][4], const float* __restrict__ x,
                                                 const float* __restrict__ whi, const float* __restrict__ wlo, int ldw,
                                                 int lane) {
  const int g = lane >> 2, t = lane & 3;
  zero_frags<NT>(acc);
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

// one k-step of the forward contraction against W[n_out][k_in] (nn.Linear layout): B pairs are adjacent floats
template <int NT>
__device__ __forceinline__ void kstep_fwd(float (&acc)[2][NT][4], const uint32_t (&ah)[2][4], const uint32_t (&al)[2][4],
                                          const float* __restrict__ whi, const float* __restrict__ wlo, int ldw, int kk,
                                          int g, int t) {
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int o = (nt * 8 + g) * ldw + kk * 8 + 2 * t;
    const float2 h2 = *reinterpret_cast<const float2*>(whi + o);
    const float2 l2 = *reinterpret_cast<const float2*>(wlo + o);
    const uint32_t bh[2] = {__float_as_uint(h2.x), __float_as_uint(h2.y)};
    const uint32_t bl[2] = {__float_as_uint(l2.x), __float_as_uint(l2.y)};
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      mma_tf32(acc[mt][nt], al[mt], bh);  // small terms first
      mma_tf32(acc[mt][nt], ah[mt], bl);
      mma_tf32(acc[mt][nt], ah[mt], bh);
    }
  }
}

// one k-step of the backward contraction g_in = g_out W: B[k = out unit][n = in unit] = W[k][n]
template <int NT>
__device__ __forceinline__ void kstep_bwd(float (&acc)[2][NT][4], const uint32_t (&ah)[2][4], const uint32_t (&al)[2][4],
                                          const float* __restrict__ whi, const float* __restrict__ wlo, int ldw, int kk,
                                          int g, int t) {
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int o = (kk * 8 + 2 * t) * ldw + nt * 8 + g;
    const uint32_t bh[2] = {__float_as_uint(whi[o]), __float_as_uint(whi[o + ldw])};
    const uint32_t bl[2] = {__float_as_uint(wlo[o]), __float_as_uint(wlo[o + ldw])};
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      mma_tf32(acc[mt][nt], al[mt], bh);
      mma_tf32(acc[mt][nt], ah[mt], bl);
      mma_tf32(acc[mt][nt], ah[mt], bh);
    }
  }
}

// A fragments of k-step kk taken from the previous layer's C fragments (register chaining)
__device__ __forceinline__ void frags_from_acc(const float (&in)[2][8][4], int kk, uint32_t (&ah)[2][4],
                                               uint32_t (&al)[2][4]) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
    split_tf32(in[mt][kk][0], ah[mt][0], al[mt][0]);  // (row g,   unit 2t)
    split_tf32(in[mt][kk][2], ah[mt][1], al[mt][1]);  // (row g+8, unit 2t)
    split_tf32(in[mt][kk][1], ah[mt][2], al[mt][2]);  // (row g,   unit 2t+1)
    split_tf32(in[mt][kk][3], ah[mt][3], al[mt][3]);  // (row g+8, unit 2t+1)
  }
}

// layer 0: acc = X[32 x 8*KT] W0^T with X in the warp's row-major shared-memory tile (leading dimension LDX == 8 mod 32)
template <int KT, int LDX>
__device__ __forceinline__ void gemm_from_tile(float (&acc)[2][8][4], const float* __restrict__ x,
                                               const float* __restrict__ whi, const float* __restrict__ wlo, int ldw,
                                               int lane) {
  const int g = lane >> 2, t = lane & 3;
  zero_frags<8>(acc);
#pragma unroll
  for (int kk = 0; kk < KT; ++kk) {
    uint32_t ah[2][4], al[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const float2 r0 = *reinterpret_cast<const float2*>(x + (mt * 16 + g) * LDX + kk * 8 + 2 * t);
      const float2 r1 = *reinterpret_cast<const float2*>(x + (mt * 16 + g + 8) * LDX + kk * 8 + 2 * t);
      split_tf32(r0.x, ah[mt][0], al[mt][0]);
      split_tf32(r1.x, ah[mt][1], al[mt][1]);
      split_tf32(r0.y, ah[mt][2], al[mt][2]);
      split_tf32(r1.y, ah[mt][3], al[mt][3]);
    }
    kstep_fwd<8>(acc, ah, al, whi, wlo, ldw, kk, g, t);
  }
}

// hidden layer l >= 1, forward: out = in W_l^T, `in` in C-fragment form
__device__ __forceinline__ void gemm_chain_fwd(float (&out)[2][8][4], const float (&in)[2][8][4],
                                               const float* __restrict__ whi, const float* __restrict__ wlo, int ldw,
                                               int lane) {
  const int g = lane >> 2, t = lane & 3;
  zero_frags<8>(out);
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    uint32_t ah[2][4], al[2][4];
    frags_from_acc(in, kk, ah, al);
    kstep_fwd<8>(out, ah, al, whi, wlo, ldw, kk, g, t);
  }
}

// backward through a layer: out[32 x 8*NT] = in[32 x 64] W   (NT = 8 for hidden layers, KP0/8 for layer 0)
template <int NT>
__device__ __forceinline__ void gemm_chain_bwd(float (&out)[2][NT][4], const float (&in)[2][8][4],
                                               const float* __restrict__ whi, const float* __restrict__ wlo, int ldw,
                                               int lane) {
  const int g = lane >> 2, t = lane & 3;
  zero_frags<NT>(out);
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    uint32_t ah[2][4], al[2][4];
    frags_from_acc(in, kk, ah, al);
    kstep_bwd<NT>(out, ah, al, whi, wlo, ldw, kk, g, t);
  }
}

// bias + (leaky) ReLU in place; returns the 64-bit mask of positive pre-activations in fragment order
// (bit mt*32 + nt*4 + c).  `bias` is 8-byte aligned.
template <int NT>
__device__ __forceinline__ uint64_t bias_act_chain(float (&acc)[2][NT][4], const float* __restrict__ bias, bool leaky,
                                                   int lane) {
  uint32_t mk[2] = {0u, 0u};
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const float2 b2 = *reinterpret_cast<const float2*>(bias + frag_col(nt, 0, lane));
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float v = acc[mt][nt][c] + ((c & 1) ? b2.y : b2.x);
        if (v > 0.f)
          mk[mt] |= 1u << (nt * 4 + c);
        else
          v = leaky ? 0.01f * v : 0.f;
        acc[mt][nt][c] = v;
      }
  }
  return (uint64_t)mk[0] | ((uint64_t)mk[1] << 32);
}

// the (leaky) ReLU derivative of a bias_act_chain mask applied to a gradient in the same fragment order
template <int NT>
__device__ __forceinline__ void mask_chain(float (&acc)[2][NT][4], uint64_t mk64, bool leaky) {
  const uint32_t mk[2] = {(uint32_t)mk64, (uint32_t)(mk64 >> 32)};
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (!((mk[mt] >> (nt * 4 + c)) & 1u)) acc[mt][nt][c] = leaky ? 0.01f * acc[mt][nt][c] : 0.f;
}

}  // namespace pinb
