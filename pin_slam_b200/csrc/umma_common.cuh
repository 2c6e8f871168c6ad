// Hopper warpgroup-MMA (wgmma) building blocks of the warp-specialised decode (wsq.cu): shared-memory matrix
// descriptors of the no-swizzle canonical K-major layout, wgmma issue (operands from shared memory or, for A, from
// registers), TF32 hi/lo split, weight staging.
//
// Accumulator fragment of a 64 x N wgmma (per warpgroup of 128 threads): warp w of the group, lane l, g = l / 4,
// c = l % 4 holds for every 8-column block j: d[4j + 0, 1] = rows 16w + g, columns 8j + 2c, 8j + 2c + 1 and
// d[4j + 2, 3] = row 16w + g + 8, same columns.
#pragma once
#include "mlp_chain.cuh"  // TF32_MASK, dec_in_pad

namespace pinb {

constexpr int UM_ROWS = 128;
constexpr int UM_A_LBO = 144;  // bytes between the 16-byte K chunks of an A row group: 128 + 16 keeps the F/4-lanes-per-row
                               // gather stores (8 lanes = 8 chunks of one row) on different banks
constexpr int UM_W_LBO = 128;


__device__ __forceinline__ uint32_t um_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// wgmma matrix descriptor, no swizzle: LBO = bytes between core matrices along K, SBO = bytes between 8-row groups
__device__ __forceinline__ uint64_t um_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
  return d;  // base offset 0, layout type 0 = no swizzle
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define PINB_WG_D32                                                                                                  \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31}"
#define PINB_WG_D32_OPS                                                                                                \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),         \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),          \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),         \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x 64] (+)= A B^T, tf32, operands from shared memory (descriptors), with the descriptors advanced by compile-time
// k-step offsets inside the asm statement: the caller keeps one base descriptor per operand live instead of one
// (uniform) register pair per k-step, which is what a 136-register warpgroup can afford.
template <int AOFF, int BOFF>
__device__ __forceinline__ void wg_mma_n64_at(float (&d)[32], uint64_t adesc, uint64_t bdesc, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b64 ad, bd;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "add.s64 ad, %32, %35;\n\t"
      "add.s64 bd, %33, %36;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " PINB_WG_D32 ", ad, bd, p, 1, 1;\n\t}\n"
      : PINB_WG_D32_OPS
      : "l"(adesc), "l"(bdesc), "r"(acc), "n"(AOFF), "n"(BOFF)
      : "memory");
}
// The same with A (64 x 8) from registers in the m16n8k8 A-fragment order
// (a0: row g, k c; a1: row g + 8, k c; a2: row g, k c + 4; a3: row g + 8, k c + 4)
template <int BOFF>
__device__ __forceinline__ void wg_mma_n64_rs_at(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                 uint64_t bdesc, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b64 bd;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "add.s64 bd, %36, %38;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " PINB_WG_D32 ", {%32, %33, %34, %35}, bd, p, 1, 1;\n\t}\n"
      : PINB_WG_D32_OPS
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(acc), "n"(BOFF)
      : "memory");
}
#undef PINB_WG_D32
#undef PINB_WG_D32_OPS

// make the generic-proxy shared-memory writes of every thread visible to the tensor core, then meet
__device__ __forceinline__ void um_publish_and_sync() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
}

__device__ __forceinline__ void um_split4(const float4 v, float4& hi, float4& lo) {
  hi.x = __uint_as_float(__float_as_uint(v.x) & TF32_MASK);
  hi.y = __uint_as_float(__float_as_uint(v.y) & TF32_MASK);
  hi.z = __uint_as_float(__float_as_uint(v.z) & TF32_MASK);
  hi.w = __uint_as_float(__float_as_uint(v.w) & TF32_MASK);
  lo.x = v.x - hi.x;
  lo.y = v.y - hi.y;
  lo.z = v.z - hi.z;
  lo.w = v.w - hi.w;
}

// byte offset of the 16-byte chunk (row m, columns 4*c .. 4*c+3) of an A tile with K columns
__device__ __forceinline__ int um_a_off(int m, int c, int K) { return (m >> 3) * ((K >> 2) * UM_A_LBO) + c * UM_A_LBO + (m & 7) * 16; }

// position of column c inside its 8-column k-step when the A operand comes from accumulator registers: register
// fragment slot k (0..3) carries accumulator column 2k, slot k + 4 column 2k + 1 (see wg_mma_n64_rs_at)
__device__ __forceinline__ int um_kperm(int c) { return (c & ~7) | ((c & 1) ? 4 + ((c & 7) >> 1) : ((c & 7) >> 1)); }

// stage the canonical K-major B tile of `rows` x `cols`: element (r, c) = src[r][c] for r < rows_src, c < cols_src,
// zero elsewhere; `src_ld` = leading dimension of the row-major source.  `kperm` stores column c at um_kperm(c), for an
// A operand taken from accumulator registers.  `transpose` stages the transposed source: element (r, c) = src[c][r].
__device__ __forceinline__ void um_stage_weight(const float* __restrict__ src, int src_ld, int rows_src, int cols_src, int rows,
                                                int cols, unsigned char* hi, unsigned char* lo, bool kperm = false,
                                                bool transpose = false) {
  for (int e = threadIdx.x; e < rows * cols; e += blockDim.x) {
    const int r = e / cols, c = e - r * cols;
    float w = 0.f;
    if (r < rows_src && c < cols_src) w = __ldg(src + (transpose ? (size_t)c * src_ld + r : (size_t)r * src_ld + c));
    const float h = __uint_as_float(__float_as_uint(w) & TF32_MASK);
    const int cs = kperm ? um_kperm(c) : c;
    const int off = (r >> 3) * ((cols >> 2) * UM_W_LBO) + (cs >> 2) * UM_W_LBO + (r & 7) * 16 + (cs & 3) * 4;
    *reinterpret_cast<float*>(hi + off) = h;
    *reinterpret_cast<float*>(lo + off) = w - h;
  }
}

template <int FT>
struct UmmaDims {
  static constexpr int K0 = dec_in_pad(FT);
};

}  // namespace pinb
