// Microbenchmark: random 16-byte gathers (one sector per lane) -- achievable sectors/cycle/SM vs resident warps and
// loads in flight per thread, for an L2-resident and a DRAM-resident table.   nvcc -arch=sm_90a -O3 -o gather_bw gather_bw.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include <vector>

template <int ILP>
__global__ void gather(const float4* __restrict__ tab, uint32_t mask, int iters, float* out, int dep) {
  uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u + 12345u;
  float acc = 0.f;
  for (int it = 0; it < iters; ++it) {
    float4 v[ILP];
#pragma unroll
    for (int j = 0; j < ILP; ++j) {
      s = s * 1664525u + 1013904223u;
      v[j] = __ldg(tab + ((s >> 4) & mask));
    }
#pragma unroll
    for (int j = 0; j < ILP; ++j) acc += v[j].x + v[j].w;
    if (dep) s += (uint32_t)acc & 1u;  // make the next round depend on this one
  }
  if (acc == 123.456f) out[0] = acc;
}

template <int ILP>
void run(const float4* tab, uint32_t mask, int warps_per_sm, int sms, float* out, const char* what) {
  const int iters = 256;
  dim3 grid(sms), block(warps_per_sm * 32);
  gather<ILP><<<grid, block>>>(tab, mask, 8, out, 1);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a);
  gather<ILP><<<grid, block>>>(tab, mask, iters, out, 1);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms;
  cudaEventElapsedTime(&ms, a, b);
  const double sectors = (double)sms * warps_per_sm * 32 * iters * ILP;
  const double cyc = ms * 1e-3 * 1.965e9;
  printf("%s warps/SM %2d ILP %2d : %.3f ms  %.3f sectors/cycle/SM  (%.0f GB/s of 32B sectors, latency/round %.0f cyc)\n", what,
         warps_per_sm, ILP, ms, sectors / cyc / sms, sectors * 32 / (ms * 1e-3) / 1e9, cyc / iters);
}

int main() {
  int sms = 148;
  float* out;
  cudaMalloc(&out, 4);
  for (int big = 0; big < 2; ++big) {
    const size_t n = big ? (1u << 26) : (1u << 20);  // 1 GiB vs 16 MiB of float4
    float4* tab;
    cudaMalloc(&tab, n * sizeof(float4));
    cudaMemset(tab, 0, n * sizeof(float4));
    const uint32_t mask = (uint32_t)(n - 1);
    const char* what = big ? "1GiB " : "16MiB";
    for (int w : {4, 8, 12, 16, 24, 32, 48}) {
      run<1>(tab, mask, w, sms, out, what);
      run<4>(tab, mask, w, sms, out, what);
      run<8>(tab, mask, w, sms, out, what);
      run<16>(tab, mask, w, sms, out, what);
    }
    cudaFree(tab);
  }
  return 0;
}
