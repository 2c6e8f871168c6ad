// Error plumbing and small host helpers of the C ABI (include/pinb200.h).
#include <stdarg.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "common.cuh"

namespace pinb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return PINB200_ERR_CUDA;
  }
  return PINB200_OK;
}

int sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev != cached_dev) {
    cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
    cached_dev = dev;
    if (cached <= 0) cached = 132;
  }
  return cached;
}

int prepare_kernel(const void* fn, const char* what, size_t smem_bytes, int threads, int* occ) {
  struct Prepared {
    int dev;
    const void* fn;
    size_t smem;
    int occ;  // 0: not asked for yet
  };
  static std::mutex mu;
  static std::vector<Prepared> done;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(mu);
  Prepared* k = nullptr;
  for (Prepared& c : done)
    if (c.dev == dev && c.fn == fn && c.smem == smem_bytes) k = &c;
  if (!k) {
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(%s): %s", what, cudaGetErrorString(e));
      return PINB200_ERR_CUDA;
    }
    done.push_back({dev, fn, smem_bytes, 0});
    k = &done.back();
  }
  if (occ) {
    if (k->occ == 0) {
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&k->occ, fn, threads, smem_bytes);
      if (k->occ < 1) k->occ = 1;
    }
    *occ = k->occ;
  }
  return PINB200_OK;
}

}  // namespace pinb

extern "C" int pinb200_version(void) { return PINB200_VERSION; }
extern "C" const char* pinb200_last_error(void) { return pinb::g_err; }

extern "C" int64_t pinb200_decoder_param_count(const pinb200_decoder_view* d) {
  if (!d) return -1;
  // [w0 | b0 | w1 | b1 | ... | w_out | b_out]; a NULL bias (mlp_bias_on False) has no slot
  int64_t n = 0;
  for (int l = 0; l < d->n_hidden; ++l) {
    const int in = l == 0 ? d->in_dim : d->hidden_dim;
    n += (int64_t)d->hidden_dim * in + (d->b[l] ? d->hidden_dim : 0);
  }
  n += (int64_t)d->out_dim * d->hidden_dim + (d->b_out ? d->out_dim : 0);
  return n;
}
