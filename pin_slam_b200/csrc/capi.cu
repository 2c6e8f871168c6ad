// Error plumbing and small host helpers of the C ABI (include/pinb200.h).
#include <stdarg.h>
#include <string.h>

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
