// Library-wide pieces of the C ABI: error reporting, version, threshold folding.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace xc {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int32_t cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
  (void)cudaGetLastError();  // clear the sticky-less error state
  return XC_ERR_CUDA;
}

float fold_threshold(int32_t op, double thr, int32_t cmp_f64) {
  // round to nearest even, as numpy does for a weak Python scalar (and for the NaN tests, which ignore thr)
  if (!cmp_f64 || op < XC_OP_GT || op > XC_OP_NE) return (float)thr;
  float f = 0.f;
  dispatch_op(op, [&](auto OPC) -> int32_t {
    f = fold_f64<decltype(OPC)::value>(thr);
    return XC_OK;
  });
  return f;
}

}  // namespace xc

extern "C" int32_t xc_version(void) { return XC_VERSION; }
extern "C" const char* xc_last_error(void) { return xc::g_err; }

extern "C" int32_t xc_device_sm_count(int32_t* out_sm_count) {
  XC_REQUIRE(out_sm_count != nullptr, "null pointer argument");
  int dev = 0, n = 0;
  XC_CHECK_CUDA(cudaGetDevice(&dev));
  XC_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  *out_sm_count = n;
  return XC_OK;
}
