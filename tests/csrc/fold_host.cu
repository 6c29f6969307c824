// TEST INFRASTRUCTURE: a HOST build of the threshold folding rule xc::fold_f64 (xclim_b200/csrc/common.cuh), which
// every float64-threshold count applies on the device and fold_threshold applies on the host.
// tests/test_fold_host.py checks it against numpy's float64 compare.  Nothing in xclim_b200/ loads this library.
#include "../../xclim_b200/csrc/common.cuh"

template <int OP>
static void fold_all(const double* t, int64_t n, float* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = xc::fold_f64<OP>(t[i]);
}

extern "C" int32_t fold_host_f64(int32_t op, const double* t, int64_t n, float* out) {
  switch (op) {
    case XC_OP_GT: fold_all<XC_OP_GT>(t, n, out); return 0;
    case XC_OP_LT: fold_all<XC_OP_LT>(t, n, out); return 0;
    case XC_OP_GE: fold_all<XC_OP_GE>(t, n, out); return 0;
    case XC_OP_LE: fold_all<XC_OP_LE>(t, n, out); return 0;
    case XC_OP_EQ: fold_all<XC_OP_EQ>(t, n, out); return 0;
    case XC_OP_NE: fold_all<XC_OP_NE>(t, n, out); return 0;
  }
  return -1;
}
