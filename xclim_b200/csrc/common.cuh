// Shared helpers for the xclim_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>

#include "../../include/xclim_b200.h"

namespace xc {

// ---- thread-local error text ------------------------------------------------------------------
void set_error(const char* fmt, ...);
int32_t cuda_fail(cudaError_t e, const char* what);

#define XC_CHECK_CUDA(expr)                                       \
  do {                                                            \
    cudaError_t _e = (expr);                                      \
    if (_e != cudaSuccess) return ::xc::cuda_fail(_e, #expr);     \
  } while (0)

#define XC_REQUIRE(cond, ...)            \
  do {                                   \
    if (!(cond)) {                       \
      ::xc::set_error(__VA_ARGS__);      \
      return XC_ERR_INVALID;             \
    }                                    \
  } while (0)

inline int32_t launch_status(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, what);
  return XC_OK;
}

// ---- streaming loads: read-once data bypasses L1 allocation -------------------------------------
__device__ __forceinline__ float ld_stream(const float* p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ float4 ld_stream4(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}

// ---- comparison against a scalar threshold ------------------------------------------------------
// A float64 threshold compared with float32 data is folded on the host into an equivalent float32
// threshold by directed rounding (see fold_threshold), so the device only ever compares in float32.
template <int OP>
__device__ __forceinline__ bool cmp(float x, float t) {
  if constexpr (OP == XC_OP_GT) return x > t;
  if constexpr (OP == XC_OP_LT) return x < t;
  if constexpr (OP == XC_OP_GE) return x >= t;
  if constexpr (OP == XC_OP_LE) return x <= t;
  if constexpr (OP == XC_OP_EQ) return x == t;
  if constexpr (OP == XC_OP_ISNAN) return x != x;
  if constexpr (OP == XC_OP_NOTNAN) return x == x;
  return x != t;  // NaN != t is True, as in numpy
}
template <int OP>
__device__ __forceinline__ bool cmpd(double x, double t) {
  if constexpr (OP == XC_OP_GT) return x > t;
  if constexpr (OP == XC_OP_LT) return x < t;
  if constexpr (OP == XC_OP_GE) return x >= t;
  if constexpr (OP == XC_OP_LE) return x <= t;
  if constexpr (OP == XC_OP_EQ) return x == t;
  return x != t;
}

// Host: float32 threshold t32 such that for every float32 x:  (x op t32)  ==  ((double)x op thr)
// when cmp_f64 != 0, or (x op (float)thr) when cmp_f64 == 0 (numpy>=2 weak-scalar promotion).
float fold_threshold(int32_t op, double thr, int32_t cmp_f64);

// dispatch a runtime operator to a compile-time constant
template <typename F>
inline int32_t dispatch_op(int32_t op, F&& f) {
  switch (op) {
    case XC_OP_GT: return f(std::integral_constant<int, XC_OP_GT>{});
    case XC_OP_LT: return f(std::integral_constant<int, XC_OP_LT>{});
    case XC_OP_GE: return f(std::integral_constant<int, XC_OP_GE>{});
    case XC_OP_LE: return f(std::integral_constant<int, XC_OP_LE>{});
    case XC_OP_EQ: return f(std::integral_constant<int, XC_OP_EQ>{});
    case XC_OP_NE: return f(std::integral_constant<int, XC_OP_NE>{});
  }
  set_error("Operation `%d` not recognized.", op);
  return XC_ERR_INVALID;
}

// the six comparison operators plus the two NaN tests (count / run-length entry points only)
template <typename F>
inline int32_t dispatch_op_nan(int32_t op, F&& f) {
  if (op == XC_OP_ISNAN) return f(std::integral_constant<int, XC_OP_ISNAN>{});
  if (op == XC_OP_NOTNAN) return f(std::integral_constant<int, XC_OP_NOTNAN>{});
  return dispatch_op(op, f);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// SMs of the current device (132 on an H100 SXM, 114 on an H100 PCIe): launchers that split a narrow grid
// into more CTAs size the split by it.  The split never changes a result, only how the work is spread.
inline int sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 132;
  }
  return n;
}

}  // namespace xc
