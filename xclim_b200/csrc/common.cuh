// Shared helpers for the xclim_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>
#include <string.h>

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

// ---- mbarriers: the completion signal of the bulk copies (cp.async.bulk) ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "XC_MBAR_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra XC_MBAR_DONE;\n"
      "bra XC_MBAR_WAIT;\n"
      "XC_MBAR_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// ---- comparison against a scalar threshold ------------------------------------------------------
// A float64 threshold compared with float32 data is folded into an equivalent float32 threshold by
// directed rounding (see fold_f64), so the device only ever compares in float32.
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

// f with d added to its bit pattern: one float32 step away from zero (d = 1) or towards it (d = -1)
__host__ __device__ __forceinline__ float add_to_bits(float f, int32_t d) {
#ifdef __CUDA_ARCH__
  return __int_as_float(__float_as_int(f) + d);
#else
  int32_t i;
  memcpy(&i, &f, sizeof i);
  i += d;
  memcpy(&f, &i, sizeof f);
  return f;
#endif
}

// The float32 threshold with the truth table of the float64 threshold t: (x op fold_f64<OP>(t)) == ((double)x op t)
// for every float32 x, NaN included, so that a float64 compare (numpy promotes float32 data against a float64
// threshold) costs one float32 compare.  > and <= take the largest float32 <= t, >= and < the smallest float32 >= t;
// == and != keep t when it is a float32 and take NaN otherwise (never equal, always different).  NaN stays NaN.
template <int OP>
__host__ __device__ __forceinline__ float fold_f64(double t) {
  float f = (float)t;
  if (t != t) return f;
  if constexpr (OP == XC_OP_EQ || OP == XC_OP_NE) {
    return (double)f == t ? f : NAN;
  } else if constexpr (OP == XC_OP_GT || OP == XC_OP_LE) {  // largest float32 <= t
    if ((double)f > t) f = add_to_bits(f, (f > 0.f) ? -1 : 1);
    if (f == 0.f && t < 0.0) f = -1.401298464e-45f;
  } else {                                                  // smallest float32 >= t
    if ((double)f < t) f = add_to_bits(f, (f >= 0.f) ? 1 : -1);
    if (f == 0.f && t > 0.0) f = 1.401298464e-45f;
  }
  return f;
}

// Host: float32 threshold t32 such that for every float32 x:  (x op t32)  ==  ((double)x op thr)
// when cmp_f64 != 0 (fold_f64), or (x op (float)thr) when cmp_f64 == 0 (numpy>=2 weak-scalar promotion).
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

// the shared-memory sort length of a series of T <= 32768 steps (the power of two >= T, at least 1024) as a
// compile-time constant
template <typename F>
inline auto dispatch_npad(int64_t T, F&& f) {
  if (T <= 1024) return f(std::integral_constant<int, 1024>{});
  if (T <= 2048) return f(std::integral_constant<int, 2048>{});
  if (T <= 4096) return f(std::integral_constant<int, 4096>{});
  if (T <= 8192) return f(std::integral_constant<int, 8192>{});
  if (T <= 16384) return f(std::integral_constant<int, 16384>{});
  return f(std::integral_constant<int, 32768>{});
}

// interpolation (0 nearest, 1 linear) and kind (0 "+", 1 "*") of a quantile-mapping adjust as compile-time constants
template <typename F>
inline auto dispatch_interp_kind(int32_t interp, int32_t kind, F&& f) {
  using I0 = std::integral_constant<int, 0>;
  using I1 = std::integral_constant<int, 1>;
  if (interp == 0) return kind == 0 ? f(I0{}, I0{}) : f(I0{}, I1{});
  return kind == 0 ? f(I1{}, I0{}) : f(I1{}, I1{});
}

// nq in [nq_lo, nq_hi], kind and interp: the arguments every quantile-mapping entry point checks (train has no interp)
inline int32_t check_qmap_args(int32_t nq, int nq_lo, int nq_hi, int32_t kind, int32_t interp = 0) {
  XC_REQUIRE(nq >= nq_lo && nq <= nq_hi, "nquantiles must be in [%d, %d]", nq_lo, nq_hi);
  XC_REQUIRE(kind == 0 || kind == 1, "kind must be 0 ('+') or 1 ('*')");
  XC_REQUIRE(interp == 0 || interp == 1, "interp must be 0 (nearest) or 1 (linear)");
  return XC_OK;
}

// lets `kernel` use `bytes` of dynamic shared memory (an opt-in above the default 48 KiB)
template <typename Kernel>
inline int32_t allow_smem(Kernel* kernel, size_t bytes, const char* what) {
  if (bytes <= 48 * 1024) return XC_OK;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  return e == cudaSuccess ? XC_OK : cuda_fail(e, what);
}

// Block-wide bitonic sort of keys[0..NPAD) ascending in shared memory by NT threads (NaN-free keys): the
// fallback sort of the EQM train and QDM rank kernels.
template <int NPAD, int NT>
__device__ void block_bitonic_sort(float* keys, int tid) {
  for (int k = 2; k <= NPAD; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < NPAD / 2; i += NT) {
        const int a = ((i & ~(j - 1)) << 1) | (i & (j - 1));  // pair (a, a | j)
        const int b = a | j;
        const bool up = ((a & k) == 0);
        const float x0 = keys[a], x1 = keys[b];
        const bool swap = up ? (x0 > x1) : (x0 < x1);
        if (swap) { keys[a] = x1; keys[b] = x0; }
      }
      __syncthreads();
    }
  }
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

// Time split of the streaming quantile-mapping kernels: blockIdx.y walks `chunks` chunks of `rows` steps.  Enough
// chunks for 16 CTAs per SM over the cblocks cell blocks, each at least min_rows steps, rounded up to whole `align`s.
struct RowSplit {
  int chunks, rows;
};
inline RowSplit split_rows(int64_t T, int64_t cblocks, int align, int min_rows) {
  int64_t chunks = (sm_count() * 16 + cblocks - 1) / cblocks;
  if (chunks < 1) chunks = 1;
  int64_t rows = (T + chunks - 1) / chunks;
  rows = (rows + align - 1) / align * align;
  if (rows < min_rows) rows = min_rows;
  return {(int)((T + rows - 1) / rows), (int)rows};
}

}  // namespace xc
