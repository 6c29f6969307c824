// Run-length / count statistics of a condition on TWO variables.
//
// Replaces indices/_multivariate.py:646-880 (`heat_wave_frequency` / `_max_length` / `_total_length`:
// cond = (tasmin op t1) & (tasmax op t2) -> rl.resample_and_rl(<run statistic>)), :1653-1716
// (`tx_tn_days_above`) and indices/generic.py:1002-1073 (`bivariate_count_occurrences`, var_reducer
// all / any).  Same lane-owns-4-cells streaming as period_stats.cu with two 128-bit loads per step;
// operators and the reducer are runtime switches (the kernel moves 8 B per element and is HBM-bound).
#include "runstat.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;
constexpr int kUnroll = 4;

// Runtime operator without a branch: (x op t) == (((x<t)&L) | ((x==t)&E) | ((x>t)&G)) != N with the
// masks below (NaN makes the three tests false, so only != is true on NaN, as in numpy).
struct OpMask {
  bool L, E, G, N;
};
inline OpMask op_mask(int op) {
  switch (op) {
    case XC_OP_GT: return {false, false, true, false};
    case XC_OP_LT: return {true, false, false, false};
    case XC_OP_GE: return {false, true, true, false};
    case XC_OP_LE: return {true, true, false, false};
    case XC_OP_EQ: return {false, true, false, false};
    default: return {false, true, false, true};
  }
}
__device__ __forceinline__ bool cmp_rt(const OpMask& m, float x, float t) {
  const bool r = ((x < t) & m.L) | ((x == t) & m.E) | ((x > t) & m.G);
  return r != m.N;
}

// RED: XC_RL_MAX / SUM / COUNT keep a single accumulator (the heat-wave indices); kRunAny keeps every
// accumulator and picks `reducer` at the end.
// GTGT: both operators are ">" (the heat-wave indices and tx_tn_days_above): two compares and one
// predicate op per element pair instead of the six + six of the operator masks.
template <int VEC, int RED, bool GTGT>
__global__ void __launch_bounds__(kThreads)
period_runstat2_kernel(const float* __restrict__ x1, const float* __restrict__ x2, int64_t T, int64_t C, int64_t ldx,
                       const int32_t* __restrict__ poff, OpMask op1, float t1, OpMask op2, float t2, int any,
                       int reducer, int window, int after, float* __restrict__ out) {
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], tend = poff[p + 1];
  int32_t cur[VEC];
  PeriodMask pm[VEC];
  RunAcc<RED> acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { cur[i] = 0; pm[i].init(); acc[i].init(); }
  auto cond = [&](float u, float v) -> bool {
    bool c1, c2;
    if constexpr (GTGT) {
      c1 = u > t1;
      c2 = v > t2;
    } else {
      c1 = cmp_rt(op1, u, t1);
      c2 = cmp_rt(op2, v, t2);
    }
    return any ? (c1 | c2) : (c1 & c2);
  };
  auto load = [&](int t, Vec<VEC>& u, Vec<VEC>& v) {
    u.load(x1 + (int64_t)t * ldx + c0);
    v.load(x2 + (int64_t)t * ldx + c0);
  };
  if (after && t0 > 0) {
    Vec<VEC> u, v;
    load(t0 - 1, u, v);
#pragma unroll
    for (int i = 0; i < VEC; ++i) pm[i].look_back(cond(u.v[i], v.v[i]));
  }
  auto step = [&](const Vec<VEC>& u, const Vec<VEC>& v) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) run_step(cur[i], acc[i], pm[i].inside(after, cond(u.v[i], v.v[i])), window);
  };
  int t = t0;
  for (; t + kUnroll <= tend; t += kUnroll) {
    Vec<VEC> u[kUnroll], v[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) load(t + k, u[k], v[k]);
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) step(u[k], v[k]);
  }
  for (; t < tend; ++t) {
    Vec<VEC> u, v;
    load(t, u, v);
    step(u, v);
  }
  if (after) {
    bool open = false;
#pragma unroll
    for (int i = 0; i < VEC; ++i) open = open || (cur[i] > 0);
    for (; open && t < (int)T; ++t) {
      Vec<VEC> u, v;
      load(t, u, v);
      open = false;
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const bool m = PeriodMask::past_end(cond(u.v[i], v.v[i]), cur[i] > 0);
        run_step(cur[i], acc[i], m, window);
        open = open || m;
      }
    }
  }
  float res[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    run_close(cur[i], acc[i], window);
    res[i] = acc[i].result(reducer);
  }
  store_vec<VEC>(out + (int64_t)p * C + c0, res);
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int32_t xc_period_runstat2_f32(const float* x1, const float* x2, int64_t T, int64_t C, int64_t ldx,
                                          const int32_t* period_offsets, int32_t P, int32_t op1, double thr1,
                                          int32_t op2, double thr2, int32_t var_any, int32_t reducer,
                                          int32_t window, int32_t resample_before_rl, float* out, void* stream) {
  XC_REQUIRE(x1 && x2 && period_offsets && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1, "window must be >= 1");
  XC_REQUIRE(op1 >= XC_OP_GT && op1 <= XC_OP_NE && op2 >= XC_OP_GT && op2 <= XC_OP_NE, "Operation not recognized.");
  XC_REQUIRE(reducer >= XC_RL_MAX && reducer <= XC_RL_STD, "unknown run-length reducer %d", reducer);
  const bool v4 = (C % 4 == 0) && (ldx % 4 == 0) && aligned16(x1) && aligned16(x2) && aligned16(out);
  const int vec = v4 ? 4 : 1;
  dim3 grid((unsigned)(((C + vec - 1) / vec + kThreads - 1) / kThreads), (unsigned)P, 1);
  cudaStream_t st = (cudaStream_t)stream;
  // thresholds are Python floats in the reference: compared in float32
  const OpMask m1 = op_mask(op1), m2 = op_mask(op2);
  const int anyf = var_any ? 1 : 0, afterf = resample_before_rl ? 0 : 1;
  const bool gtgt = (op1 == XC_OP_GT) && (op2 == XC_OP_GT);
#define XC_LAUNCH2(VEC, RED)                                                                                       \
  do {                                                                                                             \
    if (gtgt)                                                                                                      \
      period_runstat2_kernel<VEC, RED, true><<<grid, kThreads, 0, st>>>(                                           \
          x1, x2, T, C, ldx, period_offsets, m1, (float)thr1, m2, (float)thr2, anyf, reducer, window, afterf, out); \
    else                                                                                                           \
      period_runstat2_kernel<VEC, RED, false><<<grid, kThreads, 0, st>>>(                                          \
          x1, x2, T, C, ldx, period_offsets, m1, (float)thr1, m2, (float)thr2, anyf, reducer, window, afterf, out); \
  } while (0)
  if (v4) {
    switch (reducer) {
      case XC_RL_MAX: XC_LAUNCH2(4, XC_RL_MAX); break;
      case XC_RL_SUM: XC_LAUNCH2(4, XC_RL_SUM); break;
      case XC_RL_COUNT: XC_LAUNCH2(4, XC_RL_COUNT); break;
      default: XC_LAUNCH2(4, kRunAny);
    }
  } else {
    XC_LAUNCH2(1, kRunAny);
  }
#undef XC_LAUNCH2
  return launch_status("period_runstat2_kernel");
}
