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
// THR1 / THR2: the threshold sources of the two variables (runstat.cuh): scalars, or day-of-year tables (the
// compound percentile days, indices/_multivariate.py:162-416).
template <int VEC, int RED, bool GTGT, typename THR1 = ScalarThr, typename THR2 = ScalarThr>
__global__ void __launch_bounds__(kThreads)
period_runstat2_kernel(const float* __restrict__ x1, const float* __restrict__ x2, int64_t T, int64_t C, int64_t ldx,
                       const int32_t* __restrict__ poff, OpMask op1, THR1 t1, OpMask op2, THR2 t2, int any,
                       int reducer, int window, int after, float* __restrict__ out) {
  using Row1 = typename THR1::template Row<VEC>;
  using Row2 = typename THR2::template Row<VEC>;
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], tend = poff[p + 1];
  int32_t cur[VEC];
  PeriodMask pm[VEC];
  RunAcc<RED> acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { cur[i] = 0; pm[i].init(); acc[i].init(); }
  auto cond = [&](float u, float v, const Row1& h1, const Row2& h2, int i) -> bool {
    bool c1, c2;
    if constexpr (GTGT) {
      c1 = u > t1.at(h1, i);
      c2 = v > t2.at(h2, i);
    } else {
      c1 = cmp_rt(op1, u, t1.at(h1, i));
      c2 = cmp_rt(op2, v, t2.at(h2, i));
    }
    return any ? (c1 | c2) : (c1 & c2);
  };
  auto load = [&](int t, Vec<VEC>& u, Vec<VEC>& v, Row1& h1, Row2& h2) {
    u.load(x1 + (int64_t)t * ldx + c0);
    v.load(x2 + (int64_t)t * ldx + c0);
    t1.load(h1, c0, t);
    t2.load(h2, c0, t);
  };
  if (after && t0 > 0) {
    Vec<VEC> u, v;
    Row1 h1;
    Row2 h2;
    load(t0 - 1, u, v, h1, h2);
#pragma unroll
    for (int i = 0; i < VEC; ++i) pm[i].look_back(cond(u.v[i], v.v[i], h1, h2, i));
  }
  auto step = [&](const Vec<VEC>& u, const Vec<VEC>& v, const Row1& h1, const Row2& h2) {
#pragma unroll
    for (int i = 0; i < VEC; ++i)
      run_step(cur[i], acc[i], pm[i].inside(after, cond(u.v[i], v.v[i], h1, h2, i)), window);
  };
  int t = t0;
  for (; t + kUnroll <= tend; t += kUnroll) {
    Vec<VEC> u[kUnroll], v[kUnroll];
    Row1 h1[kUnroll];
    Row2 h2[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) load(t + k, u[k], v[k], h1[k], h2[k]);
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) step(u[k], v[k], h1[k], h2[k]);
  }
  for (; t < tend; ++t) {
    Vec<VEC> u, v;
    Row1 h1;
    Row2 h2;
    load(t, u, v, h1, h2);
    step(u, v, h1, h2);
  }
  if (after) {
    bool open = false;
#pragma unroll
    for (int i = 0; i < VEC; ++i) open = open || (cur[i] > 0);
    for (; open && t < (int)T; ++t) {
      Vec<VEC> u, v;
      Row1 h1;
      Row2 h2;
      load(t, u, v, h1, h2);
      open = false;
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const bool m = PeriodMask::past_end(cond(u.v[i], v.v[i], h1, h2, i), cur[i] > 0);
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

// Per-period statistic of the daily range d[t] = hi[t] - lo[t], formed in float32 (indices/_multivariate.py:514-557,
// `daily_temperature_range`: `select_resample_op(tasmax - tasmin, op)`), NaN skipped as xc_period_reduce_f32 does.
// VAR: the mean of |d[t] - d[t-1]| instead (:561-598, `daily_temperature_range_variability`): the difference
// labelled with its later step, so that a period's first difference reaches back to the previous period's last day
// and the series' first step has none.  Both inputs are read once; d is never stored.
template <int VEC, bool VAR>
__global__ void __launch_bounds__(kThreads)
period_range_stat_kernel(const float* __restrict__ lo, const float* __restrict__ hi, int64_t C, int64_t ldx,
                         const int32_t* __restrict__ poff, int stat, float* __restrict__ out) {
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], tend = poff[p + 1];
  StatAcc acc[VEC];
  float prev[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { acc[i].init(stat); prev[i] = NAN; }
  auto load = [&](int t, Vec<VEC>& a, Vec<VEC>& b) {
    a.load(lo + (int64_t)t * ldx + c0);
    b.load(hi + (int64_t)t * ldx + c0);
  };
  if (VAR && t0 > 0) {
    Vec<VEC> a, b;
    load(t0 - 1, a, b);
#pragma unroll
    for (int i = 0; i < VEC; ++i) prev[i] = b.v[i] - a.v[i];
  }
  auto step = [&](const Vec<VEC>& a, const Vec<VEC>& b) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float d = b.v[i] - a.v[i];
      if constexpr (VAR) {
        acc[i].take(fabsf(d - prev[i]));
        prev[i] = d;
      } else {
        acc[i].take(d);
      }
    }
  };
  int t = t0;
  for (; t + kUnroll <= tend; t += kUnroll) {
    Vec<VEC> a[kUnroll], b[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) load(t + k, a[k], b[k]);
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) step(a[k], b[k]);
  }
  for (; t < tend; ++t) {
    Vec<VEC> a, b;
    load(t, a, b);
    step(a, b);
  }
  float res[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) res[i] = acc[i].result(stat);
  store_vec<VEC>(out + (int64_t)p * C + c0, res);
}

inline bool pair_vec4(const float* a, const float* b, int64_t C, int64_t ldx, const void* out) {
  return (C % 4 == 0) && (ldx % 4 == 0) && aligned16(a) && aligned16(b) && aligned16(out);
}

inline dim3 pair_grid(int64_t C, bool v4, int32_t P) {
  const int vec = v4 ? 4 : 1;
  return dim3((unsigned)(((C + vec - 1) / vec + kThreads - 1) / kThreads), (unsigned)P, 1);
}

template <typename F>
int32_t dispatch_order_op(int32_t op, F&& f) {
  switch (op) {
    case XC_OP_GT: return f(std::integral_constant<int, XC_OP_GT>{});
    case XC_OP_LT: return f(std::integral_constant<int, XC_OP_LT>{});
    case XC_OP_GE: return f(std::integral_constant<int, XC_OP_GE>{});
    default: return f(std::integral_constant<int, XC_OP_LE>{});
  }
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
          x1, x2, T, C, ldx, period_offsets, m1, ScalarThr{(float)thr1}, m2, ScalarThr{(float)thr2}, anyf, reducer, \
          window, afterf, out);                                                                                    \
    else                                                                                                           \
      period_runstat2_kernel<VEC, RED, false><<<grid, kThreads, 0, st>>>(                                          \
          x1, x2, T, C, ldx, period_offsets, m1, ScalarThr{(float)thr1}, m2, ScalarThr{(float)thr2}, anyf, reducer, \
          window, afterf, out);                                                                                    \
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

extern "C" int32_t xc_doy_count2_f32(const float* x1, const float* x2, int64_t T, int64_t C, int64_t ldx,
                                     const int32_t* period_offsets, int32_t P, const int16_t* doy_index,
                                     const double* table1, const double* table2, int32_t n_doy, int32_t op1,
                                     int32_t op2, float* out, void* stream) {
  XC_REQUIRE(x1 && x2 && period_offsets && doy_index && table1 && table2 && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL && n_doy > 0, "bad shape");
  XC_REQUIRE(op1 >= XC_OP_GT && op1 <= XC_OP_LE && op2 >= XC_OP_GT && op2 <= XC_OP_LE,
             "Operation not permitted for indice.");
  const bool v4 = pair_vec4(x1, x2, C, ldx, out) && aligned16(table1) && aligned16(table2);
  const dim3 grid = pair_grid(C, v4, P);
  cudaStream_t st = (cudaStream_t)stream;
  const OpMask m1 = op_mask(op1), m2 = op_mask(op2);
  // windowed_run_count with window 1 of the AND of the two table tests, runs cut at the period edges: the count
  return dispatch_order_op(op1, [&](auto O1) -> int32_t {
    return dispatch_order_op(op2, [&](auto O2) -> int32_t {
      constexpr int OP1 = decltype(O1)::value, OP2 = decltype(O2)::value;
      constexpr bool GTGT = OP1 == XC_OP_GT && OP2 == XC_OP_GT;
      using S1 = TableThr<OP1, true>;
      using S2 = TableThr<OP2, true>;
      const S1 s1{doy_index, table1, C};
      const S2 s2{doy_index, table2, C};
      if (v4)
        period_runstat2_kernel<4, XC_RL_SUM, GTGT, S1, S2><<<grid, kThreads, 0, st>>>(
            x1, x2, T, C, ldx, period_offsets, m1, s1, m2, s2, 0, XC_RL_SUM, 1, 0, out);
      else
        period_runstat2_kernel<1, XC_RL_SUM, GTGT, S1, S2><<<grid, kThreads, 0, st>>>(
            x1, x2, T, C, ldx, period_offsets, m1, s1, m2, s2, 0, XC_RL_SUM, 1, 0, out);
      return launch_status("period_runstat2_kernel");
    });
  });
}

extern "C" int32_t xc_period_range_stat_f32(const float* lo, const float* hi, int64_t T, int64_t C, int64_t ldx,
                                            const int32_t* period_offsets, int32_t P, int32_t stat,
                                            int32_t variability, float* out, void* stream) {
  XC_REQUIRE(lo && hi && period_offsets && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(stat >= XC_STAT_SUM && stat <= XC_STAT_COUNT, "unknown reduction %d", stat);
  XC_REQUIRE(!variability || stat == XC_STAT_MEAN, "the variability is a mean (stat %d given)", stat);
  const bool v4 = pair_vec4(lo, hi, C, ldx, out);
  const dim3 grid = pair_grid(C, v4, P);
  cudaStream_t st = (cudaStream_t)stream;
  if (v4) {
    if (variability)
      period_range_stat_kernel<4, true><<<grid, kThreads, 0, st>>>(lo, hi, C, ldx, period_offsets, stat, out);
    else
      period_range_stat_kernel<4, false><<<grid, kThreads, 0, st>>>(lo, hi, C, ldx, period_offsets, stat, out);
  } else {
    if (variability)
      period_range_stat_kernel<1, true><<<grid, kThreads, 0, st>>>(lo, hi, C, ldx, period_offsets, stat, out);
    else
      period_range_stat_kernel<1, false><<<grid, kThreads, 0, st>>>(lo, hi, C, ldx, period_offsets, stat, out);
  }
  return launch_status("period_range_stat_kernel");
}
