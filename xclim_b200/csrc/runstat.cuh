// Run-length reducers and per-period statistics shared by the streaming kernels: one copy of the rules.
#pragma once
#include "common.cuh"

namespace xc {

// Reducer value of a RunAcc that keeps every quantity and picks the reducer at run time (result(int)).
constexpr int kRunAny = -1;

// mean and std of n run lengths with sum s and sum of squares q; 0 when there is no run
__device__ __forceinline__ float run_mean(int32_t n, int32_t s) {
  return n == 0 ? 0.f : (float)((double)s / (double)n);
}
__device__ __forceinline__ float run_std(int32_t n, int32_t s, unsigned long long q) {
  if (n == 0) return 0.f;
  double nn = (double)n, m = (double)s / nn;
  double var = (double)q / nn - m * m;
  return (float)sqrt(var > 0.0 ? var : 0.0);
}

// Per-cell accumulator over the run lengths L >= window attributed to the period.
template <int RED>
struct RunAcc {
  int32_t a;        // MAX: max L ; MIN: min L ; SUM: sum L ; COUNT/MEAN/STD/any: n runs
  int32_t s;        // MEAN/STD/any: sum L
  unsigned long long q;  // STD/any: sum L^2
  int32_t mx, mn;   // any: max L, min L
  __device__ __forceinline__ void init() {
    a = (RED == XC_RL_MIN) ? 0x7fffffff : 0;
    s = 0;
    q = 0ull;
    if constexpr (RED == kRunAny) {
      mx = 0;
      mn = 0x7fffffff;
    }
  }
  __device__ __forceinline__ void add(int32_t L, bool take) {
    if constexpr (RED == XC_RL_MAX) a = take ? max(a, L) : a;
    if constexpr (RED == XC_RL_MIN) a = take ? min(a, L) : a;
    if constexpr (RED == XC_RL_SUM) a += take ? L : 0;
    if constexpr (RED == XC_RL_COUNT) a += take ? 1 : 0;
    if constexpr (RED == XC_RL_MEAN || RED == XC_RL_STD) {
      a += take ? 1 : 0;
      s += take ? L : 0;
    }
    if constexpr (RED == XC_RL_STD) q += take ? (unsigned long long)L * (unsigned long long)L : 0ull;
    if constexpr (RED == kRunAny) {
      // a branch, not selects: five branch-free updates with a 64-bit square cost registers on every step
      if (take) {
        a += 1;
        s += L;
        q += (unsigned long long)L * (unsigned long long)L;
        mx = max(mx, L);
        mn = min(mn, L);
      }
    }
  }
  __device__ __forceinline__ float result() const {
    if constexpr (RED == XC_RL_MAX || RED == XC_RL_SUM || RED == XC_RL_COUNT) return (float)a;
    if constexpr (RED == XC_RL_MIN) return a == 0x7fffffff ? 0.f : (float)a;
    if constexpr (RED == XC_RL_MEAN) return run_mean(a, s);
    if constexpr (RED == XC_RL_STD) return run_std(a, s, q);
    return 0.f;
  }
  // the reducer chosen at run time (any); a fixed RED ignores `reducer`
  __device__ __forceinline__ float result(int reducer) const {
    if constexpr (RED != kRunAny) return result();
    switch (reducer) {
      case XC_RL_MAX: return (float)mx;
      case XC_RL_MIN: return a ? (float)mn : 0.f;
      case XC_RL_SUM: return (float)s;
      case XC_RL_COUNT: return (float)a;
      case XC_RL_MEAN: return run_mean(a, s);
      default: return run_std(a, s, q);
    }
  }
};

// Statistic of n non-NaN values with float64 sum s and sum of squares q and their min or max m.  Mean, min and
// max of no values are NaN; std and var are q/n - mean^2 clamped at 0.
__device__ __forceinline__ float stat_result(int stat, int32_t n, double s, double q, float m) {
  const double nn = (double)n;
  switch (stat) {
    case XC_STAT_SUM: return (float)s;
    case XC_STAT_COUNT: return (float)n;
    case XC_STAT_MEAN: return n ? (float)(s / nn) : NAN;
    case XC_STAT_MIN:
    case XC_STAT_MAX: return n ? m : NAN;
    default: {
      if (!n) return NAN;
      const double mean = s / nn;
      double var = q / nn - mean * mean;
      var = var > 0.0 ? var : 0.0;
      return (stat == XC_STAT_STD) ? (float)sqrt(var) : (float)var;
    }
  }
}

// Per-period statistic `stat` of a stream of values, NaN skipped.
struct StatAcc {
  int32_t n;
  double s, q;
  float m;         // min for XC_STAT_MIN, else max
  bool is_min;
  __device__ __forceinline__ void init(int stat) {
    n = 0;
    s = 0.0;
    q = 0.0;
    is_min = (stat == XC_STAT_MIN);
    m = is_min ? INFINITY : -INFINITY;
  }
  __device__ __forceinline__ void take(float r) {
    if (r == r) {
      ++n;
      s += (double)r;
      q += (double)r * (double)r;
      m = is_min ? fminf(m, r) : fmaxf(m, r);
    }
  }
  __device__ __forceinline__ float result(int stat) const { return stat_result(stat, n, s, q, m); }
};

}  // namespace xc
