// Hyndman-Fan quantile finalisation shared by the percentile_doy and bootstrap kernels.
//
// Follows core/utils.py of the reference bit for bit:
//   :370-395  virtual index        vi = n*q + (alpha + q*(1 - alpha - beta)) - 1        (float64)
//   :417-461  neighbour indexes    vi >= n-1 -> max ; vi < 0 -> min ; n < 2 -> the lone value / NaN
//   :464-491  lerp                 diff = right - left in the DATA dtype (float32), weight float64,
//                                  left + diff*g  if g < 0.5 else  right - diff*(1-g)
// All float64 products/sums use the *_rn intrinsics so that nvcc cannot contract them into FMAs
// (numpy evaluates each operation separately).
#pragma once
#include "common.cuh"

namespace xc {

#define XC_NEG_INF (__int_as_float(0xff800000))

struct QuantSpec {
  double q;      // quantile in [0, 1]
  double c;      // alpha + q*(1 - alpha - beta)   (evaluated on the host with the same operations)
  int top;       // 1: list holds the LARGEST values, descending; 0: the SMALLEST (negated), ascending
};

// host: number of order statistics that must be kept for samples of up to n_max values
// (returns the list length needed on the chosen side and fills spec).
inline int plan_quantile(double per, double alpha, double beta, int n_max, QuantSpec* spec) {
  const double q = per / 100.0;
  const double c = alpha + q * (1 - alpha - beta);
  int ktop = 1, kbot = 1;
  for (int n = 2; n <= n_max; ++n) {
    const double vi = (double)n * q + c - 1;
    if (vi >= n - 1 || vi < 0) continue;
    const int lo = (int)floor(vi);
    if (n - lo > ktop) ktop = n - lo;   // needs sorted[n-1-lo], sorted[n-2-lo] counted from the top
    if (lo + 2 > kbot) kbot = lo + 2;   // needs sorted[lo], sorted[lo+1] counted from the bottom
  }
  spec->q = q;
  spec->c = c;
  // the clamps need the extreme of the kept side: vi >= n-1 -> max (top side), vi < 0 -> min (bottom)
  bool top_ok = true, bot_ok = true;
  for (int n = 2; n <= n_max; ++n) {
    const double vi = (double)n * q + c - 1;
    if (vi < 0) top_ok = false;
    if (vi >= n - 1) bot_ok = false;
  }
  if (top_ok && (ktop <= kbot || !bot_ok)) { spec->top = 1; return ktop; }
  if (bot_ok) { spec->top = 0; return kbot; }
  return -1;  // alpha/beta outside [0, 1] with a mid quantile: not supported
}

// inserts v into the descending list lst, dropping its smallest entry (2K min/max)
template <int K>
__device__ __forceinline__ void insert_desc(float (&lst)[K], float v) {
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float hi = fmaxf(lst[k], v);
    v = fminf(lst[k], v);
    lst[k] = hi;
  }
}

template <int K>
__device__ __forceinline__ float pick(const float (&lst)[K], int idx) {
  float v = lst[0];
#pragma unroll
  for (int k = 1; k < K; ++k) v = (idx == k) ? lst[k] : v;
  return v;
}

// lst: the K extreme values of the sample on the chosen side, sorted (largest first on the top
// side; on the bottom side the values are NEGATED so "largest first" is smallest x first).
// n: number of non-NaN values in the whole sample.
template <int K>
__device__ __forceinline__ double finalize_quantile(const float (&lst)[K], int n, const QuantSpec& s) {
  if (n == 0) return __longlong_as_double(0x7ff8000000000000LL);
  const float sgn = s.top ? 1.f : -1.f;
  if (n == 1) return (double)(sgn * lst[0]);
  const double nd = (double)n;
  const double vi = __dadd_rn(__dadd_rn(__dmul_rn(nd, s.q), s.c), -1.0);
  if (s.top) {
    if (vi >= nd - 1.0) return (double)lst[0];
  } else {
    // both neighbours clamp to the minimum; for a -inf minimum their difference is NaN, which the caller
    // replaces by the sample maximum (lerp_is_nan)
    if (vi < 0.0) return isinf(lst[0]) ? __longlong_as_double(0x7ff8000000000000LL) : (double)(-lst[0]);
  }
  const double lo = floor(vi);
  const int ilo = (int)lo;
  float left, right;
  if (s.top) {
    left = pick<K>(lst, n - 1 - ilo);
    right = pick<K>(lst, n - 2 - ilo);
  } else {
    left = -pick<K>(lst, ilo);
    right = -pick<K>(lst, ilo + 1);
  }
  const double g = __dadd_rn(vi, -lo);
  const float diff = __fsub_rn(right, left);
  double r;
  if (g >= 0.5)
    r = __dadd_rn((double)right, -__dmul_rn((double)diff, __dadd_rn(1.0, -g)));
  else
    r = __dadd_rn((double)left, __dmul_rn((double)diff, g));
  return r;
}


// Per-lane virtual index pieces, shared by the full and the rank-only finalisation.
struct QuantIdx {
  double vi, lo;
  int ilo;
};
__device__ __forceinline__ QuantIdx quant_index(int n, const QuantSpec& s) {
  QuantIdx r;
  r.vi = __dadd_rn(__dadd_rn(__dmul_rn((double)n, s.q), s.c), -1.0);
  r.lo = floor(r.vi);
  r.ilo = (int)r.lo;
  return r;
}
// lerp of core/utils.py:464-491 given the two neighbours (already de-negated)
__device__ __forceinline__ double quant_lerp(float left, float right, const QuantIdx& qi) {
  const double g = __dadd_rn(qi.vi, -qi.lo);
  const float diff = __fsub_rn(right, left);
  if (g >= 0.5) return __dadd_rn((double)right, -__dmul_rn((double)diff, __dadd_rn(1.0, -g)));
  return __dadd_rn((double)left, __dmul_rn((double)diff, g));
}

// core/utils.py:554: an interpolation that comes out NaN (an infinite neighbour, or two neighbours whose
// difference overflows float32) is replaced by the largest value of the sample.  With n >= 2 values a NaN
// result can only come from there, so the kernels test the result after the lerp and only then look the
// maximum up (the bottom-side lists do not hold it).
__device__ __forceinline__ bool lerp_is_nan(double r, int n) { return n >= 2 && r != r; }

}  // namespace xc
