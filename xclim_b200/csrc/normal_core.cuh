// The standard normal CDF and its inverse (Phi, ndtri) for host and device, shared by the standardized-index
// transform (stdindex_core.cuh) and the frequency-analysis transform (evfit_core.cuh).  Written from the published
// algorithms with exp / log / sqrt / expm1 only, so the CPU test-suite's host builds run the same code as the
// device.  Compile WITHOUT floating-point contraction (nvcc -fmad=false, g++ -ffp-contract=off).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define XC_NRM_HD __host__ __device__ __forceinline__
#define XC_NRM_HDN static __host__ __device__ __noinline__   // static: included by several translation units
#else
#define XC_NRM_HD inline
#define XC_NRM_HDN inline
#endif

namespace xc {
namespace si {

constexpr double kSqrt2Pi = 2.5066282746310002;     // sqrt(2 pi)
constexpr double kSqrtPi = 1.7724538509055160;      // Gamma(1/2)

// P(1/2, y) = erf(sqrt(y)) for 0 <= y < 1.5 by the power series (relative accuracy: no cancellation).
XC_NRM_HD double erf_sqrt_series(double y) {
  if (y == 0.0) return 0.0;
  const double f = exp(0.5 * log(y) - y) / kSqrtPi;
  double term = 1.0, sum = 1.0;
  for (int n = 1; n < 200; ++n) {
    term *= y / (0.5 + (double)n);
    sum += term;
    if (term < sum * 1e-17) break;
  }
  return f / 0.5 * sum;
}

// The Legendre continued fraction of Q(1/2, y) without its prefactor y^(1/2) e^-y / Gamma(1/2), y >= 1.5.
XC_NRM_HD double erfc_cf_scaled(double y) {
  const double tiny = 1e-300;
  double b = y + 0.5, c = 1.0 / tiny, dd = 1.0 / b, h = dd;
  for (int n = 1; n < 2000; ++n) {
    const double an = -(double)n * ((double)n - 0.5);
    b += 2.0;
    dd = an * dd + b;
    if (fabs(dd) < tiny) dd = tiny;
    c = b + an / c;
    if (fabs(c) < tiny) c = tiny;
    dd = 1.0 / dd;
    const double del = dd * c;
    h *= del;
    if (fabs(del - 1.0) < 1e-16) break;
  }
  return h;
}

// Upper tail Q(1/2, y) = erfc(sqrt(y)) for y >= 0, the same two expansions with the constant Gamma(1/2).
XC_NRM_HD double erfc_sqrt(double y) {
  if (isinf(y)) return 0.0;
  if (y < 1.5) return 1.0 - erf_sqrt_series(y);
  return exp(0.5 * log(y) - y) / kSqrtPi * erfc_cf_scaled(y);
}

// Standard normal CDF Phi(z) = erfc(-z / sqrt 2) / 2.
XC_NRM_HDN double ndtr(double z) {
  if (z != z) return NAN;
  const double q = 0.5 * erfc_sqrt(0.5 * (z * z));
  return z < 0.0 ? q : 1.0 - q;
}

// Inverse of Phi: Acklam's rational approximation (relative error 1.2e-9) refined by two Halley steps on the
// lower half; p > 1/2 through the exact complement 1 - p.
XC_NRM_HDN double ndtri(double p) {
  if (p != p || p < 0.0 || p > 1.0) return NAN;
  if (p == 0.0) return -INFINITY;
  if (p == 1.0) return INFINITY;
  const bool upper = p > 0.5;
  const double q = upper ? 1.0 - p : p;
  double x;
  if (q < 0.02425) {
    const double r = sqrt(-2.0 * log(q));
    x = (((((-7.784894002430293e-03 * r - 3.223964580411365e-01) * r - 2.400758277161838e+00) * r -
           2.549732539343734e+00) * r + 4.374664141464968e+00) * r + 2.938163982698783e+00) /
        ((((7.784695709041462e-03 * r + 3.224671290700398e-01) * r + 2.445134137142996e+00) * r +
          3.754408661907416e+00) * r + 1.0);
  } else {
    const double r0 = q - 0.5, r = r0 * r0;
    x = (((((-3.969683028665376e+01 * r + 2.209460984245205e+02) * r - 2.759285104469687e+02) * r +
           1.383577518672690e+02) * r - 3.066479806614716e+01) * r + 2.506628277459239e+00) * r0 /
        (((((-5.447609879822406e+01 * r + 1.615858368580409e+02) * r - 1.556989798598866e+02) * r +
           6.680131188771972e+01) * r - 1.328068155288572e+01) * r + 1.0);
  }
  const double log_q = log(q);
  for (int it = 0; it < 2; ++it) {           // Halley on Phi(x) = q, x <= 0, with u = (Phi(x) - q) / phi(x)
    const double y = 0.5 * (x * x);
    double u;
    if (y < 1.5) {
      // in the centre as (1/2 - q) - erf(|x| / sqrt 2) / 2, both terms exact or accurate to an ulp
      u = ((0.5 - q) - 0.5 * erf_sqrt_series(y)) * kSqrt2Pi * exp(y);
    } else {
      // in the tail through logarithms, (Phi / q - 1) (q / phi): Phi, q and phi underflow to subnormals or zero
      // below q ~ 1e-308 while both ratios stay near 1 and 1 / |x|
      const double log_phi_cdf = log(0.5 * erfc_cf_scaled(y)) + 0.5 * log(y) - y - 0.5723649429247001;
      u = expm1(log_phi_cdf - log_q) * exp(log_q + y + 0.9189385332046728);
    }
    x = x - u / (1.0 + 0.5 * x * u);
  }
  return upper ? -x : x;
}

}  // namespace si
}  // namespace xc
