// Ensemble robustness: the Student-t distribution and the per-member t-tests, shared by the CUDA kernel
// (ensemble.cu) and by a host build of the very same code that the CPU test-suite checks against
// scipy.special.stdtr (tests/csrc/ensemble_host.cpp).
//
// Replaces the p-values of ensembles/_robustness.py `_ttest` (:518-549: scipy.stats.ttest_1samp against the
// reference mean) and `_welch_ttest` (:552-581: scipy.stats.ttest_ind(equal_var=False)), both with
// nan_policy="omit".  Everything is float64: scipy evaluates these tests in float32 for float32 samples, so the
// kernel's p-values are the more accurate ones, not scipy's bits (DESIGN.md section 4).
//
// The t distribution function is the regularised incomplete beta I_x(df/2, 1/2), x = df / (df + t^2), evaluated
// by its continued fraction (modified Lentz), with the symmetry I_x(a, b) = 1 - I_{1-x}(b, a) above the
// fraction's convergence point.  The prefactor x^a (1-x)^b / B(a, b) is taken in logs with
// ln Gamma(a + 1/2) - ln Gamma(a) written from the Stirling series for large a, so it keeps its relative
// accuracy up to df = 1e4 and beyond.  Compile WITHOUT floating-point contraction (nvcc -fmad=false,
// g++ -ffp-contract=off) so that both builds round the same way.
#pragma once
#include <math.h>
#include <stdint.h>

#include "stdindex_core.cuh"

#if defined(__CUDACC__)
#define XC_ENS_HD __host__ __device__ __forceinline__
#else
#define XC_ENS_HD inline
#endif

namespace xc {
namespace ens {

constexpr double kLnSqrtPi = 0.57236494292470008707;   // ln Gamma(1/2)
constexpr int kMaxIter = 20000;                        // continued-fraction terms (df = 1e6 needs ~1500)

// ln(Gamma(a + 1/2) / Gamma(a)), a > 0
XC_ENS_HD double log_gamma_half_ratio(double a) {
  if (a < 10.0) return log(si::gamma_lanczos(a + 0.5) / si::gamma_lanczos(a));
  // lnGamma(z) = (z - 1/2) ln z - z + ln(2 pi) / 2 + lgs(z): the difference has no large terms left
  return a * log1p(0.5 / a) - 0.5 + 0.5 * log(a) + si::log_gamma_star(a + 0.5) - si::log_gamma_star(a);
}

// Continued fraction of I_x(a, b) / (x^a (1-x)^b / (a B(a, b))) (modified Lentz); converges fast for
// x < (a + 1) / (a + b + 2).
XC_ENS_HD double beta_cf(double a, double b, double x) {
  const double tiny = 1e-300, eps = 2.220446049250313e-16;
  const double qab = a + b, qap = a + 1.0, qam = a - 1.0;
  double c = 1.0, d = 1.0 - qab * x / qap;
  if (fabs(d) < tiny) d = tiny;
  d = 1.0 / d;
  double h = d;
  for (int m = 1; m <= kMaxIter; ++m) {
    const double m2 = 2.0 * m;
    double aa = m * (b - m) * x / ((qam + m2) * (a + m2));
    d = 1.0 + aa * d;
    if (fabs(d) < tiny) d = tiny;
    c = 1.0 + aa / c;
    if (fabs(c) < tiny) c = tiny;
    d = 1.0 / d;
    h *= d * c;
    aa = -(a + m) * (qab + m) * x / ((a + m2) * (qap + m2));
    d = 1.0 + aa * d;
    if (fabs(d) < tiny) d = tiny;
    c = 1.0 + aa / c;
    if (fabs(c) < tiny) c = tiny;
    d = 1.0 / d;
    const double del = d * c;
    h *= del;
    if (fabs(del - 1.0) < eps) break;
  }
  return h;
}

// P(T < t) for Student's t with df > 0 degrees of freedom (scipy.special.stdtr(df, t)); NaN for a NaN
// argument or df <= 0.
XC_ENS_HD double stdtr(double df, double t) {
  if (t != t || df != df || !(df > 0.0)) return NAN;
  if (t == 0.0) return 0.5;
  if (isinf(t)) return t > 0.0 ? 1.0 : 0.0;
  const double a = 0.5 * df, b = 0.5;
  const double t2 = t * t;
  double x, y, lx, ly;   // x = df / (df + t^2), y = 1 - x, and their logs
  if (isinf(t2)) {
    x = 0.0;
    y = 1.0;
    lx = log(df) - 2.0 * log(fabs(t));
    ly = 0.0;
  } else {
    x = df / (df + t2);
    y = t2 / (df + t2);
    lx = -log1p(t2 / df);
    ly = -log1p(df / t2);
  }
  // f = x^a y^b / B(a, b), B(a, 1/2) = Gamma(a) Gamma(1/2) / Gamma(a + 1/2).  In the far tail (x < 1/2) the
  // log of f is large and its last bit would cost ~|ln f| ulp in exp(): take x^a by pow there.  Near the centre
  // x = 1 - O(1/df), and a * log1p(t^2 / df) keeps the relative accuracy that pow(x, a) would lose.
  const double lg = log_gamma_half_ratio(a) - kLnSqrtPi;
  const double f = (x < 0.5 && x > 0.0) ? pow(x, a) * sqrt(y) * exp(lg) : exp(a * lx + b * ly + lg);
  double tail;   // P(T < -|t|) = I_x(a, b) / 2
  if (x < (a + 1.0) / (a + b + 2.0))
    tail = 0.5 * (f * beta_cf(a, b, x) / a);
  else
    tail = 0.5 * (1.0 - f * beta_cf(b, a, y) / b);
  return t < 0.0 ? tail : 1.0 - tail;
}

// two-sided p-value of a t statistic (NaN stays NaN, +-inf gives 0)
XC_ENS_HD double t_pvalue(double t, double df) { return 2.0 * stdtr(df, -fabs(t)); }

// scipy.stats.ttest_1samp(f, popmean, nan_policy="omit")[1] from the n non-NaN values of f, their mean m and
// ss = sum((f - m)^2): ddof-1 variance, df = n - 1 (NaN below 2 values).
XC_ENS_HD double ttest_1samp_p(int n, double m, double ss, double popmean) {
  const double v = ss / (double)(n - 1);
  const double t = (m - popmean) / sqrt(v / (double)n);
  return t_pvalue(t, (double)(n - 1));
}

// scipy.stats.ttest_ind(f, r, equal_var=False, nan_policy="omit")[1]: Welch's t with the Welch-Satterthwaite
// df, which scipy sets to 1 where it is undefined (both variances zero).
XC_ENS_HD double welch_ttest_p(int n1, double m1, double ss1, int n2, double m2, double ss2) {
  const double vn1 = ss1 / (double)(n1 - 1) / (double)n1;
  const double vn2 = ss2 / (double)(n2 - 1) / (double)n2;
  const double s = vn1 + vn2;
  double df = s * s / (vn1 * vn1 / (double)(n1 - 1) + vn2 * vn2 / (double)(n2 - 1));
  if (df != df) df = 1.0;
  const double t = (m1 - m2) / sqrt(s);
  return t_pvalue(t, df);
}

// Standard deviation (ddof 0) of the residuals of the least-squares line through the non-NaN points (x[p], y(p)),
// p < P: `detrend(refy, deg=1).std("time")` of _robustness.py:653-654 (xarray's polyfit and polyval on the time
// coordinate, the residuals, their NaN-skipping std).  x holds the actual YS timestamps (any origin and unit: the
// residuals of a line do not depend on them), so leap years weigh in.  NaN without points; 0 with one.
template <class Y>
XC_ENS_HD double detrended_std(Y y, const double* x, int64_t P) {
  int n = 0;
  double sx = 0.0, sy = 0.0;
  for (int64_t p = 0; p < P; ++p) {
    const double v = y(p);
    if (v == v) {
      sx += x[p];
      sy += v;
      ++n;
    }
  }
  if (n == 0) return NAN;
  const double mx = sx / n, my = sy / n;
  double sxx = 0.0, sxy = 0.0;
  for (int64_t p = 0; p < P; ++p) {
    const double v = y(p);
    if (v == v) {
      const double dx = x[p] - mx;
      sxx += dx * dx;
      sxy += dx * (v - my);
    }
  }
  const double b = sxx > 0.0 ? sxy / sxx : 0.0;
  double ss = 0.0;
  for (int64_t p = 0; p < P; ++p) {
    const double v = y(p);
    if (v == v) {
      const double r = (v - my) - b * (x[p] - mx);
      ss += r * r;
    }
  }
  return sqrt(ss / n);
}

// the ipcc-ar6-c threshold without pre-industrial data: sqrt(2 / 20) * 1.645 * sigma_1yr (_robustness.py:654)
XC_ENS_HD double ipcc_ar6_c_gamma(double sigma) { return sqrt(2.0 / 20.0) * 1.645 * sigma; }

}  // namespace ens
}  // namespace xc
