// Standardized indices (SPI / SPEI): the per-sample distribution fit and the probability transform, shared by
// the CUDA kernels (stdindex.cu) and by a host build of the very same code that the CPU test-suite checks
// against scipy and the oracle (tests/csrc/stdindex_host.cpp).
//
// Replaces indices/stats.py `_fitfunc_1d` (:45-112) with `_fit_start` (:576-684) for gamma / fisk / lognorm,
// scipy's `gamma_gen.fit` and `lognorm_gen.fit` with a fixed `floc`, and the transform of `standardized_index`
// (:1155-1191): `rv_continuous.cdf`, the zero-inflation algebra, `norm.ppf` and the clip to +-8.21.
//
// Arithmetic follows numpy's for float32 samples: means are float32 pairwise sums (npsum.cuh), the moment
// expressions are float32 (NEP 50: Python scalars take the array's type), and every log / exp of a float32
// value is the float64 function rounded once to float32 (numpy's own float32 log / exp are SIMD code that
// differs between CPUs).  The special functions below are written from the published algorithms and use only
// exp / log / sqrt / pow / fma, so the host build runs the same code as the device.  Compile WITHOUT
// floating-point contraction (nvcc -fmad=false, g++ -ffp-contract=off).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/xclim_b200.h"
#include "normal_core.cuh"
#include "npsum.cuh"

#if defined(__CUDACC__)
#define XC_SI_HD __host__ __device__ __forceinline__
#define XC_SI_HDN static __host__ __device__ __noinline__   // static: ensemble_core.cuh includes this header too
#else
#define XC_SI_HD inline
#define XC_SI_HDN inline
#endif

namespace xc {
namespace si {

constexpr double kPi = 3.14159265358979323846;
constexpr double kClip = 8.21;                      // stats.py:1191
constexpr int kMaxIter = 20000;                     // series / continued fraction terms (a <= 1e5 needs ~3000)

XC_SI_HD float log_f32(float x) { return (float)log((double)x); }
XC_SI_HD float exp_f32(float x) { return (float)exp((double)x); }

// ---- Gamma function pieces ------------------------------------------------------------------------------
// Lanczos approximation (g = 7, n = 9), Gamma(z + 1) = sqrt(2 pi) t^(z + 1/2) e^-t A(z), t = z + 7.5; relative
// error ~1e-15 for 0 < a < 10 (the only range it serves).
XC_SI_HD double gamma_lanczos(double a) {
  const bool small = a < 0.5;                       // Gamma(a) = Gamma(a + 1) / a, without a recursive call
  const double z = small ? a : a - 1.0;
  double s = 0.99999999999980993;
  s += 676.5203681218851 / (z + 1.0);
  s += -1259.1392167224028 / (z + 2.0);
  s += 771.32342877765313 / (z + 3.0);
  s += -176.61502916214059 / (z + 4.0);
  s += 12.507343278686905 / (z + 5.0);
  s += -0.13857109526572012 / (z + 6.0);
  s += 9.9843695780195716e-6 / (z + 7.0);
  s += 1.5056327351493116e-7 / (z + 8.0);
  const double t = z + 7.5;
  const double g = kSqrt2Pi * pow(t, z + 0.5) * exp(-t) * s;
  return small ? g / a : g;
}

// log of Gamma*(a) = Gamma(a) / (sqrt(2 pi / a) (a / e)^a), the Stirling series (a >= 10: the B16 term is
// below 1e-16).
XC_SI_HD double log_gamma_star(double a) {
  const double r = 1.0 / a, r2 = r * r;
  double s = -3617.0 / 122400.0;
  s = s * r2 + 1.0 / 156.0;
  s = s * r2 - 691.0 / 360360.0;
  s = s * r2 + 1.0 / 1188.0;
  s = s * r2 - 1.0 / 1680.0;
  s = s * r2 + 1.0 / 1260.0;
  s = s * r2 - 1.0 / 360.0;
  s = s * r2 + 1.0 / 12.0;
  return s * r;
}

// u - log(1 + u) for |u| < 0.3 by its series (sum over k >= 2 of (-u)^k / k, sign flipped), else directly.
XC_SI_HD double u_minus_log1p(double u) {
  if (fabs(u) >= 0.3) return u - log1p(u);
  double term = u * u, s = 0.0;
  for (int k = 2; k < 60; ++k) {
    const double c = term / (double)k;
    s += (k & 1) ? -c : c;
    term *= u;
    if (fabs(c) < 1e-18 * fabs(s)) break;
  }
  return s;
}

// x^a e^-x / Gamma(a), the prefactor of both incomplete-gamma expansions.  For a >= 10 it is written as
// exp(-a phi(lambda)) sqrt(a / 2 pi) / Gamma*(a) with lambda = x / a and phi = lambda - 1 - log(lambda); the
// rounding of u = (x - a) / a is carried to first order (TwoSum for x - a, fma for the quotient's remainder),
// because a phi reaches 700 and every ulp of u there is an ulp of a times u in the exponent.
XC_SI_HD double igam_prefactor(double a, double x) {
  if (a < 10.0) return exp(a * log(x) - x) / gamma_lanczos(a);
  if (x < 0.1 * a) {
    // far below the mode (u = (x - a) / a < -0.9, and u rounds to -1 once x < a 2^-53): the plain logarithmic
    // form, log Gamma(a) by Stirling
    const double lg = (a - 0.5) * log(a) - a + 0.9189385332046728 + log_gamma_star(a);
    return exp(a * log(x) - x - lg);
  }
  const double d = x - a;
  const double bb = d - x;
  const double d_lo = (x - (d - bb)) + (-a - bb);   // TwoSum: x - a = d + d_lo exactly
  const double u = d / a;
  const double r = fma(-u, a, d) + d_lo;            // a * (true u - u)
  const double e = a * u_minus_log1p(u) + r * (u / (1.0 + u));
  return exp(-e - log_gamma_star(a)) * sqrt(a / (2.0 * kPi));
}

// Regularized lower incomplete gamma P(a, x), a > 0: the power series below x = a + 1, else 1 - Q with Q from
// the Legendre continued fraction (modified Lentz).  NaN for a <= 0 or NaN arguments.
XC_SI_HDN double gammainc(double a, double x) {
  if (!(a > 0.0) || x != x) return NAN;
  if (x <= 0.0) return 0.0;
  if (isinf(x)) return 1.0;
  if (isinf(a)) return NAN;
  const double f = igam_prefactor(a, x);
  if (x < a + 1.0) {
    double term = 1.0, sum = 1.0;
    for (int n = 1; n < kMaxIter; ++n) {
      term *= x / (a + (double)n);
      sum += term;
      if (term < sum * 1e-17) break;
    }
    return f / a * sum;
  }
  if (f == 0.0) return 1.0;
  const double tiny = 1e-300;
  double b = x + 1.0 - a, c = 1.0 / tiny, dd = 1.0 / b, h = dd;
  for (int n = 1; n < kMaxIter; ++n) {
    const double an = -(double)n * ((double)n - a);
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
  return 1.0 - f * h;
}

// ---- digamma / trigamma (x > 0 by recurrence up to 10, then the asymptotic series; reflection below 0) -----
XC_SI_HDN double digamma(double x) {
  if (x != x || x == -INFINITY) return NAN;
  if (x == INFINITY) return INFINITY;
  double acc = 0.0;
  if (x <= 0.0) {
    if (x == floor(x)) return NAN;
    // psi(1 - x) - psi(x) = pi cot(pi x)
    const double r = x - floor(x);
    acc = -kPi / tan(kPi * r);
    x = 1.0 - x;
  }
  while (x < 10.0) {
    acc -= 1.0 / x;
    x += 1.0;
  }
  const double r2 = 1.0 / (x * x);
  double s = -1.0 / 12.0;                    // -B_2k / (2k x^2k), k = 7 down to 1
  s = s * r2 + 691.0 / 32760.0;
  s = s * r2 - 1.0 / 132.0;
  s = s * r2 + 1.0 / 240.0;
  s = s * r2 - 1.0 / 252.0;
  s = s * r2 + 1.0 / 120.0;
  s = s * r2 - 1.0 / 12.0;
  s = s * r2;
  return acc + (log(x) - 0.5 / x + s);
}

XC_SI_HD double trigamma(double x) {         // x > 0
  double acc = 0.0;
  while (x < 10.0) {
    acc += 1.0 / (x * x);
    x += 1.0;
  }
  const double r = 1.0 / x, r2 = r * r;
  double s = 5.0 / 66.0;                     // B_2k / x^(2k+1), k = 1..5
  s = s * r2 - 1.0 / 30.0;
  s = s * r2 + 1.0 / 42.0;
  s = s * r2 - 1.0 / 30.0;
  s = s * r2 + 1.0 / 6.0;
  return acc + r + 0.5 * r2 + s * r2 * r;
}

// ---- the fit -------------------------------------------------------------------------------------------
enum : int { kGamma = XC_SI_GAMMA, kFisk = XC_SI_FISK, kLognorm = XC_SI_LOGNORM };
enum : int { kApp = XC_SI_APP, kMl = XC_SI_ML };

// Root of log(a) - psi(a) = s on scipy's bracket [xa, xb] (gamma_gen.fit; brentq with xtol 2e-12,
// rtol 4 eps): Newton steps kept inside a shrinking bracket (bisection where a step leaves it), converged to a
// few ulp of the true root.  The decreasing function gives the bracket's orientation.  Status bits as
// brentq raises: a NaN end value, or ends of one sign.
XC_SI_HD double gamma_ml_shape(double s, double xa, double xb, int* status) {
  auto f = [&](double a) { return (log(a) - digamma(a)) - s; };
  const double fa = f(xa), fb = f(xb);
  if (fa != fa || fb != fb) { *status |= XC_SI_STATUS_ROOT_NAN; return NAN; }
  if (fa == 0.0) return xa;
  if (fb == 0.0) return xb;
  if ((fa > 0.0) == (fb > 0.0)) { *status |= XC_SI_STATUS_ROOT_SIGN; return NAN; }
  double lo = fa > 0.0 ? xa : xb, hi = fa > 0.0 ? xb : xa;     // f(lo) > 0 > f(hi)
  double a = 0.5 * (xa + xb);
  for (int it = 0; it < 100; ++it) {
    const double fv = f(a);
    if (fv == 0.0) return a;
    if (fv > 0.0) lo = a; else hi = a;
    const double d = 1.0 / a - trigamma(a);
    double an = a - fv / d;
    if (!(an > fmin(lo, hi) && an < fmax(lo, hi))) an = 0.5 * (lo + hi);
    if (fabs(an - a) <= 4e-16 * fabs(an)) return an;
    if (fabs(hi - lo) <= 4e-16 * fabs(an)) return an;
    a = an;
  }
  return a;
}

struct Fit {
  double p[3];
};

XC_SI_HD Fit nan_fit() { return Fit{{NAN, NAN, NAN}}; }

// One (cell, group) sample.  n_all: finite values (zeros left out when zero-inflated) -- <= 1 gives NaN
// (stats.py:49-51).  at(k), k < n_pos: the float32 values x - floc that are > 0, in time order.  any_le: some
// finite value is <= floc (ML: scipy raises FitDataError; the caller has set the status).
template <class At>
XC_SI_HD Fit fit_sample(At at, int n_all, int n_pos, int dist, int method, double floc, int* status) {
  if (n_all <= 1) return nan_fit();
  Fit out;
  out.p[1] = floc;
  if (dist == kGamma && method == kApp) {                        // stats.py:640-651
    const float m = np::mean_f32(at, n_pos);
    const float lm = log_f32(m);
    const float ml = np::mean_f32([&](int k) { return log_f32(at(k)); }, n_pos);
    const float A = lm - ml;
    const float a0 = (1.0f + sqrtf(1.0f + 4.0f * A / 3.0f)) / (4.0f * A);
    out.p[0] = a0;
    out.p[2] = m / a0;
  } else if (dist == kFisk) {                                    // stats.py:653-671
    const float m = np::mean_f32(at, n_pos);
    const float m2 = np::mean_f32([&](int k) { const float v = at(k); return v * v; }, n_pos);
    const float mm = m * m;
    const float m3 = (float)((double)m * (double)m * (double)m);
    out.p[2] = (2.0f * m3) / (m2 + mm);
    out.p[0] = ((double)((float)kPi * m) / 1.7320508075688772) / (double)sqrtf(m2 - mm);
  } else if (dist == kLognorm && method == kApp) {               // stats.py:673-682
    const float mu = np::mean_f32([&](int k) { return log_f32(at(k)); }, n_pos);
    const float var = np::mean_f32([&](int k) { const float d = log_f32(at(k)) - mu; return d * d; }, n_pos);
    out.p[0] = sqrtf(var);
    out.p[2] = exp_f32(mu);
  } else if (dist == kGamma) {                                   // scipy gamma_gen.fit, floc fixed
    if (*status & XC_SI_STATUS_FITDATA) return nan_fit();
    const float xbar = np::mean_f32(at, n_pos);
    const float s = log_f32(xbar) - np::mean_f32([&](int k) { return log_f32(at(k)); }, n_pos);
    const float sm3 = s - 3.0f;
    const float aest = ((3.0f - s) + sqrtf(sm3 * sm3 + 24.0f * s)) / (12.0f * s);
    const float xa = aest * 0.6f, xb = aest * 1.4f;
    const double a = gamma_ml_shape((double)s, (double)xa, (double)xb, status);
    out.p[0] = a;
    out.p[2] = xbar / (float)a;                                  // float32 / Python float stays float32
  } else {                                                       // scipy lognorm_gen.fit, floc fixed
    if (*status & XC_SI_STATUS_FITDATA) return nan_fit();
    const float mu = np::mean_f32([&](int k) { return log_f32(at(k)); }, n_pos);
    const float scale = exp_f32(mu);
    const float ls = log_f32(scale);
    const float var = np::mean_f32([&](int k) { const float d = log_f32(at(k)) - ls; return d * d; }, n_pos);
    const float shape = sqrtf(var);
    if (!(shape > 0.0f && scale > 0.0f)) {                       // scipy falls back to the generic optimiser
      *status |= XC_SI_STATUS_LOGNORM_FALLBACK;
      return nan_fit();
    }
    out.p[0] = shape;
    out.p[2] = scale;
  }
  if (out.p[0] != out.p[0] || out.p[1] != out.p[1] || out.p[2] != out.p[2]) return nan_fit();  // :108-110
  return out;
}

// Every group of cell c (the body of si_fit_kernel, also run by the host build): the group's calibration rows
// are read in time order, zeros and non-NaN values counted, and the values entering the fit, minus floc,
// packed into the cell's workspace column col[k * C] (coalesced across a warp's cells).  Returns the OR of
// the samples' status bits.
XC_SI_HD int fit_cell(const float* x, int64_t C, int64_t ldx, int64_t c, const int32_t* goff, const int32_t* steps,
                      int32_t G, int32_t dist, int32_t method, int32_t zi, double floc, double* params,
                      int32_t* n_zeros, int32_t* n_notnull, float* col) {
  const float floc_f = (float)floc;     // numpy compares / subtracts the Python float in float32 (NEP 50)
  int st_all = 0;
  for (int g = 0; g < G; ++g) {
    const int k0 = goff[g], k1 = goff[g + 1];
    int n_all = 0, n_pos = 0, zeros = 0, notnull = 0;
    bool le = false;
    for (int k = k0; k < k1; ++k) {
      const float v = x[(int64_t)steps[k] * ldx + c];
      if (v != v) continue;
      ++notnull;
      if (v == 0.0f) ++zeros;
      if (isinf(v) || (zi && v == 0.0f)) continue;      // masked_invalid drops +-inf; zeros are NaN when zi
      ++n_all;
      le = le || (v <= floc_f);
      const float xp = v - floc_f;
      if (xp > 0.0f) col[(int64_t)(n_pos++) * C] = xp;
    }
    int st = (method == kMl && le && n_all > 1) ? XC_SI_STATUS_FITDATA : 0;
    const Fit f = fit_sample([&](int k) { return col[(int64_t)k * C]; }, n_all, n_pos, dist, method, floc, &st);
    st_all |= st;
    double* p = params + (int64_t)g * 3 * C + c;
    p[0] = f.p[0];
    p[C] = f.p[1];
    p[2 * C] = f.p[2];
    if (n_zeros) n_zeros[(int64_t)g * C + c] = zeros;
    if (n_notnull) n_notnull[(int64_t)g * C + c] = notnull;
  }
  return st_all;
}

// ---- the transform -------------------------------------------------------------------------------------
// rv_continuous.cdf(x, shape, loc, scale): NaN for invalid parameters or x, 0 at or below the support,
// 1 at +inf.
XC_SI_HD double cdf(int dist, double x, double shape, double loc, double scale) {
  const double y = (x - loc) / scale;
  if (!(shape > 0.0) || !(scale > 0.0) || y != y) return NAN;
  if (y <= 0.0) return 0.0;
  if (isinf(y)) return 1.0;
  if (dist == kGamma) return gammainc(shape, y);
  if (dist == kFisk) return 1.0 / (1.0 + pow(y, -shape));
  return ndtr(log(y) / shape);
}

// norm.ppf(prob) clipped to +-8.21 (stats.py:1177-1191).
XC_SI_HD double prob_to_index(double prob) {
  const double z = ndtri(prob);
  if (z != z) return z;
  return z < -kClip ? -kClip : (z > kClip ? kClip : z);
}

// One element of the standardized index.  zi: the zero-inflated branch of stats.py:1156-1173 with the
// counts of the group and the plotting position (alpha, beta), interpolation factor `interp`.
XC_SI_HD double standardized(int dist, float xv, double shape, double loc, double scale, bool zi, int32_t n_zeros,
                             int32_t n_notnull, double interp, double alpha, double beta) {
  if (!zi) return prob_to_index(cdf(dist, (double)xv, shape, loc, scale));
  const double den = (((double)n_notnull + 1.0) - alpha) - beta;
  const double r1 = (1.0 - alpha) / den;
  const double rn = ((double)n_zeros - alpha) / den;
  double prob;
  if (xv != 0.0f) {
    prob = rn + (1.0 - rn) * cdf(dist, (double)xv, shape, loc, scale);
  } else {
    prob = (1.0 - interp) * r1 + interp * rn;
  }
  return prob_to_index(prob);
}

}  // namespace si
}  // namespace xc
