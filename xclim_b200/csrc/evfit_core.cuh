// Frequency analysis: the per-cell maximum-likelihood fit of the normal, Gumbel and GEV laws and their quantile /
// CDF transforms, shared by the CUDA kernels (evfit.cu) and by a host build of the very same code that the CPU
// test-suite checks against scipy and the oracle (tests/csrc/evfit_host.cpp).
//
// Replaces indices/stats.py `_fitfunc_1d` (:45-112) with `_fit_start` (:576-684) under method "ML" for norm,
// gumbel_r and genextreme -- scipy's `norm_gen.fit`, `gumbel_r_gen.fit` and, for genextreme, the generic
// `rv_continuous.fit` (a Nelder-Mead simplex on the penalised negative log-likelihood) -- and the scipy `ppf` /
// `isf` / `cdf` calls of `parametric_quantile` (:221-289) and `parametric_cdf` (:294-360).
//
// norm follows numpy's float32 arithmetic and matches scipy bit for bit.  gumbel_r solves scipy's own free-loc
// equation to a few ulp (scipy stops brentq at an absolute xtol of 1e-14).  genextreme converges to the optimum
// of the likelihood by damped Newton steps: scipy's simplex stops wherever its tolerances let it, so its
// parameters are not a reproducible target, the likelihood and the return levels are (DESIGN s5).
// Compile WITHOUT floating-point contraction (nvcc -fmad=false, g++ -ffp-contract=off).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/xclim_b200.h"
#include "normal_core.cuh"
#include "npsum.cuh"

#if defined(__CUDACC__)
#define XC_EV_HD __host__ __device__ __forceinline__
#else
#define XC_EV_HD inline
#endif

namespace xc {
namespace ev {

enum : int { kNorm = XC_EV_NORM, kGumbel = XC_EV_GUMBEL_R, kGev = XC_EV_GENEXTREME };
enum : int { kPpf = XC_EV_PPF, kIsf = XC_EV_ISF, kCdf = XC_EV_CDF };

constexpr int kGevMaxIter = 200;           // Newton iterations
constexpr double kGevTol = 1e-13;          // Newton decrement relative to max(1, |nnlf|), on two steps running
constexpr double kSeriesU = 0.25;          // |c y| below which the c-derivatives use their power series

XC_EV_HD int nparams(int dist) { return dist == kGev ? 3 : 2; }

// ---- norm: scipy norm_gen.fit on float32 data -------------------------------------------------------------
// loc = data.mean(), scale = sqrt(((data - loc)**2).mean()), all float32 (numpy's pairwise sums).
template <class At>
XC_EV_HD void fit_norm(At at, int n, double* p) {
  const float m = np::mean_f32(at, n);
  const float v = np::mean_f32([&](int k) { const float d = at(k) - m; return d * d; }, n);
  p[0] = m;
  p[1] = sqrtf(v);
}

// ---- gumbel_r: scipy gumbel_r_gen.fit, loc and scale free ------------------------------------------------
// The scale is the root of f(s) = mean(x) - wavg(x; log-weights -x/s) - s, evaluated in float64 as scipy does on
// float64 data (on float32 data scipy evaluates it in float32, and its root carries float32 noise).
// f is decreasing: f'(s) = -var_w(x) / s^2 - 1.
struct GumbelEval {
  double f, df;
};

template <class At>
XC_EV_HD GumbelEval gumbel_eq(At at, int n, double mean, float xmin, double s) {
  // the log-weights as scipy forms them, -x/s minus their maximum -xmin/s (NaN at a tiny s on a constant
  // sample, as scipy's -inf - -inf)
  const double lmax = -(double)xmin / s;
  double sw = 0.0, swx = 0.0;
  for (int k = 0; k < n; ++k) {
    const double x = at(k);
    const double w = exp(-x / s - lmax);
    sw += w;
    swx += w * x;
  }
  const double wavg = swx / sw;
  double swd = 0.0;
  for (int k = 0; k < n; ++k) {
    const double x = at(k);
    const double w = exp(-x / s - lmax);
    const double d = x - wavg;
    swd += w * d * d;
  }
  GumbelEval e;
  e.f = ((mean - wavg) - s);
  e.df = -(swd / sw) / (s * s) - 1.0;
  return e;
}

XC_EV_HD int sign_of(double v) { return v > 0.0 ? 1 : (v < 0.0 ? -1 : (v == 0.0 ? 0 : 2)); }   // 2: NaN

template <class At>
XC_EV_HD void fit_gumbel(At at, int n, double* p, int* status) {
  double mean = 0.0;
  float xmin = at(0);
  for (int k = 0; k < n; ++k) {
    mean += (double)at(k);
    xmin = fminf(xmin, at(k));
  }
  mean /= (double)n;
  // scipy's bracket: [1/2, 2] (no scale guess from _fit_start), widened by halving / doubling until the signs
  // at the ends differ (a NaN end counts as different) or it spans [0, inf]
  double lb = 0.5, rb = 2.0;
  double flb = gumbel_eq(at, n, mean, xmin, lb).f, frb = gumbel_eq(at, n, mean, xmin, rb).f;
  while (sign_of(flb) == sign_of(frb) && (lb > 0.0 || rb < INFINITY)) {
    lb *= 0.5;
    rb *= 2.0;
    flb = gumbel_eq(at, n, mean, xmin, lb).f;
    frb = gumbel_eq(at, n, mean, xmin, rb).f;
  }
  p[0] = p[1] = NAN;
  if (flb != flb || frb != frb) { *status |= XC_EV_STATUS_ROOT_NAN; return; }
  double s;
  if (flb == 0.0) {
    s = lb;
  } else if (frb == 0.0) {
    s = rb;
  } else if ((flb > 0.0) == (frb > 0.0)) {
    *status |= XC_EV_STATUS_ROOT_SIGN;
    return;
  } else {
    // Newton steps kept inside the shrinking bracket, f(lo) > 0 > f(hi); where a step leaves it, bisection --
    // geometric while the bracket spans more than a factor 4 (the walk above can leave it 60 decades wide)
    double lo = flb > 0.0 ? lb : rb, hi = flb > 0.0 ? rb : lb;
    auto bisect = [&]() {
      const double a = fmin(lo, hi), b = fmax(lo, hi);
      return b > 4.0 * a ? sqrt(a) * sqrt(b) : 0.5 * (a + b);
    };
    s = bisect();
    bool done = false;
    for (int it = 0; it < 400 && !done; ++it) {
      const GumbelEval e = gumbel_eq(at, n, mean, xmin, s);
      if (e.f == 0.0) { done = true; break; }
      if (e.f > 0.0) lo = s; else hi = s;
      double sn = s - e.f / e.df;
      if (!(sn > fmin(lo, hi) && sn < fmax(lo, hi))) sn = bisect();
      done = fabs(sn - s) <= 4e-16 * fabs(sn) || fabs(hi - lo) <= 4e-16 * fabs(sn);
      s = sn;
    }
    if (!done) { *status |= XC_EV_STATUS_NOT_CONVERGED; return; }
  }
  // loc = -s (logsumexp(-x / s) - log n)
  const double lmax = -(double)xmin / s;
  double sw = 0.0;
  for (int k = 0; k < n; ++k) sw += exp(-(double)at(k) / s - lmax);
  const double loc = -s * ((lmax + log(sw)) - log((double)n));
  if (loc != loc || s != s) return;
  p[0] = loc;
  p[1] = s;
}

// ---- genextreme: maximum likelihood in (c, loc, log scale), scipy's sign of c ------------------------------
// With y = (x - loc) / scale, t = 1 - c y > 0, L = log t and a = -L / c (a = y at c = 0), one value's
// negative log-likelihood is  g(c, y) = exp(-a) + a + L,  and nnlf = n log(scale) + sum g.
struct GevPoint {
  double a, L, ac, acc;      // a, log t, da/dc, d2a/dc2
};

XC_EV_HD GevPoint gev_point(double c, double y) {
  GevPoint q;
  const double u = c * y;
  q.L = log1p(-u);
  q.a = c == 0.0 ? y : -q.L / c;
  if (fabs(u) < kSeriesU) {
    // a = sum_k c^(k-1) y^k / k, so da/dc = sum_{k>=2} (k-1) u^(k-2) y^2 / k and
    // d2a/dc2 = sum_{k>=3} (k-1)(k-2) u^(k-3) y^3 / k: no cancellation as c -> 0
    double s1 = 0.5, s2 = 0.0, pw = 1.0;          // the k = 2 term of s1; pw = u^(k-3) at the top of the loop
    for (int k = 3; k < 80; ++k) {
      s2 += (double)(k - 1) * (double)(k - 2) / (double)k * pw;
      pw *= u;
      s1 += (double)(k - 1) / (double)k * pw;
      if (fabs(pw) < 1e-18) break;
    }
    q.ac = s1 * y * y;
    q.acc = s2 * y * y * y;
  } else {
    const double t = 1.0 - u;
    q.ac = q.L / (c * c) + y / (c * t);
    q.acc = -2.0 * q.L / (c * c * c) - 2.0 * y / (c * c * t) + y * y / (c * t * t);
  }
  return q;
}

// nnlf at theta = (c, loc, log scale); +inf when a value lies outside the open support
template <class At>
XC_EV_HD double gev_nnlf(At at, int n, const double* th) {
  const double c = th[0], mu = th[1], is = exp(-th[2]);
  double s = 0.0;
  for (int k = 0; k < n; ++k) {
    const double y = ((double)at(k) - mu) * is;
    const double u = c * y;
    if (!(u < 1.0)) return INFINITY;
    const double L = log1p(-u);
    const double a = c == 0.0 ? y : -L / c;
    s += (exp(-a) + a) + L;
  }
  const double r = (double)n * th[2] + s;
  return r == r ? r : INFINITY;
}

// gradient and Hessian of nnlf in theta
template <class At>
XC_EV_HD void gev_derivs(At at, int n, const double* th, double* g, double* H) {
  const double c = th[0], mu = th[1], is = exp(-th[2]);
  double gc = 0, gm = 0, gp = 0, hcc = 0, hcm = 0, hcp = 0, hmm = 0, hmp = 0, hpp = 0;
  for (int k = 0; k < n; ++k) {
    const double y = ((double)at(k) - mu) * is;
    const GevPoint q = gev_point(c, y);
    const double t = 1.0 - c * y;
    const double E = exp(-q.a), omE = 1.0 - E;
    const double ay = 1.0 / t, ayy = c / (t * t), acy = y / (t * t);
    const double Ly = -c / t, Lc = -y / t, Lyy = -(c * c) / (t * t), Lcy = -1.0 / (t * t), Lcc = -(y * y) / (t * t);
    const double g_y = ay * omE + Ly;
    const double g_c = q.ac * omE + Lc;
    const double g_yy = ayy * omE + ay * ay * E + Lyy;
    const double g_cy = acy * omE + q.ac * ay * E + Lcy;
    const double g_cc = q.acc * omE + q.ac * q.ac * E + Lcc;
    gc += g_c;
    gm += g_y;                    // times -1/scale below
    gp += g_y * y;                // d/dphi = n - sum y g_y
    hcc += g_cc;
    hcm += g_cy;                  // times -1/scale
    hcp += g_cy * y;              // times -1
    hmm += g_yy;                  // times 1/scale^2
    hmp += g_yy * y + g_y;        // times 1/scale
    hpp += g_yy * y * y + g_y * y;
  }
  g[0] = gc;
  g[1] = -gm * is;
  g[2] = (double)n - gp;
  H[0] = hcc;
  H[1] = H[3] = -hcm * is;
  H[2] = H[6] = -hcp;
  H[4] = hmm * is * is;
  H[5] = H[7] = hmp * is;
  H[8] = hpp;
}

// Solve H d = -g by Cholesky; false when H is not positive definite.
XC_EV_HD bool newton_dir(const double* H, const double* g, double* d) {
  const double l00s = H[0];
  if (!(l00s > 0.0)) return false;
  const double l00 = sqrt(l00s);
  const double l10 = H[3] / l00, l20 = H[6] / l00;
  const double l11s = H[4] - l10 * l10;
  if (!(l11s > 0.0)) return false;
  const double l11 = sqrt(l11s);
  const double l21 = (H[7] - l20 * l10) / l11;
  const double l22s = H[8] - l20 * l20 - l21 * l21;
  if (!(l22s > 0.0)) return false;
  const double l22 = sqrt(l22s);
  const double z0 = -g[0] / l00;
  const double z1 = (-g[1] - l10 * z0) / l11;
  const double z2 = (-g[2] - l20 * z0 - l21 * z1) / l22;
  d[2] = z2 / l22;
  d[1] = (z1 - l21 * d[2]) / l11;
  d[0] = (z0 - l10 * d[1] - l20 * d[2]) / l00;
  return true;
}

template <class At>
XC_EV_HD void fit_gev(At at, int n, double* p, int* status) {
  p[0] = p[1] = p[2] = NAN;
  // xclim's start (stats.py:608-610): m, v = x.mean(), x.var() (float32), s = sqrt(6 v) / pi,
  // loc = m - 0.57722 s, c = 0.1
  const float m = np::mean_f32(at, n);
  const float v = np::mean_f32([&](int k) { const float d = at(k) - m; return d * d; }, n);
  const float s0 = sqrtf(6.0f * v) / (float)3.14159265358979323846;
  double loc0 = m - 0.57722f * s0, sc0 = s0;
  if (!(s0 > 0.0f) || isinf(s0) || loc0 != loc0 || isinf(loc0)) {
    // the float32 variance under- or overflows (values near 1e-30 or 1e30): the same start in float64
    double m64 = 0.0, v64 = 0.0;
    for (int k = 0; k < n; ++k) m64 += (double)at(k);
    m64 /= (double)n;
    for (int k = 0; k < n; ++k) { const double d = (double)at(k) - m64; v64 += d * d; }
    sc0 = sqrt(6.0 * (v64 / (double)n)) / 3.14159265358979323846;
    loc0 = m64 - 0.57722 * sc0;
    if (!(sc0 > 0.0) || isinf(sc0)) { *status |= XC_EV_STATUS_NOT_CONVERGED; return; }
  }
  double th[3] = {0.1, loc0, log(sc0)};
  double f = gev_nnlf(at, n, th);
  if (isinf(f)) {                  // a value beyond 1/c: start from the Gumbel law, whose support is the line
    th[0] = 0.0;
    f = gev_nnlf(at, n, th);
    if (isinf(f)) { *status |= XC_EV_STATUS_NOT_CONVERGED; return; }
  }
  int small = 0;
  bool converged = false;
  for (int it = 0; it < kGevMaxIter && !converged; ++it) {
    double g[3], H[9], d[3];
    gev_derivs(at, n, th, g, H);
    bool newton = newton_dir(H, g, d);
    if (!newton) {                 // not positive definite: a diagonally scaled gradient step
      for (int j = 0; j < 3; ++j) d[j] = -g[j] / fmax(fabs(H[4 * j]), 1e-300);
    }
    const double slope = g[0] * d[0] + g[1] * d[1] + g[2] * d[2];     // -(Newton decrement)^2
    if (!(slope == slope)) break;
    const double tol = kGevTol * fmax(1.0, fabs(f));
    small = (newton && -slope <= tol) ? small + 1 : 0;
    // backtracking (Armijo); once the decrement is at the rounding level, a full step that does not raise the
    // nnlf beyond that level is taken
    double alpha = 1.0, ft = INFINITY, tt[3];
    bool ok = false;
    for (int ls = 0; ls < 60; ++ls) {
      for (int j = 0; j < 3; ++j) tt[j] = th[j] + alpha * d[j];
      // c < 1: beyond, the likelihood has no maximum; a local optimum inside is what scipy's simplex finds
      ft = tt[0] < 1.0 ? gev_nnlf(at, n, tt) : INFINITY;
      if (ft <= f + 1e-4 * alpha * slope || (small && ft <= f + tol)) { ok = true; break; }
      alpha *= 0.5;
    }
    if (!ok) break;
    th[0] = tt[0]; th[1] = tt[1]; th[2] = tt[2];
    f = ft;
    if (small >= 2) converged = true;
  }
  if (!converged) {                // iterates running into c -> 1 have no interior optimum to reach
    *status |= th[0] > 0.999 ? XC_EV_STATUS_UNBOUNDED : XC_EV_STATUS_NOT_CONVERGED;
    return;
  }
  const double sc = exp(th[2]);
  if (th[0] != th[0] || th[1] != th[1] || !(sc > 0.0) || isinf(sc)) { *status |= XC_EV_STATUS_NOT_CONVERGED; return; }
  p[0] = th[0];
  p[1] = th[1];
  p[2] = sc;
}

// The fit of one cell: the finite values of x[t * ldx + c], t < T, compacted in time order into the cell's
// workspace column col[k * C] (coalesced across a warp's cells), then fitted; params[j * C + c] in scipy order.
// NaN when <= 1 finite value is left or a parameter is NaN (stats.py:49-51, :108-110), and for gumbel_r /
// genextreme when every value is the same (no maximum of the likelihood).  Returns status bits.
XC_EV_HD int fit_cell(const float* x, int64_t T, int64_t C, int64_t ldx, int64_t c, int dist, double* params,
                      float* col) {
  int n = 0;
  float lo = INFINITY, hi = -INFINITY;
  for (int64_t t = 0; t < T; ++t) {
    const float v = x[t * ldx + c];
    if (v == v && !isinf(v)) {
      col[(int64_t)(n++) * C] = v;
      lo = fminf(lo, v);
      hi = fmaxf(hi, v);
    }
  }
  double p[3] = {NAN, NAN, NAN};
  int st = 0;
  if (n > 1 && dist != kNorm && lo == hi) {
    st = XC_EV_STATUS_UNBOUNDED;      // one value repeated: the likelihood grows without bound as scale -> 0
  } else if (n > 1) {
    auto at = [&](int k) { return col[(int64_t)k * C]; };
    if (dist == kNorm) fit_norm(at, n, p);
    else if (dist == kGumbel) fit_gumbel(at, n, p, &st);
    else fit_gev(at, n, p, &st);
  }
  const int np_ = nparams(dist);
  bool any_nan = false;
  for (int j = 0; j < np_; ++j) any_nan = any_nan || p[j] != p[j];
  for (int j = 0; j < np_; ++j) params[(int64_t)j * C + c] = any_nan ? NAN : p[j];
  return st;
}

// ---- the transforms ------------------------------------------------------------------------------------
// The standardised quantile functions of scipy's _ppf / _isf and the CDF of the standardised variable.
XC_EV_HD double std_ppf(int dist, double q, double c) {
  if (dist == kNorm) return si::ndtri(q);
  const double x = -log(-log(q));
  if (dist == kGumbel || c == 0.0 || x != x) return x;
  return -expm1(-c * x) / c;
}

XC_EV_HD double std_isf(int dist, double q, double c) {
  if (dist == kNorm) return -si::ndtri(q);
  const double x = -log(-log1p(-q));
  if (dist == kGumbel || c == 0.0 || x != x) return x;
  return -expm1(-c * x) / c;
}

XC_EV_HD double std_cdf(int dist, double y, double c) {
  if (dist == kNorm) return si::ndtr(y);
  if (dist == kGumbel) return exp(-exp(-y));
  const double llc = (c != 0.0) ? log1p(-c * y) / c : -y;
  return exp(-exp(llc));
}

// One element of ppf / isf (q a probability) or cdf (q a value) under params (shape,) loc, scale, with
// rv_continuous's argument checks and support edges: NaN for a non-finite shape, scale <= 0, a NaN loc or a
// probability outside [0, 1]; the support's ends at probabilities 0 and 1; cdf 0 / 1 outside the support.
XC_EV_HD double transform(int dist, int kind, double q, double c, double loc, double scale) {
  if (dist != kGev) c = 0.0;
  if (!(scale > 0.0) || isinf(c) || c != c || loc != loc) return NAN;
  // support [lo, hi] of the standardised law (genextreme: 1/c on the bounded side)
  const double lo = (dist == kGev && c < 0.0) ? 1.0 / c : -INFINITY;
  const double hi = (dist == kGev && c > 0.0) ? 1.0 / c : INFINITY;
  if (kind == kCdf) {
    const double y = (q - loc) / scale;
    if (y != y) return NAN;
    if (y >= hi) return 1.0;
    if (y <= lo) return 0.0;
    return std_cdf(dist, y, c);
  }
  if (q != q || q < 0.0 || q > 1.0) return NAN;
  if (kind == kPpf) {
    if (q == 0.0) return lo * scale + loc;
    if (q == 1.0) return hi * scale + loc;
    return std_ppf(dist, q, c) * scale + loc;
  }
  if (q == 1.0) return lo * scale + loc;
  if (q == 0.0) return hi * scale + loc;
  return std_isf(dist, q, c) * scale + loc;
}

}  // namespace ev
}  // namespace xc
