// Host build of the spatial-analogue device code (xclim_b200/csrc/analog_core.cuh) for the CPU test-suite: the
// per-cell orchestration of analog_cell in analog.cu with its 32 lanes run one after the other and their partials
// added by the same xor butterfly, compiled with g++ -ffp-contract=off.  Samples are float64 here, so float64
// inputs are checked too; the device reads float32 candidates.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../xclim_b200/csrc/analog_core.cuh"

using namespace xc::an;

namespace {

template <class Pool>
double ks_pivot(Pool P, int nA, int nB, int d) {
  std::vector<uint32_t> codes(nA + nB);
  double best[kLanes] = {};
  for (int b = 0; b < nA; ++b) {
    for (int a = 0; a < nA + nB; ++a) codes[a] = ks_code(P, b, a, d);
    for (int l = 0; l < kLanes; ++l) best[l] = fmax(best[l], ks_diff(codes.data(), nA, nB, l, kLanes));
  }
  return *std::max_element(best, best + kLanes);
}

template <int DB>
double cell(const double* x, const double* y, int n, int m, int d, int method, double param, const double* cst,
            int* status) {
  auto X = [&](int i, int k) { return x[i * d + k]; };
  auto Y = [&](int s, int k) { return y[s * d + k]; };
  auto P = [&](int p, int k) { return p < n ? X(p, k) : Y(p - n, k); };
  for (int i = 0; i < n * d; ++i)
    if (isnan(x[i])) return NAN;
  for (int i = 0; i < m * d; ++i)
    if (isnan(y[i])) return NAN;
  std::vector<double> st(5 * d);
  double *mx = st.data(), *sx = mx + d, *my = mx + 2 * d, *sy = mx + 3 * d, *v = mx + 4 * d;
  for (int k = 0; k < d; ++k) {
    col_stats(X, n, k, mx + k, sx + k);
    col_stats(Y, m, k, my + k, sy + k);
    v[k] = method == kNearest ? sqrt(sx[k] * sy[k]) : sx[k] * sy[k];
  }
  if (method == kSeuclidean) {
    bool bad = false;
    const double r = seuclidean(mx, my, cst, d, &bad);
    if (bad) *status |= XC_AN_STATUS_CHKFINITE;
    return r;
  }
  if (method == kMaha) return mahalanobis(mx, my, cst, d);
  if (method == kZech || method == kSzekely) {
    const bool zech = method == kZech;
    double part[3][kLanes], s[3];
    for (int l = 0; l < kLanes; ++l) {
      pair_sums<DB>(P, n, m, d, zech || param != 0.0 ? v : nullptr, zech, param, l, kLanes, s);
      for (int t = 0; t < 3; ++t) part[t][l] = s[t];
    }
    for (int t = 0; t < 3; ++t) s[t] = butterfly_sum(part[t]);
    return zech ? zech_finish(s, n, m) : szekely_finish(s, n, m);
  }
  if (method == kNearest) {
    for (int i = 0; i < (n + m) * d; ++i)
      if (!isfinite(P(i / d, i % d) / v[i % d])) {
        *status |= XC_AN_STATUS_NOT_FINITE;
        return NAN;
      }
    int cnt[kLanes];
    for (int l = 0; l < kLanes; ++l) cnt[l] = nn_count<DB>(P, n, m, d, v, l, kLanes);
    return (double)butterfly_sum(cnt) / (n + m);
  }
  if (method == kKs) {
    auto Q = [&](int p, int k) { return p < m ? Y(p, k) : X(p - m, k); };
    const double pxy = ks_pivot(P, n, m, d), pyx = ks_pivot(Q, m, n, d);
    return pxy >= pyx ? pxy : pyx;
  }
  if (method == kKldiv) {
    if (n < 5 || m < 5) return NAN;
    for (int i = 0; i < (n + m) * d; ++i)
      if (isinf(P(i / d, i % d))) {
        *status |= XC_AN_STATUS_NOT_FINITE;
        return NAN;
      }
    const int k = (int)param;
    double part[kLanes];
    for (int l = 0; l < kLanes; ++l)
      part[l] = k <= 1 ? kl_partial<DB, 2>(P, n, m, d, k, l, kLanes)
                       : kl_partial<DB, XC_AN_KLDIV_MAX_K + 1>(P, n, m, d, k, l, kLanes);
    return kl_finish(butterfly_sum(part), n, m, d);
  }
  return NAN;
}

}  // namespace

extern "C" {

// xc_analog_f32 on host float64 arrays: target (K, n, d), candidates (C, m, d) (one sample per cell), consts
// (K, d) or (K, d, d) or NULL, out (K, C).  Returns the OR-ed XC_AN_STATUS_* bits.
int32_t an_host_analog(const double* target, int32_t n, int32_t K, const double* cand, int32_t m, int64_t C,
                       int32_t d, int32_t method, double param, const double* consts, double* out) {
  int status = 0;
  const int nc = method == kSeuclidean ? d : method == kMaha ? d * d : 0;
  for (int t = 0; t < K; ++t)
    for (int64_t c = 0; c < C; ++c)
      out[t * C + c] = cell<XC_AN_MAX_D>(target + (int64_t)t * n * d, cand + c * m * d, n, m, d, method, param,
                                         consts ? consts + (int64_t)t * nc : nullptr, &status);
  return status;
}

}  // extern "C"
