// Spatial analogues: the per-cell dissimilarity metrics between a target sample (n, d) and a candidate sample
// (m, d), shared by the CUDA kernel (analog.cu) and by a host build of the very same code that the CPU test-suite
// checks against the oracle (tests/csrc/analog_host.cpp).
//
// Replaces the metric functions of analog.py (:181-628) behind `_metric_overhead` (:154-170).  The pooled
// sample is read through an accessor P(p, k) -> double: points p < n are the target's, the others the
// candidate's.  The pair loops are split over L lanes by their first point (p = lane, lane + L, ...); each lane
// returns its partial sums and the caller adds the L partials by the xor butterfly of `butterfly_sum` (a warp
// shuffle on the device, the same additions in the same order on the host), so both builds agree bit for bit.
// Everything is float64 from the float32 (or float64) samples; the reference takes mean and std in the input
// dtype (DESIGN.md section 4).  Compile WITHOUT floating-point contraction (nvcc -fmad=false,
// g++ -ffp-contract=off) so that both builds round the same way.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/xclim_b200.h"

#if defined(__CUDACC__)
#define XC_AN_HD __host__ __device__ __forceinline__
#else
#define XC_AN_HD inline
#endif

namespace xc {
namespace an {

enum : int {
  kSeuclidean = XC_AN_SEUCLIDEAN, kNearest = XC_AN_NEAREST_NEIGHBOR, kZech = XC_AN_ZECH_ASLAN,
  kSzekely = XC_AN_SZEKELY_RIZZO, kKs = XC_AN_KOLMOGOROV_SMIRNOV, kKldiv = XC_AN_KLDIV, kMaha = XC_AN_MAHALANOBIS
};
constexpr int kLanes = 32;

// mean and std(ddof=1) of column k of an (cnt, d) sample, summed in sample order
template <class At>
XC_AN_HD void col_stats(At at, int cnt, int k, double* mean, double* sd) {
  double s = 0.0;
  for (int i = 0; i < cnt; ++i) s += at(i, k);
  const double mu = s / cnt;
  double q = 0.0;
  for (int i = 0; i < cnt; ++i) {
    const double e = at(i, k) - mu;
    q += e * e;
  }
  *mean = mu;
  *sd = sqrt(q / (cnt - 1));
}

// ---- seuclidean (:210-213): scipy's minkowski(mx, my, 2, w=1/V): sqrt(w) * (mx - my), then its 2-norm.
// scipy.linalg.norm refuses a non-finite vector: *bad is set, the caller raises.
XC_AN_HD double seuclidean(const double* mx, const double* my, const double* V, int d, bool* bad) {
  double s = 0.0;
  for (int k = 0; k < d; ++k) {
    const double t = sqrt(1.0 / V[k]) * (mx[k] - my[k]);
    if (!isfinite(t)) *bad = true;
    s += t * t;
  }
  return sqrt(s);
}

// ---- mahalanobis (:620-628): sqrt((delta @ VI) @ delta), delta = mx - my, IEEE arithmetic throughout
XC_AN_HD double mahalanobis(const double* mx, const double* my, const double* VI, int d) {
  double m = 0.0;
  for (int j = 0; j < d; ++j) {
    double t = 0.0;
    for (int i = 0; i < d; ++i) t += (mx[i] - my[i]) * VI[i * d + j];
    m += t * (mx[j] - my[j]);
  }
  return sqrt(m);
}

// load pooled point p into registers (DB >= d: a compile-time bound keeps the array in registers)
template <int DB, class Pool>
XC_AN_HD void load_point(Pool P, int p, int d, double* z) {
#pragma unroll
  for (int k = 0; k < DB; ++k)
    if (k < d) z[k] = P(p, k);
}

// squared distance between z and pooled point q, divided per indicator by v (standardized) or not (v == nullptr)
template <int DB, class Pool>
XC_AN_HD double dist2(Pool P, const double* z, int q, int d, const double* v) {
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < DB; ++k)
    if (k < d) {
      const double e = z[k] - P(q, k);
      s += v ? e * e / v[k] : e * e;
    }
  return s;
}

// ---- zech_aslan (:307-319) and szekely_rizzo (:370-385): the lane's partial sums over pairs (i < j within x:
// sum[0], within y: sum[1], x with y: sum[2]) of -log(clip(dist, dmin)) (zech) or dist (szekely).  v: the
// per-indicator products std_x * std_y (seuclidean distances), or nullptr (plain Euclidean).
template <int DB, class Pool>
XC_AN_HD void pair_sums(Pool P, int n, int m, int d, const double* v, bool zech, double dmin, int lane, int L,
                        double* sum) {
  double sxx = 0.0, syy = 0.0, sxy = 0.0;
  double z[DB];
  for (int i = lane; i < n + m; i += L) {
    load_point<DB>(P, i, d, z);
    for (int j = i + 1; j < n + m; ++j) {
      double r = sqrt(dist2<DB>(P, z, j, d, v));
      if (zech) r = -log(r < dmin ? dmin : r);     // ndarray.clip keeps NaN
      if (i >= n)
        syy += r;
      else if (j < n)
        sxx += r;
      else
        sxy += r;
    }
  }
  sum[0] = sxx;
  sum[1] = syy;
  sum[2] = sxy;
}

XC_AN_HD double zech_finish(const double* s, int n, int m) {
  const double phix = s[0] / (double)((int64_t)n * (n - 1));
  const double phiy = s[1] / (double)((int64_t)m * (m - 1));
  const double phixy = s[2] / (double)((int64_t)n * m);
  return phix + phiy - phixy;
}

XC_AN_HD double szekely_finish(const double* s, int n, int m) {
  const double sXY = s[2] / (double)((int64_t)n * m);
  const double sXX = s[0] * 2 / (double)((int64_t)n * n);
  const double sYY = s[1] * 2 / (double)((int64_t)m * m);
  const double w = (double)((int64_t)n * m) / (double)(n + m);
  return w * (sXY + sXY - sXX - sYY);
}

// ---- nearest_neighbor (:239-251) with the stated tie rule: the neighbour of p is the nearest other pooled
// point, ties to the lowest pooled index.  Points are standardized by s (sqrt(std_x * std_y)) on the fly.
// Returns the lane's count of points whose neighbour is from their own sample.
template <int DB, class Pool>
XC_AN_HD int nn_count(Pool P, int n, int m, int d, const double* s, int lane, int L) {
  auto Z = [&](int p, int k) { return P(p, k) / s[k]; };
  int same = 0;
  double z[DB];
  for (int p = lane; p < n + m; p += L) {
    load_point<DB>(Z, p, d, z);
    double best = INFINITY;
    int q_best = p == 0 ? 1 : 0;
    for (int q = 0; q < n + m; ++q) {
      if (q == p) continue;
      const double e = dist2<DB>(Z, z, q, d, nullptr);
      if (e < best) {
        best = e;
        q_best = q;
      }
    }
    same += (p < n) == (q_best < n);
  }
  return same;
}

// ---- kolmogorov_smirnov (:457-495): pivot b of sample A gives pooled point a the quadrant code
// sum_k 2^k [A_b,k <= a_k]; the pivot's statistic is the largest |count_A(code) / nA - count_B(code) / nB|
// over the codes present.  Comparisons and exact divisions only: order-free and bit for bit.
template <class Pool>
XC_AN_HD uint32_t ks_code(Pool P, int b, int a, int d) {
  uint32_t c = 0;
  for (int k = 0; k < d; ++k) c |= (uint32_t)(P(b, k) <= P(a, k)) << k;
  return c;
}

// the lane's max over its points a of the pivot difference at a's code; codes[0, nA) are sample A's, the rest B's
XC_AN_HD double ks_diff(const uint32_t* codes, int nA, int nB, int lane, int L) {
  double best = 0.0;
  for (int a = lane; a < nA + nB; a += L) {
    const uint32_t c = codes[a];
    int ca = 0, cb = 0;
    for (int q = 0; q < nA; ++q) ca += codes[q] == c;
    for (int q = nA; q < nA + nB; ++q) cb += codes[q] == c;
    const double diff = fabs(1.0 * ca / nA - 1.0 * cb / nB);
    best = diff > best ? diff : best;
  }
  return best;
}

// insert e into the ascending list b of the KB smallest values seen (unrolled: b stays in registers)
template <int KB>
XC_AN_HD void keep_smallest(double (&b)[KB], double e) {
#pragma unroll
  for (int t = 0; t < KB; ++t)
    if (e < b[t]) {
      const double o = b[t];
      b[t] = e;
      e = o;
    }
}

// ---- kldiv (:551-587): for target point i, r = the (k + 1)-th smallest distance to the target's points
// (itself included), s = the k-th smallest to the candidate's; inf where there are fewer points, as cKDTree
// fills its answer.  The lane's partial sum of -log(r / s).  KB >= k + 1.
template <int DB, int KB, class Pool>
XC_AN_HD double kl_partial(Pool P, int n, int m, int d, int k, int lane, int L) {
  double acc = 0.0;
  double z[DB];
  for (int i = lane; i < n; i += L) {
    load_point<DB>(P, i, d, z);
    double bx[KB], by[KB];
#pragma unroll
    for (int t = 0; t < KB; ++t) bx[t] = by[t] = INFINITY;
    for (int q = 0; q < n + m; ++q) {
      const double e = dist2<DB>(P, z, q, d, nullptr);
      if (q < n)
        keep_smallest<KB>(bx, e);
      else
        keep_smallest<KB>(by, e);
    }
    double r = INFINITY, s = INFINITY;
#pragma unroll
    for (int t = 0; t < KB; ++t) {
      if (t == k) r = bx[t];
      if (t == k - 1) s = by[t];
    }
    acc += -log(sqrt(r) / sqrt(s));
  }
  return acc;
}

XC_AN_HD double kl_finish(double sum, int n, int m, int d) {
  return sum * d / n + log(m / (n - 1.0));
}

// a value per lane -> their sum, added by the xor butterfly (host order of the device's __shfl_xor_sync sum)
template <class T>
inline T butterfly_sum(T* v) {
  for (int off = kLanes / 2; off > 0; off >>= 1) {
    T nv[kLanes];
    for (int l = 0; l < kLanes; ++l) nv[l] = v[l] + v[l ^ off];
    for (int l = 0; l < kLanes; ++l) v[l] = nv[l];
  }
  return v[0];
}

}  // namespace an
}  // namespace xc
