// Ensemble statistics across realizations (xc_ens_percentiles_f32, xc_ens_moments_f32, xc_ens_robustness_f32,
// include/xclim_b200.h e1).
//
// Percentiles and moments see the ensemble as an (R, N) matrix of N independent columns, x[r * ldr + n]: one lane
// per column, so a warp reads one coalesced 128-byte row segment per member.  A column of R <= 32 members is
// sorted in registers by the networks of sortnet.cuh (padded to the power of two >= R with -inf); 33 <= R <= 128
// members are sorted by a per-lane bitonic network in shared memory.  The sorted column is left in shared memory
// (k-th largest at s[k * threads + lane]) and the quantiles of its n non-NaN values are finalised there with the
// index and lerp rules of quantile.cuh, which follow the reference's _nan_quantile bit for bit.  NaN members sort
// below every value as -inf; only the count n says how many of the top entries are values.
//
// Robustness: one lane per cell walks every member's fut and ref series along time (rows coalesced across
// cells), twice per series: the float64 sum, then the float64 sum of squared deviations from the mean.  The
// t-tests and the Student-t distribution are in ensemble_core.cuh, which the CPU tests also build for the host.
// Built with -fmad=false so that both builds round every operation the same way.
#include "common.cuh"
#include "ensemble_core.cuh"
#include "quantile.cuh"
#include "sortnet.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;       // register-sort and moments kernels
constexpr int kThreadsSmem = 64;    // shared-memory sort: 64 lanes x 128 floats = 32 KiB
constexpr int kMaxPer = 32;         // percentiles per launch

struct PercSpecs {
  QuantSpec s[kMaxPer];
  int np;
};

__device__ __forceinline__ float member(const float* x, int64_t ldr, int64_t n, int r) {
  return ld_stream(x + (int64_t)r * ldr + n);
}

// the percentiles of one sorted column: kth(k) is its k-th largest entry, n its count of non-NaN values
// (R members, n of them not NaN).  The clamps interpolate as _get_indexes / _linear_interpolation do: vi >= n - 1
// takes index -1, the last sorted entry (a NaN member when n < R, giving the maximum; else the maximum itself, so
// max - 0 * (1 - g) turns a -0 maximum into +0), vi < 0 takes index 0 twice.
template <class Kth>
__device__ __forceinline__ double column_quantile(Kth kth, int n, int R, const QuantSpec& s) {
  if (n == 0) return __longlong_as_double(0x7ff8000000000000LL);
  const float vmax = kth(0);
  if (n == 1) return (double)vmax;
  QuantIdx qi = quant_index(n, s);
  float left, right;
  if (qi.vi >= (double)n - 1.0) {
    if (n < R) return (double)vmax;
    qi.lo = -1.0;
    left = right = vmax;
  } else if (qi.vi < 0.0) {
    qi.lo = 0.0;
    left = right = kth(n - 1);
  } else {
    left = kth(n - 1 - qi.ilo);
    right = kth(n - 2 - qi.ilo);
  }
  const double r = quant_lerp(left, right, qi);
  return lerp_is_nan(r, n) ? (double)vmax : r;
}

template <typename OutT, int NT>
__device__ __forceinline__ void store_percentiles(const float* col, int n, int R, bool enough, const PercSpecs& P,
                                                  OutT* out, int64_t N, int64_t c) {
  auto kth = [&](int k) { return col[k * NT]; };
  for (int p = 0; p < P.np; ++p) {
    const double q = enough ? column_quantile(kth, n, R, P.s[p]) : __longlong_as_double(0x7ff8000000000000LL);
    out[(int64_t)p * N + c] = (OutT)q;
  }
}

// R <= NR <= 32 members sorted in registers; R == 1 writes float32 (the reference's np.take branch)
template <int NR, typename OutT>
__global__ void __launch_bounds__(kThreads)
ens_perc_reg_kernel(const float* __restrict__ x, int R, int64_t N, int64_t ldr, PercSpecs P, int min_members,
                    OutT* __restrict__ out) {
  __shared__ float s[NR * kThreads];
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= N) return;
  float a[NR];
  int n = 0;
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    const float v = r < R ? member(x, ldr, c, r) : XC_NEG_INF;
    n += (r < R && v == v);
    a[r] = (v == v) ? v : XC_NEG_INF;
  }
  sort_desc<NR>(a);
  float* col = s + threadIdx.x;
#pragma unroll
  for (int k = 0; k < NR; ++k) col[k * kThreads] = a[k];
  store_percentiles<OutT, kThreads>(col, n, R, n >= min_members, P, out, N, c);
}

// 32 < R <= RP members: per-lane bitonic sort (descending) of s[k * kThreadsSmem], k < RP
template <int RP>
__global__ void __launch_bounds__(kThreadsSmem)
ens_perc_smem_kernel(const float* __restrict__ x, int R, int64_t N, int64_t ldr, PercSpecs P, int min_members,
                     double* __restrict__ out) {
  __shared__ float s[RP * kThreadsSmem];
  const int64_t c = (int64_t)blockIdx.x * kThreadsSmem + threadIdx.x;
  if (c >= N) return;
  float* col = s + threadIdx.x;
  int n = 0;
  for (int r = 0; r < RP; ++r) {
    const float v = r < R ? member(x, ldr, c, r) : XC_NEG_INF;
    n += (r < R && v == v);
    col[r * kThreadsSmem] = (v == v) ? v : XC_NEG_INF;
  }
#pragma unroll
  for (int k = 2; k <= RP; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll 8
      for (int i = 0; i < RP; ++i) {
        const int l = i ^ j;
        if (l > i) {
          const float u = col[i * kThreadsSmem], w = col[l * kThreadsSmem];
          const float hi = fmaxf(u, w), lo = fminf(u, w);
          const bool desc = (i & k) == 0;
          col[i * kThreadsSmem] = desc ? hi : lo;
          col[l * kThreadsSmem] = desc ? lo : hi;
        }
      }
    }
  }
  store_percentiles<double, kThreadsSmem>(col, n, R, n >= min_members, P, out, N, c);
}

// count, mean, std (ddof 0), min, max of each column's non-NaN values; unweighted: float64 sums in member order,
// each result rounded once to float32; weighted (w != NULL): xarray's Weighted.mean / .std in float64
__global__ void __launch_bounds__(kThreads)
ens_moments_kernel(const float* __restrict__ x, int R, int64_t N, int64_t ldr, const double* __restrict__ w,
                   int min_members, void* __restrict__ mean_out, void* __restrict__ std_out, float* __restrict__ vmin_out,
                   float* __restrict__ vmax_out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= N) return;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  int n = 0;
  double sw = 0.0, s = 0.0;
  float vmin = __int_as_float(0x7f800000), vmax = XC_NEG_INF;
  for (int r = 0; r < R; ++r) {
    const float v = member(x, ldr, c, r);
    if (v == v) {
      ++n;
      const double wr = w ? __ldg(w + r) : 1.0;
      sw += wr;
      s += w ? (double)v * wr : (double)v;
      vmin = fminf(vmin, v);
      vmax = fmaxf(vmax, v);
    }
  }
  // xarray: the sum of weights over valid members is NaN where it is 0 (no valid member, or zero weights)
  const double m = (n == 0 || sw == 0.0) ? nan : s / sw;
  double ss = 0.0;
  for (int r = 0; r < R; ++r) {
    const float v = member(x, ldr, c, r);
    if (v == v) {
      const double d = (double)v - m;
      ss += w ? d * d * __ldg(w + r) : d * d;
    }
  }
  const double sd = sqrt(ss / sw);
  const bool enough = n >= min_members && n > 0;
  if (w) {
    ((double*)mean_out)[c] = enough ? m : nan;
    ((double*)std_out)[c] = enough ? sd : nan;
  } else {
    ((float*)mean_out)[c] = enough ? (float)m : (float)nan;
    ((float*)std_out)[c] = enough ? (float)sd : (float)nan;
  }
  vmin_out[c] = enough ? vmin : (float)nan;
  vmax_out[c] = enough ? vmax : (float)nan;
}

// NaN-omitting float64 moments of one series p[t * ldt], t < T
struct SeriesStats {
  int n;
  double mean, ss;   // ss = sum of squared deviations from the mean
};
__device__ __forceinline__ SeriesStats series_stats(const float* p, int64_t T, int64_t ldt) {
  SeriesStats st{0, 0.0, 0.0};
  double s = 0.0;
  for (int64_t t = 0; t < T; ++t) {
    const float v = ld_stream(p + t * ldt);
    if (v == v) {
      s += (double)v;
      ++st.n;
    }
  }
  st.mean = st.n ? s / st.n : __longlong_as_double(0x7ff8000000000000LL);
  for (int64_t t = 0; t < T; ++t) {
    const float v = p[t * ldt];
    if (v == v) {
      const double d = (double)v - st.mean;
      st.ss += d * d;
    }
  }
  return st;
}

__global__ void __launch_bounds__(kThreads)
ens_robustness_kernel(const float* __restrict__ fut, int64_t Tf, int64_t ldf_r, int64_t ldf_t,
                      const float* __restrict__ ref, int64_t Tr, int64_t ldr_r, int64_t ldr_t,
                      const float* __restrict__ refy, int64_t P, int64_t ldy_r, const double* __restrict__ yx,
                      int R, int64_t C, const double* __restrict__ w, int test, double param, int strict_sign,
                      double* __restrict__ frac, float* __restrict__ pvals) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  double sv = 0.0, sc = 0.0, sp = 0.0, sn = 0.0, scp = 0.0, scn = 0.0;
  for (int r = 0; r < R; ++r) {
    const SeriesStats f = series_stats(fut + (int64_t)r * ldf_r + c, Tf, ldf_t);
    SeriesStats g{0, 0.0, 0.0};
    if (ref) g = series_stats(ref + (int64_t)r * ldr_r + c, Tr, ldr_t);
    const double delta = ref ? f.mean - g.mean : f.mean;
    const bool valid = f.n == Tf && (!ref || g.n == Tr);
    bool changed = true;
    double p = __longlong_as_double(0x7ff8000000000000LL);
    if (test == XC_ENS_TEST_ABS) changed = fabs(delta) > param;
    else if (test == XC_ENS_TEST_REL) changed = fabs(delta / g.mean) > param;
    else if (test == XC_ENS_TEST_IPCC) {
      const float* y = refy + (int64_t)r * ldy_r + c;
      const double sigma = ens::detrended_std([&](int64_t k) { return (double)y[k * C]; }, yx, P);
      changed = fabs(delta) > ens::ipcc_ar6_c_gamma(sigma);
    }
    else if (test == XC_ENS_TEST_TTEST || test == XC_ENS_TEST_WELCH) {
      p = test == XC_ENS_TEST_TTEST ? ens::ttest_1samp_p(f.n, f.mean, f.ss, g.mean)
                                    : ens::welch_ttest_p(f.n, f.mean, f.ss, g.n, g.mean, g.ss);
      changed = p < param;
      if (pvals) pvals[(int64_t)r * C + c] = (float)p;
    }
    const bool pos = strict_sign ? delta > 0.0 : delta >= 0.0;
    const bool neg = strict_sign ? delta < 0.0 : delta <= 0.0;
    if (valid) {
      const double wr = w ? __ldg(w + r) : 1.0;
      sv += wr;
      sc += changed ? wr : 0.0;
      sp += pos ? wr : 0.0;
      sn += neg ? wr : 0.0;
      scp += (pos && changed) ? wr : 0.0;
      scn += (neg && changed) ? wr : 0.0;
    }
  }
  // ensembles/_robustness.py:257-271, then out.fillna(0) (:319)
  auto fill0 = [](double v) { return v != v ? 0.0 : v; };
  const double pf = sp / sv, nf = sn / sv;
  const double agree = fmax(fmax(pf, nf), 1.0 - pf - nf);
  const double vals[7] = {sc / sv, pf, scp / sv, nf, scn / sv, sv / (double)R, agree};
#pragma unroll
  for (int k = 0; k < 7; ++k) frac[(int64_t)k * C + c] = fill0(vals[k]);
}

}  // namespace
}  // namespace xc

using namespace xc;

static int32_t check_columns(const float* x, int64_t R, int64_t N, int64_t ldr) {
  XC_REQUIRE(x, "null pointer argument");
  XC_REQUIRE(R >= 1 && R <= XC_ENS_MAX_MEMBERS, "the realization dimension must have 1 to %d members, got %lld",
             XC_ENS_MAX_MEMBERS, (long long)R);
  XC_REQUIRE(N > 0 && ldr >= N && N <= 2147483647LL * kThreadsSmem, "bad shape");
  return XC_OK;
}

template <int NR, typename OutT>
static int32_t launch_reg(const float* x, int R, int64_t N, int64_t ldr, const PercSpecs& P, int min_members,
                          void* out, cudaStream_t st) {
  ens_perc_reg_kernel<NR, OutT><<<(unsigned)((N + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      x, R, N, ldr, P, min_members, (OutT*)out);
  return launch_status("ens_perc_reg_kernel");
}

template <int RP>
static int32_t launch_smem(const float* x, int R, int64_t N, int64_t ldr, const PercSpecs& P, int min_members,
                           void* out, cudaStream_t st) {
  ens_perc_smem_kernel<RP><<<(unsigned)((N + kThreadsSmem - 1) / kThreadsSmem), kThreadsSmem, 0, st>>>(
      x, R, N, ldr, P, min_members, (double*)out);
  return launch_status("ens_perc_smem_kernel");
}

extern "C" int32_t xc_ens_percentiles_f32(const float* x, int64_t R, int64_t N, int64_t ldr,
                                          const double* percentiles, int32_t n_per, double alpha, double beta,
                                          int32_t min_members, void* out, void* stream) {
  if (int32_t e = check_columns(x, R, N, ldr)) return e;
  XC_REQUIRE(percentiles && out, "null pointer argument");
  XC_REQUIRE(n_per >= 1 && n_per <= kMaxPer, "1 to %d percentiles per call, got %d", kMaxPer, n_per);
  XC_REQUIRE(alpha >= 0.0 && alpha <= 1.0 && beta >= 0.0 && beta <= 1.0, "alpha and beta must be in [0, 1]");
  XC_REQUIRE(min_members >= 0, "min_members must be >= 0");
  PercSpecs P{};
  P.np = n_per;
  for (int p = 0; p < n_per; ++p) {
    const double per = percentiles[p];
    XC_REQUIRE(per >= 0.0 && per <= 100.0, "percentiles must be in [0, 100]");
    P.s[p].q = per / 100.0;
    P.s[p].c = alpha + P.s[p].q * (1 - alpha - beta);
    P.s[p].top = 1;
  }
  const int r = (int)R;
  cudaStream_t st = (cudaStream_t)stream;
  if (r == 1) return launch_reg<1, float>(x, r, N, ldr, P, min_members, out, st);
  if (r <= 2) return launch_reg<2, double>(x, r, N, ldr, P, min_members, out, st);
  if (r <= 4) return launch_reg<4, double>(x, r, N, ldr, P, min_members, out, st);
  if (r <= 8) return launch_reg<8, double>(x, r, N, ldr, P, min_members, out, st);
  if (r <= 16) return launch_reg<16, double>(x, r, N, ldr, P, min_members, out, st);
  if (r <= 32) return launch_reg<32, double>(x, r, N, ldr, P, min_members, out, st);
  if (r <= 64) return launch_smem<64>(x, r, N, ldr, P, min_members, out, st);
  return launch_smem<128>(x, r, N, ldr, P, min_members, out, st);
}

extern "C" int32_t xc_ens_moments_f32(const float* x, int64_t R, int64_t N, int64_t ldr, const double* weights,
                                      int32_t min_members, void* mean, void* std, float* vmin, float* vmax,
                                      void* stream) {
  if (int32_t e = check_columns(x, R, N, ldr)) return e;
  XC_REQUIRE(mean && std && vmin && vmax, "null pointer argument");
  XC_REQUIRE(min_members >= 0, "min_members must be >= 0");
  ens_moments_kernel<<<(unsigned)((N + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      x, (int)R, N, ldr, weights, min_members, mean, std, vmin, vmax);
  return launch_status("ens_moments_kernel");
}

extern "C" int32_t xc_ens_robustness_f32(const float* fut, int64_t Tf, int64_t ldf_r, int64_t ldf_t,
                                         const float* ref, int64_t Tr, int64_t ldr_r, int64_t ldr_t,
                                         const float* ref_annual, int64_t P, int64_t lda_r, const double* ys_time,
                                         int64_t R, int64_t C, const double* weights, int32_t test, double param,
                                         int32_t strict_sign, double* fractions, float* pvals, void* stream) {
  XC_REQUIRE(fut && fractions, "null pointer argument");
  XC_REQUIRE(R >= 1 && R <= 2147483647LL && C > 0 && C <= 2147483647LL * kThreads && Tf > 0, "bad shape");
  XC_REQUIRE(ldf_r >= C && (Tf == 1 || ldf_t >= C), "bad shape");
  XC_REQUIRE(!ref || (Tr > 0 && ldr_r >= C && (Tr == 1 || ldr_t >= C)), "bad shape");
  XC_REQUIRE(test >= XC_ENS_TEST_NONE && test <= XC_ENS_TEST_IPCC, "unknown test %d", test);
  XC_REQUIRE(test != XC_ENS_TEST_IPCC || (ref_annual && ys_time && P > 0 && lda_r >= P * C),
             "ipcc-ar6-c needs the annual means of ref and their YS timestamps");
  XC_REQUIRE(ref || test == XC_ENS_TEST_NONE || test == XC_ENS_TEST_ABS,
             "When deltas are given (ref=None), 'test' must be None or 'threshold'.");
  XC_REQUIRE(!pvals || test == XC_ENS_TEST_TTEST || test == XC_ENS_TEST_WELCH, "pvals are given by the t-tests only");
  XC_REQUIRE(param == param, "the test parameter is NaN");
  ens_robustness_kernel<<<(unsigned)((C + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      fut, Tf, ldf_r, ldf_t, ref, Tr, ldr_r, ldr_t, ref_annual, P, lda_r, ys_time, (int)R, C, weights, test, param,
      strict_sign, fractions, pvals);
  return launch_status("ens_robustness_kernel");
}
