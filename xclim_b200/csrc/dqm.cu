// Detrended quantile mapping (sdba / xsdba `DetrendedQuantileMapping`, group="time"): the polynomial trend and the
// adjust pass; and the trend removal of xclim.indices.generic.detrend (indices/generic.py:1711-1736).
//
// The arithmetic of DQM lives in the third-party package xsdba (re-exported by sdba.py:11) whose sources are not part
// of the reference tree: this file restates the published algorithm (PARITY UNPINNED, see DESIGN.md).  Its train
// step is EQM's selection on mean-normalised series (eqm.cu, xc_dqm_train_f32).  adjust, per cell of sim:
//   y      : float32(sim (+|*) scaling)                           (xsdba dqm_adjust: sim scaled by the mean ratio)
//   trend  : tau = least-squares polynomial of degree D over the valid steps of y (PolyDetrend: xarray polyfit /
//            polyval); the daily axis is gap-free, so the nanosecond coordinate is affine in the step index t and
//            the fitted values are those of the fit in the basis u_t = (2t - (T - 1)) / max(T - 1, 1);
//   detrend: d = y - tau ("+") or y * (1 / tau) ("*"), float64;
//   factor : scipy interp1d(hist_q, af, kind=interp, bounds_error=False, fill_value=(first, last)) at d over the
//            entries where neither table is NaN (xsdba's _interp_on_quantiles_1D), float32;
//   retrend: scen = float32((d (+|*) f) (+|*) tau), inner operations in float64.
// generic.detrend is x - tau with the trend of x itself, float64.
//
// Design.  The fit is one streaming pass in (time, cell) order: a lane owns one cell (four with 128-bit loads, as
// the period kernels do) and accumulates sum u^k (k <= 2D) and sum u^k y (k <= D) in float64 over its valid steps,
// then solves the (D + 1)^2 normal equations (well conditioned on [-1, 1]: the Gram matrix of 1, u, u^2 has a
// condition number near 20).  adjust and detrend are a second streaming pass that evaluates the trend from the
// coefficients.  The sums run in time order within a lane, so the coefficients are deterministic.
//
// The file is compiled with -fmad=false (_build.EXTRA_FLAGS): the trend, the detrend and the retrend are then the
// float64 operations of the oracle one by one, bit for bit given the same coefficients.  The interpolation, the
// position table and the row loop come from qmap.cuh, shared with the kernels compiled with fused multiply-adds
// allowed: that code is explicit rounding intrinsics, comparisons and integer arithmetic only, so -fmad cannot
// change it.
#include <float.h>

#include <algorithm>

#include "qmap.cuh"

namespace xc {
namespace {

constexpr int kFitThreads = 128;
constexpr int kAdjThreads = 128;
constexpr int kLut = 32;          // coarse position table per cell
constexpr int kMaxDeg = 2;

__device__ __forceinline__ double basis_u(int64_t t, int64_t T) {
  return (double)(2 * t - (T - 1)) / (double)(T > 1 ? T - 1 : 1);
}

// ((c2 u + c1) u + c0), Horner from the highest coefficient of the fit's degree (no fused multiply-add here)
__device__ __forceinline__ double trend_at(double c0, double c1, double c2, int deg, double u) {
  if (deg == 2) return (c2 * u + c1) * u + c0;
  if (deg == 1) return c1 * u + c0;
  return c0;
}

// y of the fit: x, or float32(x (+|*) s) (mode 1 "+", 2 "*")
__device__ __forceinline__ float fit_input(float x, int mode, float s) {
  if (mode == 1) return __fadd_rn(x, s);
  if (mode == 2) return __fmul_rn(x, s);
  return x;
}

template <int VEC>
struct FVec {
  float v[VEC];
};
template <int VEC>
__device__ __forceinline__ FVec<VEC> ld_vec(const float* p) {
  FVec<VEC> r;
  if constexpr (VEC == 4) {
    const float4 q = ld_stream4(p);
    r.v[0] = q.x; r.v[1] = q.y; r.v[2] = q.z; r.v[3] = q.w;
  } else {
    r.v[0] = ld_stream(p);
  }
  return r;
}

// Normal equations G c = b of degree d (d + 1 unknowns), G[i][j] = S[i + j], b[i] = R[i]; Gaussian elimination
// with partial pivoting in float64.  Coefficients above d are 0.
template <int D>
__device__ __forceinline__ void solve_normal(const double* S, const double* R, int d, double* c) {
  double a[D + 1][D + 2];
#pragma unroll
  for (int i = 0; i <= D; ++i) {
#pragma unroll
    for (int j = 0; j <= D; ++j) a[i][j] = (i <= d && j <= d) ? S[i + j] : (i == j ? 1.0 : 0.0);
    a[i][D + 1] = (i <= d) ? R[i] : 0.0;
  }
#pragma unroll
  for (int k = 0; k <= D; ++k) {
    int p = k;
    double best = fabs(a[k][k]);
#pragma unroll
    for (int i = k + 1; i <= D; ++i) {
      if (fabs(a[i][k]) > best) { best = fabs(a[i][k]); p = i; }
    }
#pragma unroll
    for (int j = 0; j <= D + 1; ++j) {   // swap rows k and p (register arrays: by selects)
      double rk = a[k][j];
#pragma unroll
      for (int i = k + 1; i <= D; ++i) {
        if (i == p) { const double tmp = a[i][j]; a[i][j] = rk; rk = tmp; }
      }
      a[k][j] = rk;
    }
#pragma unroll
    for (int i = k + 1; i <= D; ++i) {
      const double f = a[i][k] / a[k][k];
#pragma unroll
      for (int j = k; j <= D + 1; ++j) a[i][j] = a[i][j] - f * a[k][j];
    }
  }
#pragma unroll
  for (int i = D; i >= 0; --i) {
    double s = a[i][D + 1];
#pragma unroll
    for (int j = i + 1; j <= D; ++j) s = s - a[i][j] * c[j];
    c[i] = s / a[i][i];
  }
}

// One lane = VEC adjacent cells; the whole series in time order, kU rows in flight.  coef: (D + 1, C) float64.
template <int D, int VEC>
__global__ void __launch_bounds__(kFitThreads)
poly_fit_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, int32_t mode,
                const float* __restrict__ scaling, double* __restrict__ coef) {
  constexpr int kU = (VEC == 4) ? 8 : 16;
  const int64_t c0 = ((int64_t)blockIdx.x * kFitThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  float s[VEC];
  double S[VEC][2 * D + 1], R[VEC][D + 1];
  int32_t n[VEC];
  bool inf[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    s[i] = (mode != 0) ? scaling[c0 + i] : 0.f;
    n[i] = 0;
    inf[i] = false;
#pragma unroll
    for (int k = 0; k <= 2 * D; ++k) S[i][k] = 0.0;
#pragma unroll
    for (int k = 0; k <= D; ++k) R[i][k] = 0.0;
  }
  auto take = [&](const FVec<VEC>& r, int64_t t) {
    const double u = basis_u(t, T);
    double pw[2 * D + 1];
    pw[0] = 1.0;
#pragma unroll
    for (int k = 1; k <= 2 * D; ++k) pw[k] = pw[k - 1] * u;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float y = fit_input(r.v[i], mode, s[i]);
      if (y == y) {
        const double yd = (double)y;
        ++n[i];
        inf[i] = inf[i] || !(fabsf(y) < INFINITY);
#pragma unroll
        for (int k = 1; k <= 2 * D; ++k) S[i][k] += pw[k];
#pragma unroll
        for (int k = 0; k <= D; ++k) R[i][k] += pw[k] * yd;
      }
    }
  };
  const float* p = x + c0;
  int64_t t = 0;
  for (; t + kU <= T; t += kU) {
    FVec<VEC> r[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) r[u] = ld_vec<VEC>(p + (int64_t)u * ldx);
#pragma unroll
    for (int u = 0; u < kU; ++u) take(r[u], t + u);
    p += (int64_t)kU * ldx;
  }
  for (; t < T; ++t) {
    take(ld_vec<VEC>(p), t);
    p += ldx;
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    double c[D + 1];
    if (n[i] == 0 || inf[i]) {
#pragma unroll
      for (int k = 0; k <= D; ++k) c[k] = NAN;
    } else {
      S[i][0] = (double)n[i];
      const int d = min(D, n[i] - 1);   // n <= D valid steps: the polynomial of degree n - 1 through them
      solve_normal<D>(S[i], R[i], d, c);
    }
#pragma unroll
    for (int k = 0; k <= D; ++k) coef[(int64_t)k * C + c0 + i] = c[k];
  }
}

// adjust: a lane owns a cell and streams rows [t0, t1) of it.  Per lane, in shared memory (column = lane): the search
// keys (linear: the compacted hist_q; nearest: interp1d's bounds between them), the compacted af, and a 32-entry
// position table lut[b] = #{keys in a lower bin than b}, a lower bound of #{keys < d} for d in bin b (the bins are a
// monotone function of the value, qmap::PosTable), from which a short forward scan finds the segment.
template <int INTERP, int KIND>
__global__ void __launch_bounds__(kAdjThreads)
dqm_adjust_kernel(const float* __restrict__ sim, int64_t T, int64_t C, int64_t ldx, const float* __restrict__ af,
                  const float* __restrict__ hist_q, const float* __restrict__ scaling, const double* __restrict__ coef,
                  int32_t nq, int32_t deg, int32_t rows_per_block, float* __restrict__ scen) {
  extern __shared__ float tab[];   // [2][nq][kAdjThreads]: keys, af; then lut [kLut][kAdjThreads] bytes
  float* ks = tab;
  float* ys = tab + (size_t)nq * kAdjThreads;
  unsigned char* lut = reinterpret_cast<unsigned char*>(ys + (size_t)nq * kAdjThreads);
  const int lane = threadIdx.x;
  const int64_t c = (int64_t)blockIdx.x * kAdjThreads + lane;
  if (c >= C) return;
  // interp1d on the entries where neither hist_q nor af is NaN
  int m = 0;
  float xprev = 0.f, x_first = 0.f, x_last = 0.f;
  for (int j = 0; j < nq; ++j) {
    const float h = hist_q[(int64_t)j * C + c], a = af[(int64_t)j * C + c];
    if (h == h && a == a) {
      if (m == 0) x_first = h;
      if (INTERP == 1) ks[m * kAdjThreads + lane] = h;
      else if (m > 0) ks[(m - 1) * kAdjThreads + lane] = qmap::nearest_bound(xprev, h);   // interp1d's nearest bounds
      ys[m * kAdjThreads + lane] = a;
      xprev = h;
      x_last = h;
      ++m;
    }
  }
  const int nk = (INTERP == 1) ? m : m - 1;   // search keys
  const double k_first = nk > 0 ? (double)ks[lane] : 0.0;
  const double k_range = nk > 0 ? (double)ks[(nk - 1) * kAdjThreads + lane] - k_first : 0.0;
  const qmap::PosTable<double, kAdjThreads, kLut, false> pos(ks + lane, lut + lane, k_first, k_range, nk >= 2);
  pos.build(nk, true);
  auto factor = [&](double q) -> float {
    float f;
    if (qmap::interp1d_edges<INTERP>(q, m, [&] { return x_first; }, [&] { return x_last; },
                                     [&](int i) { return ys[i * kAdjThreads + lane]; }, f))
      return f;
    int i = pos.count_below(q, nk);
    if (INTERP == 1) {
      i = min(max(i, 1), m - 1);
      const float x0 = ks[(i - 1) * kAdjThreads + lane], x1 = ks[i * kAdjThreads + lane];
      const float y0 = ys[(i - 1) * kAdjThreads + lane], y1 = ys[i * kAdjThreads + lane];
      return qmap::linear_two_weight(q, x0, x1, y0, y1);
    }
    return ys[i * kAdjThreads + lane];   // nearest: ties to the lower node
  };
  const double c0 = coef[c];
  const double c1 = deg >= 1 ? coef[C + c] : 0.0;
  const double c2 = deg >= 2 ? coef[2 * C + c] : 0.0;
  const float sc = scaling[c];
  const double den = (double)(T > 1 ? T - 1 : 1);
  auto one = [&](float x, int64_t t) -> float {
    const float y = (KIND == 0) ? __fadd_rn(x, sc) : __fmul_rn(x, sc);
    const double tau = trend_at(c0, c1, c2, deg, __ddiv_rn((double)(2 * t - (T - 1)), den));   // basis_u
    const double d = (KIND == 0) ? (double)y - tau : (double)y * (1.0 / tau);
    const double f = (double)factor(d);
    return (float)((KIND == 0) ? (d + f) + tau : (d * f) * tau);
  };
  const int64_t t0 = (int64_t)blockIdx.y * rows_per_block;
  qmap::stream_rows<8>(sim + c, ldx, scen + c, C, t0, min(T, t0 + rows_per_block), one);
}

// generic.detrend: out = x - tau in float64, a lane per cell, rows [t0, t1)
__global__ void __launch_bounds__(kAdjThreads)
detrend_apply_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, const double* __restrict__ coef,
                     int32_t deg, int32_t rows_per_block, double* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kAdjThreads + threadIdx.x;
  if (c >= C) return;
  const double c0 = coef[c];
  const double c1 = deg >= 1 ? coef[C + c] : 0.0;
  const double c2 = deg >= 2 ? coef[2 * C + c] : 0.0;
  const int64_t t0 = (int64_t)blockIdx.y * rows_per_block;
  qmap::stream_rows<8>(x + c, ldx, out + c, C, t0, min(T, t0 + rows_per_block),
                       [&](float v, int64_t t) { return (double)v - trend_at(c0, c1, c2, deg, basis_u(t, T)); });
}

}  // namespace
}  // namespace xc

using namespace xc;

static int32_t check_series(const void* x, int64_t T, int64_t C, int64_t ldx, int32_t degree) {
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C, "bad shape");
  XC_REQUIRE(T < 2147483647LL && C <= 2147483647LL, "series too long or too many cells for one launch");
  XC_REQUIRE(degree >= 0 && degree <= kMaxDeg, "degree must be 0, 1 or 2, got %d", degree);
  (void)x;
  return XC_OK;
}

extern "C" int32_t xc_poly_fit_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t degree, int32_t kind,
                                   const float* scaling, double* coef, void* stream) {
  XC_REQUIRE(x && coef, "null pointer argument");
  if (int32_t e = check_series(x, T, C, ldx, degree)) return e;
  XC_REQUIRE(kind == 0 || kind == 1, "kind must be 0 ('+') or 1 ('*')");
  cudaStream_t st = (cudaStream_t)stream;
  const int32_t mode = scaling ? 1 + kind : 0;
  const bool v4 = (C % 4 == 0) && (ldx % 4 == 0) && aligned16(x);
  auto go = [&](auto DC, auto VC) -> int32_t {
    constexpr int D = decltype(DC)::value, VEC = decltype(VC)::value;
    const int64_t lanes = (C + VEC - 1) / VEC;
    poly_fit_kernel<D, VEC><<<(unsigned)((lanes + kFitThreads - 1) / kFitThreads), kFitThreads, 0, st>>>(
        x, T, C, ldx, mode, scaling, coef);
    return launch_status("poly_fit_kernel");
  };
  auto by_vec = [&](auto DC) -> int32_t {
    return v4 ? go(DC, std::integral_constant<int, 4>{}) : go(DC, std::integral_constant<int, 1>{});
  };
  if (degree == 0) return by_vec(std::integral_constant<int, 0>{});
  if (degree == 1) return by_vec(std::integral_constant<int, 1>{});
  return by_vec(std::integral_constant<int, 2>{});
}

extern "C" int32_t xc_dqm_adjust_f32(const float* sim, int64_t T, int64_t C, int64_t ldx, const float* af,
                                     const float* hist_q, const float* scaling, const double* coef, int32_t nq,
                                     int32_t kind, int32_t interp, int32_t degree, float* scen, void* stream) {
  XC_REQUIRE(sim && af && hist_q && scaling && coef && scen, "null pointer argument");
  if (int32_t e = check_series(sim, T, C, ldx, degree)) return e;
  if (int32_t e = check_qmap_args(nq, 2, 200, kind, interp)) return e;   // node counts fit the 8-bit position table
  const int64_t cblocks = (C + kAdjThreads - 1) / kAdjThreads;
  const RowSplit split = split_rows(T, cblocks, 1, 64);
  const size_t smem = (size_t)2 * nq * kAdjThreads * 4 + (size_t)kLut * kAdjThreads;
  auto kernel = dispatch_interp_kind(interp, kind, [](auto I, auto K) { return dqm_adjust_kernel<I.value, K.value>; });
  if (int32_t e = allow_smem(kernel, smem, "cudaFuncSetAttribute(dqm_adjust_kernel)")) return e;
  kernel<<<dim3((unsigned)cblocks, (unsigned)split.chunks, 1), kAdjThreads, smem, (cudaStream_t)stream>>>(
      sim, T, C, ldx, af, hist_q, scaling, coef, nq, degree, split.rows, scen);
  return launch_status("dqm_adjust_kernel");
}

extern "C" int32_t xc_detrend_apply_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const double* coef,
                                        int32_t degree, double* out, void* stream) {
  XC_REQUIRE(x && coef && out, "null pointer argument");
  if (int32_t e = check_series(x, T, C, ldx, degree)) return e;
  const int64_t cblocks = (C + kAdjThreads - 1) / kAdjThreads;
  const RowSplit split = split_rows(T, cblocks, 1, 64);
  detrend_apply_kernel<<<dim3((unsigned)cblocks, (unsigned)split.chunks, 1), kAdjThreads, 0, (cudaStream_t)stream>>>(
      x, T, C, ldx, coef, degree, split.rows, out);
  return launch_status("detrend_apply_kernel");
}
