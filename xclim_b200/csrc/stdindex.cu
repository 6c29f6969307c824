// Standardized indices (SPI, SPEI) on the device: the per-(cell, group) distribution fit and the probability
// transform (xc_si_fit_f32, xc_si_apply_f32, include/xclim_b200.h).
//
// Replaces indices/stats.py `standardized_index_fit_params` (:944-953), where every (cell, group) sample is one
// scipy call inside xr.apply_ufunc(vectorize=True), and the transform of `standardized_index` (:1155-1191), a
// per-element scipy cdf then ppf.  The arithmetic lives in stdindex_core.cuh, which the CPU test-suite also
// compiles for the host; this file adds the thread mapping and the argument checks.
//
// Fit: one lane per cell walks the groups in turn.  For each group it reads the group's calibration rows (one
// coalesced row segment per step across the warp), counts zeros and non-NaN values, and packs the values that
// enter the fit, minus floc, into a per-cell column of the workspace (value k of cell c at k * C + c, so the
// warp's writes and later reads are coalesced).  The float32 means then walk that column in numpy's pairwise
// order.  Work per cell is a few passes over its calibration values: the fit is a small fraction of the
// preprocessing's HBM traffic.
// Apply: one lane per element, each thread a cell and a run of kApplyRows steps; the CDF (incomplete gamma,
// power or normal CDF) and the inverse normal are float64 iterations, so the kernel is FP64-pipe bound like
// fwi_kernel.  Built with -fmad=false: numpy's float32 moment expressions never fuse a multiply and an add.
#include "common.cuh"
#include "stdindex_core.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;
constexpr int kApplyRows = 16;

__global__ void __launch_bounds__(kThreads)
si_fit_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, const int32_t* __restrict__ goff,
              const int32_t* __restrict__ steps, int32_t G, int32_t dist, int32_t method, int32_t zi, double floc,
              double* __restrict__ params, int32_t* __restrict__ n_zeros, int32_t* __restrict__ n_notnull,
              int32_t* __restrict__ status, float* __restrict__ ws) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int st = si::fit_cell(x, C, ldx, c, goff, steps, G, dist, method, zi, floc, params, n_zeros, n_notnull,
                              ws + c);
  if (st) atomicOr(status, st);
}

__global__ void __launch_bounds__(kThreads)
si_apply_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                const int16_t* __restrict__ gos, const double* __restrict__ params,
                const int32_t* __restrict__ n_zeros, const int32_t* __restrict__ n_notnull, int32_t dist,
                int32_t zi, double interp, double alpha, double beta, double* __restrict__ out, int64_t ldo) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int t0 = blockIdx.y * kApplyRows;
  const int t1 = min((int)T, t0 + kApplyRows);
  for (int t = t0; t < t1; ++t) {
    const int g = __ldg(gos + t);
    double r = NAN;
    if (g >= 0) {
      const double* p = params + (int64_t)g * 3 * C + c;
      const float v = ld_stream(x + (int64_t)t * ldx + c);
      const int32_t nz = zi ? __ldg(n_zeros + (int64_t)g * C + c) : 0;
      const int32_t nn = zi ? __ldg(n_notnull + (int64_t)g * C + c) : 0;
      r = si::standardized(dist, v, __ldg(p), __ldg(p + C), __ldg(p + 2 * C), zi != 0, nz, nn, interp, alpha, beta);
    }
    out[(int64_t)t * ldo + c] = r;
  }
}

}  // namespace
}  // namespace xc

using namespace xc;

static int32_t check_dist_method(int32_t dist, int32_t method) {
  XC_REQUIRE(dist == XC_SI_GAMMA || dist == XC_SI_FISK || dist == XC_SI_LOGNORM, "unknown distribution %d", dist);
  XC_REQUIRE(method == XC_SI_APP || method == XC_SI_ML, "unknown fitting method %d", method);
  if (method == XC_SI_ML && dist == XC_SI_FISK) {
    set_error("fisk ML has no closed form with a fixed loc: scipy optimises it numerically");
    return XC_ERR_UNSUPPORTED;
  }
  return XC_OK;
}

extern "C" int64_t xc_si_fit_workspace_bytes(int64_t C, int32_t max_n) {
  if (C <= 0 || max_n < 0) return -1;
  return (int64_t)(max_n > 0 ? max_n : 1) * C * 4;
}

extern "C" int32_t xc_si_fit_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* group_offsets,
                                 const int32_t* steps, int32_t G, int32_t max_n, int32_t dist, int32_t method,
                                 int32_t zero_inflated, double floc, double* params, int32_t* n_zeros,
                                 int32_t* n_notnull, int32_t* status, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  XC_REQUIRE(x && group_offsets && steps && params && status && workspace, "null pointer argument");
  XC_REQUIRE(!zero_inflated || (n_zeros && n_notnull), "zero-inflated fits need the n_zeros / n_notnull outputs");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && T < 2147483647LL && C <= 2147483647LL, "bad shape");
  XC_REQUIRE(G > 0 && max_n >= 0, "bad group count");
  XC_REQUIRE(workspace_bytes >= xc_si_fit_workspace_bytes(C, max_n), "workspace too small");
  XC_REQUIRE(floc == floc && !isinf(floc), "floc must be finite");
  if (int32_t e = check_dist_method(dist, method)) return e;
  si_fit_kernel<<<(unsigned)((C + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      x, C, ldx, group_offsets, steps, G, dist, method, zero_inflated, floc, params,
      zero_inflated ? n_zeros : nullptr, zero_inflated ? n_notnull : nullptr, status, (float*)workspace);
  return launch_status("si_fit_kernel");
}

extern "C" int32_t xc_si_apply_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const int16_t* group_of_step,
                                   int32_t G, const double* params, const int32_t* n_zeros, const int32_t* n_notnull,
                                   int32_t dist, int32_t zero_inflated, double interp, double alpha, double beta,
                                   double* out, int64_t ldo, void* stream) {
  XC_REQUIRE(x && group_of_step && params && out, "null pointer argument");
  XC_REQUIRE(!zero_inflated || (n_zeros && n_notnull), "zero-inflated transforms need the n_zeros / n_notnull counts");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && ldo >= C && T < 2147483647LL && C <= 2147483647LL, "bad shape");
  XC_REQUIRE(G > 0 && G <= 32767, "bad group count");
  XC_REQUIRE(dist == XC_SI_GAMMA || dist == XC_SI_FISK || dist == XC_SI_LOGNORM, "unknown distribution %d", dist);
  XC_REQUIRE((T + kApplyRows - 1) / kApplyRows <= 65535, "series longer than %d steps", 65535 * kApplyRows);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)((T + kApplyRows - 1) / kApplyRows), 1);
  si_apply_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(x, T, C, ldx, group_of_step, params, n_zeros, n_notnull,
                                                              dist, zero_inflated, interp, alpha, beta, out, ldo);
  return launch_status("si_apply_kernel");
}
