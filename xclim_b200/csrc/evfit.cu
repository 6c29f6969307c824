// Frequency analysis on the device: the per-cell maximum-likelihood fit of norm / gumbel_r / genextreme and the
// quantile / CDF transform of the fitted laws (xc_ev_fit_f32, xc_ev_transform_f64, include/xclim_b200.h).
//
// Replaces indices/stats.py `fit` (:115-218), where every cell is one scipy call inside
// xr.apply_ufunc(vectorize=True), and the per-cell scipy ppf / isf / cdf of `parametric_quantile` (:221-289)
// and `parametric_cdf` (:294-360).  The arithmetic lives in evfit_core.cuh, which the CPU test-suite also
// compiles for the host; this file adds the thread mapping and the argument checks.
//
// Fit: one lane per cell.  The lane reads its column of the (T, C) input (one coalesced row segment per step
// across the warp), compacts the finite values into its workspace column (value k of cell c at k * C + c) and
// runs every later pass over that column, again coalesced across the warp.  The GEV Newton iterations are
// float64 log1p / exp per value and pass, so the kernel is FP64-pipe bound.  Built with -fmad=false: the
// normal fit follows numpy's float32 expressions, which never fuse a multiply and an add.
// Transform: one thread per (probability, cell) element.
#include "common.cuh"
#include "evfit_core.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads)
ev_fit_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, int32_t dist,
              double* __restrict__ params, int32_t* __restrict__ status, float* __restrict__ ws) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int st = ev::fit_cell(x, T, C, ldx, c, dist, params, ws + c);
  if (st) atomicOr(status, st);
}

__global__ void __launch_bounds__(kThreads)
ev_transform_kernel(const double* __restrict__ params, int64_t C, int32_t dist, int32_t kind,
                    const double* __restrict__ q, double* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int j = blockIdx.y;
  const bool gev = dist == ev::kGev;
  const double shape = gev ? __ldg(params + c) : 0.0;
  const double loc = __ldg(params + (gev ? C : 0) + c);
  const double scale = __ldg(params + (gev ? 2 * C : C) + c);
  out[(int64_t)j * C + c] = ev::transform(dist, kind, __ldg(q + j), shape, loc, scale);
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int64_t xc_ev_fit_workspace_bytes(int64_t T, int64_t C) {
  if (T <= 0 || C <= 0) return -1;
  return T * C * 4;
}

extern "C" int32_t xc_ev_fit_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t dist, double* params,
                                 int32_t* status, void* workspace, int64_t workspace_bytes, void* stream) {
  XC_REQUIRE(x && params && status && workspace, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && T < 2147483647LL && C <= 2147483647LL, "bad shape");
  XC_REQUIRE(dist == XC_EV_NORM || dist == XC_EV_GUMBEL_R || dist == XC_EV_GENEXTREME, "unknown distribution %d",
             dist);
  XC_REQUIRE(workspace_bytes >= xc_ev_fit_workspace_bytes(T, C), "workspace too small");
  ev_fit_kernel<<<(unsigned)((C + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      x, T, C, ldx, dist, params, status, (float*)workspace);
  return launch_status("ev_fit_kernel");
}

extern "C" int32_t xc_ev_transform_f64(const double* params, int64_t C, int32_t dist, int32_t kind, const double* q,
                                       int32_t nq, double* out, void* stream) {
  XC_REQUIRE(params && q && out, "null pointer argument");
  XC_REQUIRE(C > 0 && C <= 2147483647LL, "bad shape");
  XC_REQUIRE(nq > 0 && nq <= 65535, "bad number of probabilities / values %d", nq);
  XC_REQUIRE(dist == XC_EV_NORM || dist == XC_EV_GUMBEL_R || dist == XC_EV_GENEXTREME, "unknown distribution %d",
             dist);
  XC_REQUIRE(kind == XC_EV_PPF || kind == XC_EV_ISF || kind == XC_EV_CDF, "unknown transform %d", kind);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)nq, 1);
  ev_transform_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(params, C, dist, kind, q, out);
  return launch_status("ev_transform_kernel");
}
