// Host build of the frequency-analysis device code (xclim_b200/csrc/evfit_core.cuh) for the CPU test-suite: the
// same per-cell fits and per-element transforms, compiled with g++ -ffp-contract=off.
#include <stdint.h>

#include "../../xclim_b200/csrc/evfit_core.cuh"

using namespace xc::ev;

extern "C" {

// xc_ev_fit_f32 on host arrays, cell by cell (workspace: T * C floats).
int32_t ev_host_fit(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t dist, double* params, float* ws) {
  int st = 0;
  for (int64_t c = 0; c < C; ++c) st |= fit_cell(x, T, C, ldx, c, dist, params, ws + c);
  return st;
}

// xc_ev_transform_f64 on host arrays.
void ev_host_transform(const double* params, int64_t C, int32_t dist, int32_t kind, const double* q, int32_t nq,
                       double* out) {
  const bool gev = dist == kGev;
  for (int32_t j = 0; j < nq; ++j)
    for (int64_t c = 0; c < C; ++c)
      out[(int64_t)j * C + c] = transform(dist, kind, q[j], gev ? params[c] : 0.0, params[(gev ? C : 0) + c],
                                          params[(gev ? 2 * C : C) + c]);
}

// The GEV negative log-likelihood of the device code at theta = (c, loc, log scale), and its gradient / Hessian.
double ev_host_gev_nnlf(const double* x, int32_t n, const double* th) {
  return gev_nnlf([&](int k) { return (float)x[k]; }, n, th);
}
void ev_host_gev_derivs(const float* x, int32_t n, const double* th, double* g, double* H) {
  gev_derivs([&](int k) { return x[k]; }, n, th, g, H);
}

}  // extern "C"
