// Host build of the chill code (xclim_b200/csrc/chill_core.cuh) for the CPU test-suite: the lane loops of
// chill_kernel and chill_generate_kernel (chill.cu) over host arrays, compiled with g++ -ffp-contract=off, behind
// the argument checks of the C-ABI entry points.
#include <stdint.h>

#include "../../xclim_b200/csrc/chill_core.cuh"

using namespace xc::chill;

extern "C" {

// xc_chill_daily_f32 (kind 0) or xc_chill_hourly (kind 1) on host arrays; returns the status, message in *msg
int32_t chill_host(int32_t kind, const float* tasmin, const float* tasmax, const void* hourly, int32_t hourly_f64,
                   int64_t T, int64_t H, int64_t C, int64_t ldx, const double* weights, int32_t L,
                   const int32_t* lat_index, const int32_t* poff, int32_t P, const uint8_t* day_mask, double k_scale,
                   double k_offset, double c_scale, double c_offset, int32_t what, double* out_cp, double* out_cu,
                   int32_t* out_valid, const char** msg) {
  Args a{};
  a.tasmin = tasmin; a.tasmax = tasmax; a.hourly = hourly; a.hourly_f64 = hourly_f64;
  a.T = T; a.H = H; a.C = C; a.ldx = ldx; a.weights = weights; a.L = L; a.lat_index = lat_index;
  a.poff = poff; a.P = P; a.day_mask = day_mask;
  a.k_scale = k_scale; a.k_offset = k_offset; a.c_scale = c_scale; a.c_offset = c_offset;
  a.what = what; a.out_cp = out_cp; a.out_cu = out_cu; a.out_valid = out_valid;
  const int32_t st = check_args(a, kind, msg);
  if (st) return st;
  for (int p = 0; p < P; ++p)
    for (int64_t c = 0; c < C; ++c) {
      if (kind == 0) run<true>(a, c, p);
      else run<false>(a, c, p);
    }
  return 0;
}

// xc_hourly_temperature_f32 on host arrays
int32_t hourly_temperature_host(const float* tasmin, const float* tasmax, int64_t T, int64_t C, int64_t ldx,
                                const double* weights, int32_t L, const int32_t* lat_index, double* out,
                                const char** msg) {
  Args a{};
  a.tasmin = tasmin; a.tasmax = tasmax; a.T = T; a.H = 24 * T; a.C = C; a.ldx = ldx;
  a.weights = weights; a.L = L; a.lat_index = lat_index; a.out_hourly = out;
  const int32_t st = check_args(a, 2, msg);
  if (st) return st;
  for (int64_t c = 0; c < C; ++c) generate(a, c);
  return 0;
}

// the Dynamic Model's E of every hour of one period (n hours in K)
void dynamic_trace(const double* tk, int64_t n, double* E, double* sum) {
  Dynamic dyn;
  for (int64_t i = 0; i < n; ++i) E[i] = dyn.step(tk[i]);
  *sum = dyn.sum;
}

}  // extern "C"
