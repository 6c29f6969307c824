// Chill portions, chill units and the hourly temperature they run on, on the device (xc_chill_*,
// include/xclim_b200.h c1).  The hourly profile and both models live in chill_core.cuh, which the CPU test-suite
// also builds for the host; this file adds the thread mapping, the argument checks and the launches.
//
// A lane owns one (cell, period) and walks the period once in time order: blockIdx.x picks 128 cells, blockIdx.y the
// period, so each day's (or hour's) row is one coalesced 128-byte segment per warp, and the weight row of a day is
// shared by the lanes of a latitude.  The fused kernel makes the 24 hours of a day in registers from that day's
// tasmin / tasmax and the next day's tasmin: the hourly series is never stored.  Bound: about four float64 exp per
// selected hour for the portions (FP64 pipe).  Built with -fmad=false: the reference's numpy arithmetic does not
// contract multiply-adds.
#include "common.cuh"
#include "chill_core.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;

template <bool FUSED>
__global__ void __launch_bounds__(kThreads) chill_kernel(const __grid_constant__ chill::Args a) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= a.C) return;
  chill::run<FUSED>(a, c, (int)blockIdx.y);
}

__global__ void __launch_bounds__(kThreads) chill_generate_kernel(const __grid_constant__ chill::Args a) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= a.C) return;
  chill::generate(a, c);
}

chill::Args daily_args(const float* tasmin, const float* tasmax, int64_t T, int64_t C, int64_t ldx,
                       const double* weights, int32_t L, const int32_t* lat_index) {
  chill::Args a{};
  a.tasmin = tasmin; a.tasmax = tasmax; a.T = T; a.C = C; a.ldx = ldx; a.H = 24 * T;
  a.weights = weights; a.L = L; a.lat_index = lat_index;
  return a;
}

void set_outputs(chill::Args& a, const int32_t* poff, int32_t P, const uint8_t* day_mask, double k_scale,
                 double k_offset, double c_scale, double c_offset, int32_t what, double* out_cp, double* out_cu,
                 int32_t* out_valid) {
  a.poff = poff; a.P = P; a.day_mask = day_mask;
  a.k_scale = k_scale; a.k_offset = k_offset; a.c_scale = c_scale; a.c_offset = c_offset;
  a.what = what; a.out_cp = out_cp; a.out_cu = out_cu; a.out_valid = out_valid;
}

template <bool FUSED>
int32_t launch(const chill::Args& a, int kind, void* stream, const char* name) {
  const char* msg = nullptr;
  const int32_t st = chill::check_args(a, kind, &msg);
  if (st != XC_OK) {
    set_error("%s", msg);
    return st;
  }
  const unsigned bx = (unsigned)((a.C + kThreads - 1) / kThreads);
  if (kind == 2) chill_generate_kernel<<<bx, kThreads, 0, (cudaStream_t)stream>>>(a);
  else chill_kernel<FUSED><<<dim3(bx, (unsigned)a.P), kThreads, 0, (cudaStream_t)stream>>>(a);
  return launch_status(name);
}

}  // namespace
}  // namespace xc

extern "C" int32_t xc_chill_daily_f32(const float* tasmin, const float* tasmax, int64_t T, int64_t C, int64_t ldx,
                                      const double* weights, int32_t L, const int32_t* lat_index,
                                      const int32_t* period_offsets, int32_t P, const uint8_t* day_mask,
                                      double k_scale, double k_offset, double c_scale, double c_offset, int32_t what,
                                      double* out_cp, double* out_cu, int32_t* out_valid, void* stream) {
  using namespace xc;
  chill::Args a = daily_args(tasmin, tasmax, T, C, ldx, weights, L, lat_index);
  set_outputs(a, period_offsets, P, day_mask, k_scale, k_offset, c_scale, c_offset, what, out_cp, out_cu, out_valid);
  return launch<true>(a, 0, stream, "chill_kernel<fused>");
}

extern "C" int32_t xc_chill_hourly(const void* x, int32_t x_f64, int64_t H, int64_t C, int64_t ldx,
                                   const int32_t* period_offsets, int32_t P, const uint8_t* day_mask, double k_scale,
                                   double k_offset, double c_scale, double c_offset, int32_t what, double* out_cp,
                                   double* out_cu, int32_t* out_valid, void* stream) {
  using namespace xc;
  chill::Args a{};
  a.hourly = x; a.hourly_f64 = x_f64 != 0; a.H = H; a.T = (H + 23) / 24; a.C = C; a.ldx = ldx;
  set_outputs(a, period_offsets, P, day_mask, k_scale, k_offset, c_scale, c_offset, what, out_cp, out_cu, out_valid);
  return launch<false>(a, 1, stream, "chill_kernel<hourly>");
}

extern "C" int32_t xc_hourly_temperature_f32(const float* tasmin, const float* tasmax, int64_t T, int64_t C,
                                             int64_t ldx, const double* weights, int32_t L, const int32_t* lat_index,
                                             double* out, void* stream) {
  using namespace xc;
  chill::Args a = daily_args(tasmin, tasmax, T, C, ldx, weights, L, lat_index);
  a.out_hourly = out;
  return launch<true>(a, 2, stream, "chill_generate_kernel");
}
