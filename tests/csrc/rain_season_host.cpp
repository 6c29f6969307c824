// Host build of the rain-season scan (xclim_b200/csrc/rain_season_core.cuh) for the CPU test-suite: the lane loop of
// rain_season_kernel (rain_season.cu) over host arrays, compiled with g++ -ffp-contract=off, behind the argument
// checks of the C-ABI entry point.
#include <stdint.h>

#include "../../xclim_b200/csrc/rain_season_core.cuh"

using namespace xc::rs;

extern "C" {

// xc_rain_season_f32 on host arrays; returns its status (0, -1 invalid, -2 unsupported) and leaves the message in *msg
int32_t rain_season_host(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* poff, int32_t P,
                         const uint8_t* mask, float scale, double thr_wet, int32_t window_wet, int32_t window_not_dry,
                         double thr_dry_start, int32_t window_dry_start, int32_t method_dry_start, double thr_dry_end,
                         int32_t window_dry_end, int32_t method_dry_end, int32_t* out_start, int32_t* out_end,
                         const char** msg) {
  const Args a = make_args(x, T, C, ldx, poff, P, mask, scale, thr_wet, window_wet, window_not_dry, thr_dry_start,
                           window_dry_start, method_dry_start, thr_dry_end, window_dry_end, method_dry_end, out_start,
                           out_end);
  const int32_t st = check_args(a, msg);
  if (st) return st;
  for (int p = 0; p < P; ++p)
    for (int64_t c = 0; c < C; ++c) scan(a, c, p);
  return 0;
}

}  // extern "C"
