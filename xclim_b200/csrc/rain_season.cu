// Rain season start, end and length on the device (xc_rain_season_f32, include/xclim_b200.h r1).  The scan lives in
// rain_season_core.cuh, which the CPU test-suite also builds for the host; this file adds the thread mapping, the
// argument checks and the launch.
//
// A lane owns one (cell, period) and walks the period once: blockIdx.x picks 128 cells, blockIdx.y the period, so
// each step's row is one coalesced 128-byte segment per warp, and the windows the scan re-reads stay in L1 / L2.
#include "common.cuh"
#include "rain_season_core.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads) rain_season_kernel(const __grid_constant__ rs::Args a) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= a.C) return;
  rs::scan(a, c, (int)blockIdx.y);
}

}  // namespace
}  // namespace xc

extern "C" int32_t xc_rain_season_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* period_offsets,
                                      int32_t P, const uint8_t* mask, float scale, double thresh_wet_start,
                                      int32_t window_wet_start, int32_t window_not_dry_start, double thresh_dry_start,
                                      int32_t window_dry_start, int32_t method_dry_start, double thresh_dry_end,
                                      int32_t window_dry_end, int32_t method_dry_end, int32_t* out_start,
                                      int32_t* out_end, void* stream) {
  using namespace xc;
  const rs::Args a = rs::make_args(x, T, C, ldx, period_offsets, P, mask, scale, thresh_wet_start, window_wet_start,
                                   window_not_dry_start, thresh_dry_start, window_dry_start, method_dry_start,
                                   thresh_dry_end, window_dry_end, method_dry_end, out_start, out_end);
  const char* msg = nullptr;
  const int32_t st = rs::check_args(a, &msg);
  if (st != XC_OK) {
    set_error("%s", msg);
    return st;
  }
  const dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P);
  rain_season_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(a);
  return launch_status("rain_season_kernel");
}
