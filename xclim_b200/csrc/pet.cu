// Potential evapotranspiration and the water budget on the device (xc_pet_daily_f32, xc_pet_monthly_f32,
// include/xclim_b200.h p1).  The arithmetic lives in pet_core.cuh, which the CPU test-suite also builds for the
// host; this file adds the thread-to-element mapping and the argument checks.
//
// Daily methods: a lane owns one cell and walks kRowsPerLane consecutive rows, so every load and store of a row
// is one coalesced 128-byte segment per warp; the solar term is one float64 read of a (row, latitude) table
// that the cells of a latitude share through L1 / L2.  Monthly methods: a lane walks one cell's whole series,
// month by month, with float64 sums.  Built with -fmad=false, like the host build (g++ -ffp-contract=off).
#include "common.cuh"
#include "pet_core.cuh"

namespace xc {
namespace {

constexpr int kThreads = 256;
constexpr int kRowsPerLane = 16;

template <int METHOD>
__global__ void __launch_bounds__(kThreads) pet_daily_kernel(const __grid_constant__ pet::Args a) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= a.C) return;
  const int64_t t0 = (int64_t)blockIdx.y * kRowsPerLane;
  const int64_t t1 = t0 + kRowsPerLane < a.T ? t0 + kRowsPerLane : a.T;
#pragma unroll 4
  for (int64_t t = t0; t < t1; ++t) a.out[t * a.ldx + c] = pet::daily_value(a, t, c, METHOD);
}

__global__ void __launch_bounds__(128) pet_monthly_kernel(const __grid_constant__ pet::Args a) {
  const int64_t c = (int64_t)blockIdx.x * 128 + threadIdx.x;
  if (c >= a.C) return;
  pet::monthly_cell(a, c);
}

pet::Args make_args(const float* const* inputs, int64_t T, int64_t C, int64_t ldx, const double* table, int64_t L,
                    const int32_t* lat_index, const XcPetParams* P, float* out) {
  pet::Args a{};
  for (int k = 0; k < XC_PET_N_IN; ++k) a.in[k] = inputs[k];
  a.T = T; a.C = C; a.ldx = ldx;
  a.table = table; a.L = L; a.lat_index = lat_index;
  a.P = *P;
  a.out = out;
  return a;
}

}  // namespace
}  // namespace xc

extern "C" int32_t xc_pet_daily_f32(const float* const* inputs, int64_t T, int64_t C, int64_t ldx,
                                    const double* table, int64_t L, const int32_t* lat_index,
                                    const XcPetParams* params_host, float* out, void* stream) {
  using namespace xc;
  XC_REQUIRE(inputs != nullptr && params_host != nullptr, "null pointer argument");
  const pet::Args a = make_args(inputs, T, C, ldx, table, L, lat_index, params_host, out);
  const char* msg = pet::check_args(a, false);
  XC_REQUIRE(msg == nullptr, "%s", msg);
  const int64_t row_blocks = (T + kRowsPerLane - 1) / kRowsPerLane;
  XC_REQUIRE(row_blocks < 65536, "series longer than %d steps", 65535 * kRowsPerLane);
  const dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)row_blocks);
  cudaStream_t s = (cudaStream_t)stream;
  switch (a.P.method) {
    case XC_PET_BR65: pet_daily_kernel<XC_PET_BR65><<<grid, kThreads, 0, s>>>(a); break;
    case XC_PET_HG85: pet_daily_kernel<XC_PET_HG85><<<grid, kThreads, 0, s>>>(a); break;
    case XC_PET_MB05: pet_daily_kernel<XC_PET_MB05><<<grid, kThreads, 0, s>>>(a); break;
    case XC_PET_ALLEN98: pet_daily_kernel<XC_PET_ALLEN98><<<grid, kThreads, 0, s>>>(a); break;
    default: pet_daily_kernel<XC_PET_GIVEN><<<grid, kThreads, 0, s>>>(a); break;
  }
  return launch_status("pet_daily_kernel");
}

extern "C" int32_t xc_pet_monthly_f32(const float* const* inputs, int64_t T, int64_t C, int64_t ldx,
                                      const int32_t* moff, int64_t M, const int32_t* yoff, int64_t Y,
                                      const double* mdays, const double* table, int64_t L, const int32_t* lat_index,
                                      const XcPetParams* params_host, float* out, void* stream) {
  using namespace xc;
  XC_REQUIRE(inputs != nullptr && params_host != nullptr, "null pointer argument");
  pet::Args a = make_args(inputs, T, C, ldx, table, L, lat_index, params_host, out);
  a.moff = moff; a.M = M; a.yoff = yoff; a.Y = Y; a.mdays = mdays;
  const char* msg = pet::check_args(a, true);
  XC_REQUIRE(msg == nullptr, "%s", msg);
  pet_monthly_kernel<<<(unsigned)((C + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
  return launch_status("pet_monthly_kernel");
}
