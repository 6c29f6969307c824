// Canadian Forest Fire Weather Index System on the device: one lane walks one grid cell through time and
// writes every requested code / index / mask in the same pass (xc_fwi_f32, include/xclim_b200.h).
//
// Replaces indices/fire/_cffwis.py `_fire_weather_calc` (:680-873), a Python loop over days around numba
// ufuncs that the reference applies per dask chunk (`fire_weather_ufunc`, :1132-1141).  The day loop itself
// lives in fwi_core.cuh, which is also compiled for the host by the CPU test-suite; this file adds the
// thread-to-cell mapping, the tables in constant memory and the argument checks.  Lanes of a warp own
// adjacent cells, so every load / store of a time step is one coalesced 128-byte row segment per array.
//
// Bound: each element costs about twenty float64 transcendental evaluations (exp / log / pow of the three
// moisture codes) against 4 loads + up to 7 stores of 4 bytes, i.e. the kernel is FP64-pipe bound, not HBM
// bound (SURVEY.md 8f.4: "same per-cell streaming shape, different math").  Built with -fmad=false: the
// reference's numba / numpy arithmetic does not contract multiply-adds.
#include "common.cuh"
#include "fwi_core.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;

__constant__ double c_day_lengths[60] = XC_FWI_DAY_LENGTHS;
__constant__ double c_day_length_factors[36] = XC_FWI_DAY_LENGTH_FACTORS;

template <bool RINGS>
__global__ void __launch_bounds__(kThreads) fwi_kernel(const __grid_constant__ fwi::Args a) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= a.C) return;
  fwi::run_cell<RINGS>(a, c, c_day_lengths, c_day_length_factors);
}

__global__ void __launch_bounds__(256)
fwi_elementwise_kernel(int kind, const float* __restrict__ a, const float* __restrict__ b, int64_t n, double p0,
                       double p1, double p2, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = fwi::elementwise(kind, a[i], b ? b[i] : 0.0f, p0, p1, p2);
}

}  // namespace
}  // namespace xc

extern "C" int32_t xc_fwi_f32(const float* tas, const float* pr, const float* hurs, const float* ws, const float* snd,
                              const uint8_t* season_mask_in, const int8_t* month, const double* lat,
                              const float* dc0, const float* dmc0, const float* ffmc0, const float* winter_pr0,
                              int64_t T, int64_t C, int64_t ldx, const XcFwiParams* params_host,
                              float* DC, float* DMC, float* FFMC, float* ISI, float* BUI, float* FWI, float* DSR,
                              uint8_t* season_mask_out, float* winter_pr_out, void* stream) {
  using namespace xc;
  XC_REQUIRE(params_host != nullptr, "null pointer argument");
  fwi::Args a{};
  a.tas = tas; a.pr = pr; a.hurs = hurs; a.ws = ws; a.snd = snd;
  a.mask_in = season_mask_in; a.month = month; a.lat = lat;
  a.dc0 = dc0; a.dmc0 = dmc0; a.ffmc0 = ffmc0; a.winter_pr0 = winter_pr0;
  a.T = T; a.C = C; a.ldx = ldx;
  a.P = *params_host;
  a.want = fwi::want_bits(DC, DMC, FFMC, ISI, BUI, FWI, DSR);
  a.DC = DC; a.DMC = DMC; a.FFMC = FFMC; a.ISI = ISI; a.BUI = BUI; a.FWI = FWI; a.DSR = DSR;
  a.mask_out = season_mask_out;
  a.winter_pr_out = winter_pr_out;
  const char* msg = fwi::check_args(a);
  XC_REQUIRE(msg == nullptr, "%s", msg);
  XC_REQUIRE(T < (1ll << 31), "series longer than 2^31 steps");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((C + kThreads - 1) / kThreads);
  if (fwi::needs_rings(a.P)) fwi_kernel<true><<<blocks, kThreads, 0, s>>>(a);
  else fwi_kernel<false><<<blocks, kThreads, 0, s>>>(a);
  return launch_status("fwi_kernel");
}

extern "C" int32_t xc_fwi_elementwise_f32(int32_t kind, const float* a, const float* b, int64_t n, double p0, double p1,
                                          double p2, float* out, void* stream) {
  using namespace xc;
  XC_REQUIRE(kind >= XC_FWI_EW_ISI && kind <= XC_FWI_EW_OWDC, "unknown element-wise fire weather function %d", kind);
  XC_REQUIRE(a && out && (b || kind == XC_FWI_EW_DSR), "null pointer argument");
  XC_REQUIRE(n > 0, "bad shape");
  const int64_t want = (n + 255) / 256;
  const int64_t cap = (int64_t)sm_count() * 16;   // grid-stride: 16 CTAs per SM at most
  const unsigned blocks = (unsigned)(want < cap ? want : cap);
  fwi_elementwise_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(kind, a, b, n, p0, p1, p2, out);
  return launch_status("fwi_elementwise_kernel");
}
