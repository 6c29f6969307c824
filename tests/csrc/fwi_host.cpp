// TEST INFRASTRUCTURE: a HOST build of the device code of the fire-weather kernel.
//
// xclim_b200/csrc/fwi_core.cuh holds the whole per-cell day loop of xc_fwi_f32 as __host__ __device__ code;
// this file compiles it with g++ (-ffp-contract=off) behind the same argument list as the C-ABI entry point,
// with host pointers and a plain loop over the cells in place of the CUDA grid.  tests/test_fire_host_core.py
// checks it against the oracle and the reference fixtures, so that the arithmetic and the state machine of
// the kernel are verified where no GPU is available.  Nothing in xclim_b200/ loads this library.
#include <cstddef>

#include "../../xclim_b200/csrc/fwi_core.cuh"

static const double h_day_lengths[60] = XC_FWI_DAY_LENGTHS;
static const double h_day_length_factors[36] = XC_FWI_DAY_LENGTH_FACTORS;
static const char* g_msg = "";

extern "C" const char* fwi_host_last_error(void) { return g_msg; }

extern "C" int32_t fwi_host_f32(const float* tas, const float* pr, const float* hurs, const float* ws, const float* snd,
                                const uint8_t* season_mask_in, const int8_t* month, const double* lat,
                                const float* dc0, const float* dmc0, const float* ffmc0, const float* winter_pr0,
                                int64_t T, int64_t C, int64_t ldx, const XcFwiParams* params,
                                float* DC, float* DMC, float* FFMC, float* ISI, float* BUI, float* FWI, float* DSR,
                                uint8_t* season_mask_out, float* winter_pr_out) {
  using namespace xc;
  fwi::Args a{};
  a.tas = tas; a.pr = pr; a.hurs = hurs; a.ws = ws; a.snd = snd;
  a.mask_in = season_mask_in; a.month = month; a.lat = lat;
  a.dc0 = dc0; a.dmc0 = dmc0; a.ffmc0 = ffmc0; a.winter_pr0 = winter_pr0;
  a.T = T; a.C = C; a.ldx = ldx;
  a.P = *params;
  a.want = fwi::want_bits(DC, DMC, FFMC, ISI, BUI, FWI, DSR);
  a.DC = DC; a.DMC = DMC; a.FFMC = FFMC; a.ISI = ISI; a.BUI = BUI; a.FWI = FWI; a.DSR = DSR;
  a.mask_out = season_mask_out;
  a.winter_pr_out = winter_pr_out;
  const char* msg = fwi::check_args(a);
  if (msg) { g_msg = msg; return XC_ERR_INVALID; }
  for (int64_t c = 0; c < C; ++c) {
    if (fwi::needs_rings(a.P)) fwi::run_cell<true>(a, c, h_day_lengths, h_day_length_factors);
    else fwi::run_cell<false>(a, c, h_day_lengths, h_day_length_factors);
  }
  return XC_OK;
}

extern "C" int32_t fwi_host_elementwise_f32(int32_t kind, const float* a, const float* b, int64_t n, double p0, double p1,
                                            double p2, float* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = xc::fwi::elementwise(kind, a[i], b ? b[i] : 0.0f, p0, p1, p2);
  return XC_OK;
}

// test hook: numpy's float32 mean of a ring (newest value at `head`)
extern "C" float fwi_host_np_mean(const float* ring, int32_t n, int32_t head) { return xc::fwi::np_mean_f32(ring, n, head); }

// test hook: the layout of XcFwiParams that the bindings must reproduce
extern "C" void fwi_host_params_layout(int64_t* out) {
  out[0] = sizeof(XcFwiParams);
  out[1] = offsetof(XcFwiParams, snow_min_cover_frac);
  out[2] = offsetof(XcFwiParams, in_scale);
}
