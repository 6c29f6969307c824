// Host build of the evapotranspiration device code (xclim_b200/csrc/pet_core.cuh) for the CPU test-suite: the
// element loop of pet_daily_kernel and the cell loop of pet_monthly_kernel (pet.cu) over host arrays, compiled with
// g++ -ffp-contract=off, behind the argument checks of the C-ABI entry points.
#include <stddef.h>
#include <stdint.h>

#include "../../xclim_b200/csrc/pet_core.cuh"

using namespace xc::pet;

static Args make(const float* const* inputs, int64_t T, int64_t C, int64_t ldx, const double* table, int64_t L,
                 const int32_t* lat_index, const XcPetParams* P, float* out) {
  Args a{};
  for (int k = 0; k < XC_PET_N_IN; ++k) a.in[k] = inputs[k];
  a.T = T; a.C = C; a.ldx = ldx;
  a.table = table; a.L = L; a.lat_index = lat_index;
  a.P = *P;
  a.out = out;
  return a;
}

extern "C" {

// xc_pet_daily_f32 on host arrays; returns 0, or -1 where the C ABI returns XC_ERR_INVALID
int32_t pet_host_daily(const float* const* inputs, int64_t T, int64_t C, int64_t ldx, const double* table, int64_t L,
                       const int32_t* lat_index, const XcPetParams* P, float* out) {
  const Args a = make(inputs, T, C, ldx, table, L, lat_index, P, out);
  if (check_args(a, false)) return -1;
  for (int64_t t = 0; t < T; ++t)
    for (int64_t c = 0; c < C; ++c) out[t * ldx + c] = daily_value(a, t, c, a.P.method);
  return 0;
}

int32_t pet_host_monthly(const float* const* inputs, int64_t T, int64_t C, int64_t ldx, const int32_t* moff, int64_t M,
                         const int32_t* yoff, int64_t Y, const double* mdays, const double* table, int64_t L,
                         const int32_t* lat_index, const XcPetParams* P, float* out) {
  Args a = make(inputs, T, C, ldx, table, L, lat_index, P, out);
  a.moff = moff; a.M = M; a.yoff = yoff; a.Y = Y; a.mdays = mdays;
  if (check_args(a, true)) return -1;
  for (int64_t c = 0; c < C; ++c) monthly_cell(a, c);
  return 0;
}

// the layout of XcPetParams that the bindings must reproduce
void pet_host_params_layout(int64_t* out) {
  out[0] = sizeof(XcPetParams);
  out[1] = offsetof(XcPetParams, in_scale);
  out[2] = offsetof(XcPetParams, peta);
}

}  // extern "C"
