// Chill portions (Dynamic Model) and chill units (Utah Model) of one (cell, period), and the hourly temperature
// profile they run on: the code shared by the CUDA kernels (chill.cu) and by a host build of the very same code that
// the CPU test-suite checks against the oracle (tests/csrc/chill_host.cpp).
//
// Hourly temperature -- `make_hourly_temperature` (indices/helpers.py:1059-1123, Linvill 1990), sunrise at 00:00:
//   day   (h < dl)  (tasmax - tasmin) * sin(pi*h / (dl + 4)) + tasmin
//   night           sunset - ((sunset - tasmin[d+1]) / log(24 - (dl - 1))) * log(clip(h + 1 - dl, 1))
//   sunset          (tasmax - tasmin) * sin(pi*dl / (dl + 4)) + tasmin
// with tasmin[T] = tasmin[T-1].  Every transcendental depends on (day, latitude) only: the host tabulates them in
// float64 with numpy (converters.hourly_weights) as one row of XC_CHILL_ROW doubles per (day, latitude):
//   [0, 24)  the day sine or the night log of each hour,  [24] sin(pi*dl/(dl+4)),  [25] log(24 - (dl - 1)),  [26] dl.
// The difference tasmax - tasmin is taken in the input's float32, as numpy does before promoting to float64; the
// rest is the reference's float64 multiply / add / divide in its order (built with -fmad=false / -ffp-contract=off),
// so the hours are bit-identical to the reference's.  A NaN day length (polar day or night without infill) gives
// 24 NaN hours.
//
// Dynamic Model -- `_chill_portion_one_season` (indices/_agro.py:1436-1465) on the selected hours in K:
//   xi = sr / (1 + sr), sr = exp(SLP*TETMLT*(T - TETMLT)/T);  xs = AA*exp(EE/T);  ak1 = A1*exp(-E1/T)
//   E = 0 at the period's first selected hour, then S = E < 1 ? E : E - E*xi_prev, E = xs - (xs - S)*exp(-ak1);
//   each hour adds E >= 1 ? E*xi : 0.  A NaN hour makes E NaN, and adds nothing, for the rest of the period.
// Utah Model -- `chill_units` (:1537-1592) on the selected hours in degC: the piecewise weights, NaN hours left out;
// with positive_only, each day's sum counts only where it is > 0.  Both sums are float64 in time order.
// Unselected days (the uint8 day mask) are skipped: `select_time(drop=True)` for the portions (the recurrence goes on
// over the gap), NaN for the units (the indicator's indexer).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/xclim_b200.h"

#if defined(__CUDACC__)
#define XC_CH_HD __host__ __device__ __forceinline__
#else
#define XC_CH_HD inline
#endif

namespace xc {
namespace chill {

// the reference's constants (Luedeling et al. 2009), as Python evaluates them
constexpr double E0 = 4153.5, E1 = 12888.8, A0 = 139500.0, A1 = 2.567e18, SLP = 1.6, TETMLT = 277.0;
constexpr double AA = A0 / A1, EE = E1 - E0, SLP_TETMLT = SLP * TETMLT;

struct Args {
  const float* tasmin;       // daily (T, C) at [t * ldx + c]   (fused and generation kernels)
  const float* tasmax;
  const void* hourly;        // hourly (H, C) at [t * ldx + c], float32 or float64 (hourly-input kernel)
  int32_t hourly_f64;
  int64_t T, C, ldx, H;      // T days; H hours (H <= 24 * T; the last day may be partial)
  const double* weights;     // (T, L, XC_CHILL_ROW)
  int32_t L;
  const int32_t* lat_index;  // (C) row of each cell in the weights
  const int32_t* poff;       // (P + 1) day offsets of the periods
  int32_t P;
  const uint8_t* day_mask;   // (T) nonzero = selected; null = every day
  double k_scale, k_offset;  // hourly value -> K   (portions)
  double c_scale, c_offset;  // hourly value -> degC (units)
  int32_t what;              // XC_CHILL_PORTIONS | XC_CHILL_UNITS | XC_CHILL_POSITIVE_ONLY
  double* out_cp;            // (P, C)
  double* out_cu;            // (P, C)
  int32_t* out_valid;        // (P, C) selected non-NaN hours, or null
  double* out_hourly;        // (24 T, C) at [h * C + c] (generation kernel)
};

// XC_OK, or the status of the C ABI with its message in *msg.  `kind`: 0 fused, 1 hourly input, 2 generation.
inline int32_t check_args(const Args& a, int kind, const char** msg) {
  *msg = nullptr;
  const bool daily = kind != 1;
  if ((daily && (!a.tasmin || !a.tasmax || !a.weights || !a.lat_index)) || (!daily && !a.hourly))
    *msg = "null pointer argument";
  else if (kind == 2 && !a.out_hourly) *msg = "null pointer argument";
  else if (kind != 2 && (!a.poff || ((a.what & XC_CHILL_PORTIONS) && !a.out_cp) ||
                         ((a.what & XC_CHILL_UNITS) && !a.out_cu)))
    *msg = "null pointer argument";
  else if (!(a.T > 0 && a.C > 0 && a.ldx >= a.C && a.T < 2147483647LL / 24)) *msg = "bad shape";
  else if (daily && a.L <= 0) *msg = "bad shape";
  else if (!daily && !(a.H > 24 * (a.T - 1) && a.H <= 24 * a.T)) *msg = "bad shape";
  else if (kind != 2 && !(a.P > 0 && a.P <= 65535)) *msg = "bad shape";
  else if (kind != 2 && (a.what & ~(XC_CHILL_PORTIONS | XC_CHILL_UNITS | XC_CHILL_POSITIVE_ONLY) ||
                         !(a.what & (XC_CHILL_PORTIONS | XC_CHILL_UNITS))))
    *msg = "bad output selection";
  return *msg ? XC_ERR_INVALID : XC_OK;
}

template <class V>
XC_CH_HD V load(const V* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// the 24 hours of day d at one cell, from the daily inputs and the day's weight row
struct DailyProfile {
  double tmin, tmax_d, diff, sunset, next, dl;
  const double* w;

  XC_CH_HD void begin(const Args& a, int64_t c, int d) {
    const float tn = load(a.tasmin + (int64_t)d * a.ldx + c);
    const float tx = load(a.tasmax + (int64_t)d * a.ldx + c);
    const float tn1 = d + 1 < a.T ? load(a.tasmin + (int64_t)(d + 1) * a.ldx + c) : tn;
    w = a.weights + ((int64_t)d * a.L + load(a.lat_index + c)) * XC_CHILL_ROW;
    tmin = (double)tn;
    diff = (double)(tx - tn);                       // numpy: float32 - float32, then promoted
    sunset = diff * load(w + 24) + tmin;
    next = (double)tn1;
    dl = load(w + 26);
  }
  XC_CH_HD double hour(int h) const {
    const double wh = load(w + h);
    if ((double)h < dl) return diff * wh + tmin;
    return sunset - ((sunset - next) / load(w + 25)) * wh;
  }
};

struct Dynamic {
  double E = 0.0, xi_prev = 0.0, sum = 0.0;
  bool started = false;

  // one hour in K; returns E (for the host trace)
  XC_CH_HD double step(double tk) {
    const double ftmprt = SLP_TETMLT * (tk - TETMLT) / tk;
    const double sr = exp(ftmprt);
    const double xi = sr / (1.0 + sr);
    const double xs = AA * exp(EE / tk);
    const double ak1 = A1 * exp(-E1 / tk);
    if (started) {
      const double S = E < 1.0 ? E : E - E * xi_prev;
      E = xs - (xs - S) * exp(-ak1);
    } else {
      E = 0.0;
      started = true;
    }
    sum += E >= 1.0 ? E * xi : 0.0;
    xi_prev = xi;
    return E;
  }
};

// the Utah weight of one hour in degC (not NaN)
XC_CH_HD double utah(double t) {
  if (t <= 1.4 || (t > 12.4 && t <= 15.9)) return 0.0;
  if ((t > 1.4 && t <= 2.4) || (t > 9.1 && t <= 12.4)) return 0.5;
  if (t > 2.4 && t <= 9.1) return 1.0;
  if (t > 15.9 && t <= 17.9) return -0.5;
  return -1.0;
}

// hour value of the hourly-input kernel
XC_CH_HD double hourly_value(const Args& a, int64_t c, int64_t t) {
  const int64_t i = t * a.ldx + c;
  return a.hourly_f64 ? load((const double*)a.hourly + i) : (double)load((const float*)a.hourly + i);
}

// one (cell, period): FUSED = the hours come from the daily inputs, else from the hourly input
template <bool FUSED>
XC_CH_HD void run(const Args& a, int64_t c, int p) {
  const int d0 = a.poff[p], d1 = a.poff[p + 1];
  const bool want_cp = a.what & XC_CHILL_PORTIONS, want_cu = a.what & XC_CHILL_UNITS;
  const bool positive_only = a.what & XC_CHILL_POSITIVE_ONLY;
  Dynamic dyn;
  double cu = 0.0;
  int32_t valid = 0;
  for (int d = d0; d < d1; ++d) {
    if (a.day_mask && !load(a.day_mask + d)) continue;
    DailyProfile prof;
    int nh = 24;
    if (FUSED) prof.begin(a, c, d);
    else if ((int64_t)d * 24 + 24 > a.H) nh = (int)(a.H - (int64_t)d * 24);
    double daily = 0.0;
    for (int h = 0; h < nh; ++h) {
      const double v = FUSED ? prof.hour(h) : hourly_value(a, c, (int64_t)d * 24 + h);
      valid += !isnan(v);
      if (want_cp) dyn.step(v * a.k_scale + a.k_offset);
      if (want_cu) {
        const double t = v * a.c_scale + a.c_offset;
        if (!isnan(t)) daily += utah(t);
      }
    }
    if (want_cu) cu += (!positive_only || daily > 0.0) ? daily : 0.0;
  }
  const int64_t o = (int64_t)p * a.C + c;
  if (want_cp) a.out_cp[o] = dyn.sum;
  if (want_cu) a.out_cu[o] = cu;
  if (a.out_valid) a.out_valid[o] = valid;
}

// the hourly series of one cell (generation kernel)
XC_CH_HD void generate(const Args& a, int64_t c) {
  for (int d = 0; d < a.T; ++d) {
    DailyProfile prof;
    prof.begin(a, c, d);
    for (int h = 0; h < 24; ++h) a.out_hourly[((int64_t)d * 24 + h) * a.C + c] = prof.hour(h);
  }
}

}  // namespace chill
}  // namespace xc
