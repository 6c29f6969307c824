// Potential evapotranspiration and the water budget: the per-element (daily methods) and per-cell (monthly
// methods) arithmetic, shared by the CUDA kernels (pet.cu) and by a host build of the very same code that the
// CPU test-suite checks against the oracle (tests/csrc/pet_host.cpp).
//
// Replaces `potential_evapotranspiration` (indices/converters.py:1890-2152) and the difference of
// `water_budget` (:2652-2739).  The solar terms are not computed here: the host tabulates them per (row,
// distinct latitude) in float64 (include/xclim_b200.h, p1), so the element loop needs no float64 sin, cos, tan
// or acos.  Inputs are float32 with their unit conversion applied in float32 (x * scale + offset); the
// formulas run in float64 and the result is rounded once to float32 (DESIGN.md section 4).  Compile WITHOUT
// floating-point contraction (nvcc -fmad=false, g++ -ffp-contract=off) so that both builds round the same way.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/xclim_b200.h"

#if defined(__CUDACC__)
#define XC_PET_HD __host__ __device__ __forceinline__
#else
#define XC_PET_HD inline
#endif

namespace xc {
namespace pet {

constexpr double kSecondsPerDay = 86400.0;
constexpr int kMaxMonthsPerYear = 12;

struct Args {
  const float* in[XC_PET_N_IN];
  int64_t T, C, ldx;
  const double* table;       // (rows, L)
  int64_t L;
  const int32_t* lat_index;  // (C)
  const int32_t* moff;       // monthly: (M + 1) row offsets
  int64_t M;
  const int32_t* yoff;       // monthly: (Y + 1) month offsets of the YS groups
  int64_t Y;
  const double* mdays;       // monthly: (M) days of each complete month
  XcPetParams P;
  float* out;
};

// x * scale + offset in float32: the reference converts each input array in its own dtype
XC_PET_HD float conv(float x, const XcPetParams& P, int slot) {
  const float y = x * P.in_scale[slot];
  return y + P.in_offset[slot];
}

// ndarray.clip(0): NaN stays NaN
XC_PET_HD double clip0(double v) { return v < 0.0 ? 0.0 : v; }

// saturation vapour pressure over water [Pa] of a temperature in K, sonntag90 (converters.py:415-422)
XC_PET_HD double esat_sonntag90(double tk) {
  return 100.0 * exp(-6096.9385 / tk + 16.635794 + -2.711193e-2 * tk + 1.673952e-5 * (tk * tk) + 2.433502 * log(tk));
}

// PET [mm/day] of one day of a daily method.  v: the converted inputs (slots XC_PET_IN_*), rad: the table value,
// has_tas: whether tas was given (HG85, MB05) rather than taken as (tasmin + tasmax) / 2.
XC_PET_HD double daily_pet(int method, const XcPetParams& P, const float* v, double rad, bool has_tas) {
  switch (method) {
    case XC_PET_BR65: {   // :2000-2009, temperatures in degF, rad in cal cm-2 d-1
      const double tn = v[XC_PET_IN_TASMIN], tx = v[XC_PET_IN_TASMAX];
      return clip0(0.094 * (-87.03 + 0.928 * tx + 0.933 * (tx - tn) + 0.0486 * rad));
    }
    case XC_PET_HG85: {   // :2011-2027, rad = 0.408 * ra [MJ m-2 d-1]; sqrt of a negative range is NaN
      const double tn = v[XC_PET_IN_TASMIN], tx = v[XC_PET_IN_TASMAX];
      const double tas = has_tas ? (double)v[XC_PET_IN_TAS] : (tn + tx) / 2.0;
      return clip0(0.0023 * rad * (tas + 17.8) * sqrt(tx - tn));
    }
    case XC_PET_MB05: {   // :2060-2080, rad in J m-2 d-1 with a 1367 W m-2 solar constant
      const double tas = has_tas ? (double)v[XC_PET_IN_TAS]
                                 : ((double)v[XC_PET_IN_TASMIN] + (double)v[XC_PET_IN_TASMAX]) / 2.0;
      const double tk = tas + 273.15;
      const double latent = 4185.5 * (751.78 - 0.5655 * tk);
      const double r = rad / latent;
      return r * P.peta * tas + r * P.petb;
    }
    case XC_PET_ALLEN98: {   // :2116-2144 and fao_allen98 (:1825-1874)
      const double tx = v[XC_PET_IN_TASMAX], tn = v[XC_PET_IN_TASMIN];
      const double u2 = (double)v[XC_PET_IN_WIND] * P.wind_num / P.wind_den;
      const double tm = (tx + tn) / 2.0;
      const double es = 0.5 * (esat_sonntag90(tx + 273.15) + esat_sonntag90(tn + 273.15)) / 1000.0;   // kPa
      const double ea = es * (double)v[XC_PET_IN_HURS];
      const double d = tm + 237.3;
      const double delta = 4098.0 * es / (d * d);
      const double rn = ((double)v[XC_PET_IN_RSDS] - (double)v[XC_PET_IN_RSUS] -
                         ((double)v[XC_PET_IN_RLUS] - (double)v[XC_PET_IN_RLDS])) * 0.0864;   // MJ m-2 d-1
      const double gamma = 0.665e-03 * 101.325;
      const double a1 = 0.408 * delta * (rn - 0.0);
      const double a2 = gamma * 900.0 / (tm + 273.15) * u2 * (es - ea);
      const double a3 = delta + gamma * (1.0 + 0.34 * u2);
      return (a1 + a2) / a3;
    }
    default:
      return NAN;
  }
}

// out[t, c] of a daily method: PET as a rate, or the water budget pr - PET, rounded once.  `method` is a.P.method;
// the kernel passes it as a compile-time constant so that each method's code is compiled alone.
XC_PET_HD float daily_value(const Args& a, int64_t t, int64_t c, int method) {
  float v[XC_PET_N_IN];
  const int64_t i = t * a.ldx + c;
#pragma unroll
  for (int k = 0; k < XC_PET_N_IN; ++k) v[k] = a.in[k] ? conv(a.in[k][i], a.P, k) : 0.0f;
  if (method == XC_PET_GIVEN) return (float)((double)v[XC_PET_IN_PR] - (double)v[XC_PET_IN_EVSPSBLPOT]);
  const double rad = method != XC_PET_ALLEN98 ? a.table[t * a.L + a.lat_index[c]] : 0.0;
  // amount2rate over one day (mm -> mm/d), then mm/d -> kg m-2 s-1
  const double rate = daily_pet(method, a.P, v, rad, a.in[XC_PET_IN_TAS] != nullptr) / 1.0 / kSecondsPerDay;
  return (float)(a.P.water_budget ? (double)v[XC_PET_IN_PR] - rate : rate);
}

// ---- monthly methods ----------------------------------------------------------------------------------
struct Mean {
  double s = 0.0;
  int n = 0;
  XC_PET_HD void add(double x) {
    if (x == x) { s += x; ++n; }
  }
  XC_PET_HD double get() const { return n ? s / n : (double)NAN; }
};

// DA02 PET [mm/month] of one month from its means (:2029-2058); ra = 0.408 * the month's radiation sum
XC_PET_HD double da02_pet(double tn, double tx, double tas, double pr, double ra) {
  double tr = tx - tn;
  tr = tr > 0.0 ? tr : 0.0;              // tr.where(tr > 0, 0): NaN gives 0
  const double ab = tr - 0.0123 * pr;
  const double p = pow(ab, 0.76);
  const double pet = 0.0013 * ra * (tas + 17.0) * p;
  return clip0(p != p ? 0.0 : pet);
}

// TW48: the heat-index exponent (:2105) and PET [mm/month] (:2107-2114) of a month mean tas (clipped at 0)
XC_PET_HD double tw48_pet(double tas, double heat, double dl) {
  const double a = 6.75e-7 * pow(heat, 3.0) - 7.71e-5 * pow(heat, 2.0) + 0.01791 * heat + 0.49239;
  const double frac = pow(10.0 * tas / heat, a);
  return 10.0 * (1.6 * dl * frac);
}

XC_PET_HD float month_value(const Args& a, int64_t m, double pet_mm, double pr_mean) {
  const double rate = pet_mm / a.mdays[m] / kSecondsPerDay;
  return (float)(a.P.water_budget ? pr_mean - rate : rate);
}

// One cell of a monthly method: walks the daily series once, year (YS group) by year.
XC_PET_HD void monthly_cell(const Args& a, int64_t c) {
  const int li = a.lat_index[c];
  const bool has_tas = a.in[XC_PET_IN_TAS] != nullptr;
  for (int64_t y = 0; y < a.Y; ++y) {
    const int64_t m0 = a.yoff[y], m1 = a.yoff[y + 1];
    if (m1 - m0 > kMaxMonthsPerYear) {   // not a calendar year: the group is NaN rather than overrun tas_m / pr_m
      for (int64_t m = m0; m < m1; ++m) a.out[m * a.C + c] = NAN;
      continue;
    }
    double tas_m[kMaxMonthsPerYear], pr_m[kMaxMonthsPerYear];
    double heat = 0.0;
    for (int64_t m = m0; m < m1; ++m) {
      Mean tn, tx, tas, pr;
      for (int64_t t = a.moff[m]; t < a.moff[m + 1]; ++t) {
        const int64_t i = t * a.ldx + c;
        const double vn = a.in[XC_PET_IN_TASMIN] ? conv(a.in[XC_PET_IN_TASMIN][i], a.P, XC_PET_IN_TASMIN) : NAN;
        const double vx = a.in[XC_PET_IN_TASMAX] ? conv(a.in[XC_PET_IN_TASMAX][i], a.P, XC_PET_IN_TASMAX) : NAN;
        double vt = has_tas ? (double)conv(a.in[XC_PET_IN_TAS][i], a.P, XC_PET_IN_TAS) : (vn + vx) / 2.0;
        if (a.P.method == XC_PET_TW48) vt = clip0(vt);
        tas.add(vt);
        if (a.P.method == XC_PET_DA02) { tn.add(vn); tx.add(vx); }
        if (a.in[XC_PET_IN_PR]) pr.add(conv(a.in[XC_PET_IN_PR][i], a.P, XC_PET_IN_PR));
      }
      const double rad = a.table[m * a.L + li];
      if (a.P.method == XC_PET_DA02) {
        a.out[m * a.C + c] = month_value(a, m, da02_pet(tn.get(), tx.get(), tas.get(), pr.get(), rad), 0.0);
      } else {
        tas_m[m - m0] = tas.get();
        pr_m[m - m0] = pr.get();
        const double id = pow(tas_m[m - m0] / 5.0, 1.514);
        if (id == id) heat += id;        // resample(time="YS").sum(): skipna
      }
    }
    if (a.P.method != XC_PET_TW48) continue;
    for (int64_t m = m0; m < m1; ++m)
      a.out[m * a.C + c] = month_value(a, m, tw48_pet(tas_m[m - m0], heat, a.table[m * a.L + li]), pr_m[m - m0]);
  }
}

// nullptr if the arguments are consistent, otherwise the reason
inline const char* check_args(const Args& a, bool monthly) {
  const int m = a.P.method;
  if (monthly ? (m != XC_PET_TW48 && m != XC_PET_DA02) : (m < XC_PET_BR65 || m > XC_PET_GIVEN || m == XC_PET_TW48
                                                            || m == XC_PET_DA02))
    return "unknown potential evapotranspiration method";
  if (a.T < 1 || a.C < 1 || a.ldx < a.C) return "bad shape";
  if (a.out == nullptr) return "null pointer argument";
  auto need = [&](int k) { return a.in[k] != nullptr; };
  const bool pair = need(XC_PET_IN_TASMIN) && need(XC_PET_IN_TASMAX);
  bool ok = true;
  switch (m) {
    case XC_PET_BR65: case XC_PET_HG85: ok = pair; break;
    case XC_PET_MB05: case XC_PET_TW48: ok = need(XC_PET_IN_TAS) || pair; break;
    case XC_PET_ALLEN98:
      for (int k = XC_PET_IN_TASMIN; k <= XC_PET_IN_WIND; ++k) ok = ok && (k == XC_PET_IN_TAS || need(k));
      break;
    case XC_PET_DA02: ok = pair && need(XC_PET_IN_PR); break;
    case XC_PET_GIVEN: ok = need(XC_PET_IN_EVSPSBLPOT) && a.P.water_budget; break;
  }
  if (!ok) return "a required input is missing";
  if (a.P.water_budget && (!need(XC_PET_IN_PR) || m == XC_PET_DA02)) return "the water budget needs pr (not DA02)";
  if (m != XC_PET_ALLEN98 && m != XC_PET_GIVEN && (a.table == nullptr || a.lat_index == nullptr || a.L < 1))
    return "the method needs the solar table";
  // yoff groups calendar years (the host builds it so); a group of more than kMaxMonthsPerYear months gives NaN
  if (monthly && (a.moff == nullptr || a.yoff == nullptr || a.mdays == nullptr || a.M < 1 || a.Y < 1))
    return "bad month offsets";
  return nullptr;
}

}  // namespace pet
}  // namespace xc
