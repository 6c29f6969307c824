// Canadian Forest Fire Weather Index System: the per-cell day loop, shared by the CUDA kernel (fwi.cu) and
// by a host build of the very same code that the CPU test-suite checks against the oracle and the
// reference fixtures (tests/csrc/fwi_host.cpp -- there is no GPU where this code is written).
//
// Replaces indices/fire/_cffwis.py `_fire_weather_calc` (:680-873) and what it calls; the section
// comments cite the lines.  Arithmetic as the reference's for float32 inputs: the numba step functions
// evaluate in float64 (but np.sqrt(w) and np.log(dmc0) on their float32 arguments are float32), results are
// stored and carried as float32; ISI / BUI / FWI / DSR are float32 numpy expressions.  This file must be
// compiled WITHOUT floating-point contraction (nvcc -fmad=false, g++ -ffp-contract=off): neither numba nor
// numpy fuse a multiply with the following add.
#pragma once
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/xclim_b200.h"
#include "npsum.cuh"

#if defined(__CUDACC__)
#define XC_FWI_HD __host__ __device__ __forceinline__
#else
#define XC_FWI_HD inline
#endif

namespace xc {
namespace fwi {

// GFWED day-length tables (_cffwis.py:186-205): rows = latitude bands, columns = months.
#define XC_FWI_DAY_LENGTHS                                                  \
  {11.5, 10.5, 9.2, 7.9, 6.8, 6.2, 6.5, 7.4, 8.7, 10, 11.2, 11.8,           \
   10.1, 9.6,  9.1, 8.5, 8.1, 7.8, 7.9, 8.3, 8.9, 9.4, 9.9, 10.2,           \
   9,    9,    9,   9,   9,   9,   9,   9,   9,   9,   9,   9,              \
   7.9,  8.4,  8.9, 9.5, 9.9, 10.2, 10.1, 9.7, 9.1, 8.6, 8.1, 7.8,          \
   6.5,  7.5,  9,   12.8, 13.9, 13.9, 12.4, 10.9, 9.4, 8,  7,   6}
#define XC_FWI_DAY_LENGTH_FACTORS                                           \
  {6.4,  5.0,  2.4,  0.4,  -1.6, -1.6, -1.6, -1.6, -1.6, 0.9,  3.8,  5.8,   \
   1.39, 1.39, 1.39, 1.39, 1.39, 1.39, 1.39, 1.39, 1.39, 1.39, 1.39, 1.39,  \
   -1.6, -1.6, -1.6, 0.9,  3.8,  5.8,  6.4,  5.0,  2.4,  0.4,  -1.6, -1.6}

enum : int { W_DC = 1, W_DMC = 2, W_FFMC = 4, W_ISI = 8, W_BUI = 16, W_FWI = 32, W_DSR = 64 };
constexpr int kMaxCondDays = 32;    // temp_condition_days, snow_condition_days
constexpr int kMaxCoverDays = 128;  // snow_cover_days

// Python / numba max(a, b) and min(a, b): b only when it compares beyond a (a NaN `a` stays).
XC_FWI_HD double pmax(double a, double b) { return (b > a) ? b : a; }
XC_FWI_HD double pmin(double a, double b) { return (b < a) ? b : a; }

// Row of the day-length table (:207-224) / of the factor table (:227-242) for a latitude; -1 = invalid.
XC_FWI_HD int day_length_band(double lat) {
  if (!(lat >= -90.0 && lat <= 90.0)) return -1;
  return lat < -30.0 ? 0 : lat < -15.0 ? 1 : lat < 15.0 ? 2 : lat < 30.0 ? 3 : 4;
}
XC_FWI_HD int day_length_factor_band(double lat) {
  if (!(lat >= -90.0 && lat <= 90.0)) return -1;
  return lat < -15.0 ? 0 : lat < 15.0 ? 1 : 2;
}

// ---- the three codes over one day ---------------------------------------------------------------
// _fine_fuel_moisture_code (:246-319).  Where the reference raises (mo == ew exactly) the moisture is kept.
XC_FWI_HD double ffmc_step(float t_, float p_, float w_, float h_, float f0_) {
  if (f0_ != f0_) return (double)NAN;   // outside the season: every path below propagates the NaN (nothing to evaluate)
  const double t = t_, p = p_, h = h_, f0 = f0_;
  const double root_w = (double)sqrtf(w_);
  double mo = (147.2 * (101.0 - f0)) / (59.5 + f0);                                   // Eq. 1
  if (p > 0.5) {
    const double rf = p - 0.5;                                                        // Eq. 2
    const double gain = 42.5 * rf * exp(-100.0 / (251.0 - mo)) * (1.0 - exp(-6.93 / rf));
    if (mo > 150.0) mo = (mo + gain) + (0.0015 * ((mo - 150.0) * (mo - 150.0))) * sqrt(rf);   // Eq. 3b
    else if (mo <= 150.0) mo = mo + gain;                                             // Eq. 3a
    mo = pmin(mo, 250.0);
  }
  // Equilibrium moisture contents.  The two powers of the humidity share one logarithm (h^a = exp(a ln h)): a few
  // float64 ulp away from pow(), eight orders of magnitude below the float32 rounding of the stored code.
  const double e10 = exp((h - 100.0) / 10.0);
  const double dry = 0.18 * (21.1 - t) * (1.0 - 1.0 / exp(0.115 * h));
  const double lh = log(h);
  const double ed = 0.942 * exp(0.679 * lh) + (11.0 * e10) + dry;                     // Eq. 4
  const double ew = 0.618 * exp(0.753 * lh) + (10.0 * e10) + dry;                     // Eq. 5
  // Drying towards ed (Eqs. 6, 8) and wetting towards ew (Eqs. 7, 9) are the same expression of
  // z = h/100 resp. (100 - h)/100 and of the target: one evaluation serves both, without a divergent branch
  // (Eq. 9, ew - (ew - mo) / 10^kw, equals ew + (mo - ew) / 10^kw bit for bit).  Between ew and ed, at mo == ed
  // and where the reference raises (mo == ew) the moisture is kept; a NaN takes the drying expression, as there.
  const bool drying = !(mo < ed) && !(mo == ed);
  const bool wetting = (mo < ed) && (mo < ew);
  double m = mo;
  if (drying || wetting) {
    const double z = drying ? h / 100.0 : (100.0 - h) / 100.0;
    const double z2 = z * z, z4 = z2 * z2;
    const double kl = 0.424 * (1.0 - exp(1.7 * log(z))) + (0.0694 * root_w) * (1.0 - z4 * z4);   // Eqs. 6a, 7a
    const double kw = kl * (0.581 * exp(0.0365 * t));                                 // Eqs. 6b, 7b
    const double target = drying ? ed : ew;
    m = target + (mo - target) / exp(kw * 2.302585092994046);                         // Eqs. 8, 9 (10^kw)
  }
  double ffmc = (59.5 * (250.0 - m)) / (147.2 + m);                                   // Eq. 10
  if (ffmc > 101.0) ffmc = 101.0;
  else if (ffmc <= 0.0) ffmc = 0.0;
  return ffmc;
}

// np.log of a float32 argument inside the reference's numba code: libm's logf, within an ulp of the exact value
// and nearly always equal to the float64 log rounded once to float32 (glibc: all but about 1 argument in 2,000).
// CUDA's logf and numpy's vectorised float32 log differ from it far more often, and an ulp in Eq. 13 is magnified
// about fifty-fold where Eq. 15 cancels to a small DMC after rain, so host and device both round the float64 log.
XC_FWI_HD float log_f32(float x) { return (float)log((double)x); }

// _duff_moisture_code (:322-393); dl = day length of the cell's band for the month.
XC_FWI_HD double dmc_step(float t_, float p_, float h_, double dl, float d0_) {
  if (d0_ != d0_) return (double)NAN;
  const double t = t_, p = p_, h = h_, d0 = d0_;
  const double rk = (t < -1.1) ? 0.0 : 1.894 * (t + 1.1) * (100.0 - h) * dl * 0.0001; // Eqs. 16, 17
  double pr;
  if (p > 1.5) {
    const double rw = 0.92 * p - 1.27;                                                // Eq. 11
    const double wmi = 20.0 + 280.0 / exp(0.023 * d0);                                // Eq. 12 (cffdrs)
    double b;
    if (d0 <= 33.0) b = 100.0 / (0.5 + 0.3 * d0);                                     // Eq. 13a
    else if (d0 <= 65.0) b = 14.0 - 1.3 * (double)log_f32(d0_);                       // Eq. 13b
    else b = 6.2 * (double)log_f32(d0_) - 17.2;                                       // Eq. 13c
    const double wmr = wmi + (1000.0 * rw) / (48.77 + b * rw);                        // Eq. 14
    pr = 43.43 * (5.6348 - log(wmr - 20.0));                                          // Eq. 15 (cffdrs)
  } else {
    pr = d0;
  }
  pr = pmax(pr, 0.0);
  return pmax(pr + rk, 0.0);
}

// _drought_code (:396-446); fl = day-length factor of the cell's band for the month.
XC_FWI_HD double dc_step(float t_, float p_, double fl, float c0_) {
  if (c0_ != c0_) return (double)NAN;   // outside the season (:439-440 and c0 + pe both give NaN)
  const double p = p_, c0 = c0_;
  const double t = pmax((double)t_, -2.8);
  const double pe = pmax((0.36 * (t + 2.8) + fl) / 2, 0.0);                           // Eq. 22
  if (p > 2.8) {
    const double rw = 0.83 * p - 1.27;                                                // Eq. 18
    const double smi = 800.0 * exp(-c0 / 400.0);                                      // Eq. 19
    const double dr = c0 - 400.0 * log(1.0 + ((3.937 * rw) / smi));                   // Eqs. 20, 21
    if (dr > 0.0) return dr + pe;
    if (c0_ != c0_) return (double)NAN;
    return pe;
  }
  return c0 + pe;
}

// _overwintering_drought_code (:549-583).
XC_FWI_HD double overwintered_dc(float last_dc, float winter_pr, double a, double b, double min_dc) {
  if (last_dc != last_dc || winter_pr != winter_pr) return (double)NAN;
  const double qf = 800.0 * exp(-(double)last_dc / 400.0);
  const double qs = a * qf + b * (3.94 * (double)winter_pr);
  return pmax(400.0 * log(800.0 / qs), min_dc);
}

// ---- the derived indices, float32 arithmetic (numpy expressions of float32 arrays) ----------------
XC_FWI_HD float isi_of(float ws, float ffmc) {                                        // :449-469
  const float mo = 147.2f * (101.0f - ffmc) / (59.5f + ffmc);
  const float ff = 19.1152f * expf(mo * -0.1386f) * (1.0f + powf(mo, 5.31f) / 49300000.0f);   // Eq. 25
  return ff * expf(0.05039f * ws);                                                    // Eq. 26
}
XC_FWI_HD float bui_of(float dmc, float dc) {                                         // :472-501
  if (dmc == 0.0f && dc == 0.0f) return 0.0f;
  const float denom = dmc + 0.4f * dc;
  float bui;
  if (dmc <= 0.4f * dc) bui = (0.8f * dc * dmc) / denom;                              // Eq. 27a
  else bui = dmc - (1.0f - 0.8f * dc / denom) * (0.92f + powf(0.0114f * dmc, 1.7f));  // Eq. 27b
  return bui < 0.0f ? 0.0f : bui;                                                     // np.clip keeps NaN
}
XC_FWI_HD float fwi_of(float isi, float bui) {                                        // :504-528
  float fwi;
  if (bui <= 80.0f) fwi = 0.1f * isi * (0.626f * powf(bui, 0.809f) + 2.0f);           // Eq. 28a
  else fwi = 0.1f * isi * (1000.0f / (25.0f + 108.64f / expf(0.023f * bui)));         // Eq. 28b
  if (fwi > 1.0f) fwi = expf(2.72f * powf(0.434f * logf(fwi), 0.647f));               // Eq. 30b
  return fwi;
}
XC_FWI_HD float dsr_of(float fwi) { return 0.0272f * powf(fwi, 1.77f); }              // :531-546

// numpy's float32 mean of n <= 128 values (one leaf of numpy's pairwise summation, npsum.cuh), oldest
// value first.  ring holds the last n values, the newest at index head.
XC_FWI_HD float np_mean_f32(const float* ring, int n, int head) {
  int i0 = head + 1;
  if (i0 >= n) i0 -= n;
  auto at = [&](int k) -> float { int j = i0 + k; if (j >= n) j -= n; return ring[j]; };
  return np::pairwise_block_f32(at, n) / (float)n;
}

// ---- per-cell state -------------------------------------------------------------------------------
struct Args {
  const float *tas, *pr, *hurs, *ws, *snd;
  const uint8_t* mask_in;
  const int8_t* month;
  const double* lat;
  const float *dc0, *dmc0, *ffmc0, *winter_pr0;
  int64_t T, C, ldx;
  XcFwiParams P;
  int want;                 // W_* bits of the codes / indices to compute
  float *DC, *DMC, *FFMC, *ISI, *BUI, *FWI, *DSR;
  uint8_t* mask_out;
  float* winter_pr_out;
};

struct Rings {              // GFWED season means and the snow-cover history of the "SNOW" dry start
  float temp[kMaxCondDays], snow[kMaxCondDays], cover[kMaxCoverDays];
};
struct NoRings {};

#if defined(__CUDA_ARCH__)
#define XC_FWI_LD(ptr) ::xc::ld_stream(ptr)
#else
#define XC_FWI_LD(ptr) (*(ptr))
#endif

// One cell through all T days: the loop of _fire_weather_calc (:721-866) with the season masks of
// _fire_season (:636-675) computed on the way.  RINGS = the modes that need window means.
// day_lengths / day_length_factors: the two tables (device constant memory / host statics).
template <bool RINGS>
XC_FWI_HD void run_cell(const Args& a, int64_t c, const double* day_lengths, const double* day_length_factors) {
  const XcFwiParams& P = a.P;
  const int want = a.want;
  const bool always = P.season_mode == XC_FWI_SEASON_ALWAYS;
  const bool ow = P.overwintering != 0;
  const int dry = P.dry_start;
  const bool gfwed_dry = dry == XC_FWI_DRY_GFWED || dry == XC_FWI_DRY_GFWED_SNOW;
  const int nt = P.temp_condition_days, ns = P.snow_condition_days, nsc = P.snow_cover_days;
  const double nan_d = (double)NAN;
  const float nan_f = NAN;

  const double lat = a.lat ? a.lat[c] : 0.0;
  const int band = day_length_band(lat), fband = day_length_factor_band(lat);
  const double* dl_row = day_lengths + 12 * (band < 0 ? 0 : band);
  const double* fl_row = day_length_factors + 12 * (fband < 0 ? 0 : fband);
  const bool bad_lat = band < 0;   // the reference raises ValueError("Invalid lat specified."): NaN codes here

  // previous codes (:683-693, 709-718)
  const float dc_in = a.dc0 ? a.dc0[c] : nan_f, dmc_in = a.dmc0 ? a.dmc0[c] : nan_f;
  float dc = dc_in, dmc = dmc_in, ffmc = a.ffmc0 ? a.ffmc0[c] : nan_f;
  if (always) {
    if (dc != dc) dc = P.dc_start;
    if (dmc != dmc) dmc = P.dmc_start;
    if (ffmc != ffmc) ffmc = P.ffmc_start;
  }
  float saved_dc = dc_in, saved_dmc = dmc_in;      // ow_DC / ow_DMC
  float winter_pr = a.winter_pr0 ? a.winter_pr0[c] : 0.0f;
  if (ow && (want & W_DC)) dc = nan_f;
  if (dry) {
    if (!ow && saved_dc != saved_dc) saved_dc = P.dc_start;
    if (saved_dmc != saved_dmc) saved_dmc = P.dmc_start;
  }
  bool wet_start = false;
  int on_prev = 0;                                 // season_mask[it - 1]
  int hot_run = 0, cold_run = 0, snowfree_run = 0;
  typename std::conditional<RINGS, Rings, NoRings>::type rings;
  (void)rings;

  const int64_t ldx = a.ldx;
  for (int64_t it = 0; it < a.T; ++it) {
    const int64_t off = it * ldx + c;
    // load + unit conversion (cffwis_indices :1369-1374: one float32 operation per array)
    const float tas = a.tas ? XC_FWI_LD(a.tas + off) * P.in_scale[0] + P.in_offset[0] : nan_f;
    const float pr = a.pr ? XC_FWI_LD(a.pr + off) * P.in_scale[1] + P.in_offset[1] : nan_f;
    const float hurs = a.hurs ? XC_FWI_LD(a.hurs + off) * P.in_scale[2] + P.in_offset[2] : nan_f;
    const float ws = a.ws ? XC_FWI_LD(a.ws + off) * P.in_scale[3] + P.in_offset[3] : nan_f;
    const float snd = a.snd ? XC_FWI_LD(a.snd + off) * P.in_scale[4] + P.in_offset[4] : nan_f;
    int mth = a.month[it];
    mth = mth < 1 ? 1 : (mth > 12 ? 12 : mth);     // the tables have twelve columns

    // ---- season mask of the day (:636-675) ----
    int on = 1;
    if (P.season_mode == XC_FWI_SEASON_MASK) {
      on = a.mask_in[off] != 0;
    } else if (P.season_mode == XC_FWI_SEASON_WF93) {       // the nt days BEFORE today
      on = 0;
      if (it >= nt + 1) on = (on_prev | (hot_run >= nt)) & !(cold_run >= nt);
      hot_run = (tas > P.temp_start_thresh) ? hot_run + 1 : 0;
      cold_run = (tas < P.temp_end_thresh) ? cold_run + 1 : 0;
    } else if (P.season_mode == XC_FWI_SEASON_LA08) {       // windows that END today
      snowfree_run = (snd <= P.snow_thresh) ? snowfree_run + 1 : 0;
      cold_run = (tas < P.temp_end_thresh) ? cold_run + 1 : 0;
      on = 0;
      if (it >= (nt > ns ? nt : ns))
        on = (on_prev | (snowfree_run >= ns)) & !((snd > P.snow_thresh) | (cold_run >= nt));
    }
    if constexpr (RINGS) {
      if (P.season_mode == XC_FWI_SEASON_GFWED) {           // window means
        const int ht = (int)(it % nt), hs = (int)(it % ns);
        rings.temp[ht] = tas;
        rings.snow[hs] = snd;
        on = 0;
        if (it >= (nt > ns ? nt : ns)) {
          const float msnow = np_mean_f32(rings.snow, ns, hs), mtemp = np_mean_f32(rings.temp, nt, ht);
          const int up = (mtemp > P.temp_start_thresh) & (msnow < P.snow_thresh);
          const int down = (msnow >= P.snow_thresh) | (mtemp < P.temp_end_thresh);
          on = (on_prev | up) & !down;
        }
      }
      if (dry == XC_FWI_DRY_GFWED_SNOW) rings.cover[(int)(it % nsc)] = snd;
    }
    if (a.mask_out) a.mask_out[off] = (uint8_t)on;

    // ---- start-ups and shut-downs (:722-836) ----
    if (!always) {
      const int delta = (it == 0) ? (P.initial_start_up ? on : 0) : on - on_prev;
      const bool closing = delta == -1, opening = delta == 1, idle = (delta == 0) && (on == 0);
      bool rainy = false;
      if (dry) {
        rainy = pr > P.prec_thresh;
        if constexpr (RINGS) {
          if (dry == XC_FWI_DRY_GFWED_SNOW && it >= nsc) {   // (:746-756)
            wet_start = false;
            if (opening) {
              int covered = 0;
              for (int k = 0; k < nsc; ++k) covered += rings.cover[k] > P.snow_thresh;
              wet_start = ((double)covered / (double)nsc >= P.snow_min_cover_frac) &&
                          (np_mean_f32(rings.cover, nsc, (int)(it % nsc)) >= P.snow_min_mean_depth);
            }
          }
        }
      }
      if (want & W_DC) {
        if (ow) {                                            // (:759-784)
          if (closing) { saved_dc = dc; winter_pr = pr; }
          if (idle) winter_pr = winter_pr + pr;
          if (opening) {
            dc = (saved_dc != saved_dc)
                     ? P.dc_start
                     : (float)overwintered_dc(saved_dc, winter_pr, P.carry_over_fraction,
                                              P.wetting_efficiency_fraction, P.min_dc);
            saved_dc = nan_f;
            winter_pr = nan_f;
          }
        } else if (dry) {                                    // (:785-806)
          if (closing) saved_dc = P.dc_start;
          if (gfwed_dry) {
            if ((opening || idle) && rainy) saved_dc = 0.0f;
            if ((opening || idle) && !rainy) saved_dc = saved_dc + P.dc_dry_factor;
          } else {
            if (idle && rainy) saved_dc = P.dc_start;
            if (idle && !rainy) saved_dc = saved_dc + P.dc_dry_factor;
          }
          if (dry == XC_FWI_DRY_GFWED_SNOW && wet_start) saved_dc = P.dc_start;
          if (opening) { dc = saved_dc; saved_dc = nan_f; }
        } else if (opening) {
          dc = P.dc_start;                                   // (:807-808)
        }
        if (closing) dc = nan_f;
      }
      if (want & W_DMC) {                                    // (:811-832)
        if (dry) {
          if (closing) saved_dmc = P.dmc_start;
          if (gfwed_dry) {
            if ((opening || idle) && rainy) saved_dmc = 0.0f;
            if ((opening || idle) && !rainy) saved_dmc = saved_dmc + P.dmc_dry_factor;
          } else {
            if (idle && rainy) saved_dmc = P.dmc_start;
            if (idle && !rainy) saved_dmc = saved_dmc + P.dmc_dry_factor;
          }
          if (dry == XC_FWI_DRY_GFWED_SNOW && wet_start) saved_dmc = P.dmc_start;
          if (opening) { dmc = saved_dmc; saved_dmc = nan_f; }
        } else if (opening) {
          dmc = P.dmc_start;
        }
        if (closing) dmc = nan_f;
      }
      if (want & W_FFMC) {                                   // (:834-836)
        if (opening) ffmc = P.ffmc_start;
        if (closing) ffmc = nan_f;
      }
    }

    // ---- the codes and indices of the day (:839-866) ----
    float isi = nan_f, bui = nan_f, fwi = nan_f;
    if (want & W_DC) {
      dc = bad_lat ? nan_f : (float)dc_step(tas, pr, fl_row[mth - 1], dc);
      if (a.DC) a.DC[off] = dc;
    }
    if (want & W_DMC) {
      dmc = bad_lat ? nan_f : (float)dmc_step(tas, pr, hurs, dl_row[mth - 1], dmc);
      if (a.DMC) a.DMC[off] = dmc;
    }
    if (want & W_FFMC) {
      ffmc = (float)ffmc_step(tas, pr, ws, hurs, ffmc);
      if (a.FFMC) a.FFMC[off] = ffmc;
    }
    if (want & W_ISI) {
      isi = isi_of(ws, ffmc);
      if (a.ISI) a.ISI[off] = isi;
    }
    if (want & W_BUI) {
      bui = bui_of(dmc, dc);
      if (a.BUI) a.BUI[off] = bui;
    }
    if (want & W_FWI) {
      fwi = fwi_of(isi, bui);
      if (a.FWI) a.FWI[off] = fwi;
    }
    if ((want & W_DSR) && a.DSR) a.DSR[off] = dsr_of(fwi);
    on_prev = on;
  }
  if (a.winter_pr_out) a.winter_pr_out[c] = winter_pr;
  (void)nan_d;
}

// One element of the element-wise entry point (xc_fwi_elementwise_f32).
XC_FWI_HD float elementwise(int kind, float a, float b, double p0, double p1, double p2) {
  switch (kind) {
    case XC_FWI_EW_ISI: return isi_of(a, b);
    case XC_FWI_EW_BUI: return bui_of(a, b);
    case XC_FWI_EW_FWI: return fwi_of(a, b);
    case XC_FWI_EW_DSR: return dsr_of(a);
    default: return (float)overwintered_dc(a, b, p0, p1, p2);
  }
}

// The W_* bits implied by the outputs asked for (:1046-1057).
inline int want_bits(bool DC, bool DMC, bool FFMC, bool ISI, bool BUI, bool FWI, bool DSR) {
  int w = (DC ? W_DC : 0) | (DMC ? W_DMC : 0) | (FFMC ? W_FFMC : 0) | (ISI ? W_ISI : 0) | (BUI ? W_BUI : 0) |
          (FWI ? W_FWI : 0) | (DSR ? W_DSR : 0);
  if (w & W_DSR) w |= W_FWI;
  if (w & W_FWI) w |= W_ISI | W_BUI;
  if (w & W_BUI) w |= W_DC | W_DMC;
  if (w & W_ISI) w |= W_FFMC;
  return w;
}

// Argument checks shared by the library and the host build; returns NULL or a message.
inline const char* check_args(const Args& a) {
  const XcFwiParams& P = a.P;
  if (a.T < 1 || a.C < 1 || a.ldx < a.C) return "bad dimensions";
  if (!a.month) return "month is required";
  if (a.want == 0 && !a.mask_out) return "no output requested";
  if ((a.want & (W_DC | W_DMC | W_FFMC)) && (!a.tas || !a.pr)) return "tas and pr are required";
  if ((a.want & (W_DMC | W_FFMC)) && !a.hurs) return "hurs is required for DMC and FFMC";
  if ((a.want & W_FFMC) && !a.ws) return "ws (sfcWind) is required for FFMC";
  if ((a.want & (W_DC | W_DMC)) && !a.lat) return "lat is required for DC and DMC";
  if (P.season_mode < XC_FWI_SEASON_ALWAYS || P.season_mode > XC_FWI_SEASON_GFWED) return "unknown season_mode";
  if (P.dry_start < XC_FWI_DRY_NONE || P.dry_start > XC_FWI_DRY_GFWED_SNOW) return "unknown dry_start";
  if (P.season_mode == XC_FWI_SEASON_MASK && !a.mask_in) return "season_mask is required";
  if (P.season_mode >= XC_FWI_SEASON_WF93 && !a.tas) return "tas is required for the season mask";
  if ((P.season_mode == XC_FWI_SEASON_LA08 || P.season_mode == XC_FWI_SEASON_GFWED) && !a.snd)
    return "snd is required for the LA08 and GFWED seasons";
  if (P.dry_start == XC_FWI_DRY_GFWED_SNOW && !a.snd) return "snd is required for the snow-aware dry start";
  if (P.overwintering && P.season_mode == XC_FWI_SEASON_ALWAYS)
    return "If overwintering is activated, either `season_method` or `season_mask` must be given.";
  if (P.temp_condition_days < 1 || P.temp_condition_days > kMaxCondDays || P.snow_condition_days < 1 ||
      P.snow_condition_days > kMaxCondDays)
    return "temp_condition_days and snow_condition_days must lie in 1..32";
  if (P.snow_cover_days < 1 || P.snow_cover_days > kMaxCoverDays) return "snow_cover_days must lie in 1..128";
  return nullptr;
}

inline bool needs_rings(const XcFwiParams& P) {
  return P.season_mode == XC_FWI_SEASON_GFWED || P.dry_start == XC_FWI_DRY_GFWED_SNOW;
}

}  // namespace fwi
}  // namespace xc
