// Rain season (onset, cessation) of one (cell, period): the scan shared by the CUDA kernel (rain_season.cu) and by a
// host build of the very same code that the CPU test-suite checks against the oracle (tests/csrc/rain_season_host.cpp).
//
// Replaces `rain_season` (indices/_agro.py:790-980), which runs per period of `freq`:
//   x     daily amounts (rate2amount, one float32 multiply by `scale` on load);
//   x_s   x inside the onset prefilter (the mask's XC_RS_PRE bit: date_min_start .. the period's last day), NaN outside;
//   wet   float32(sum x_s[p-ww+1 .. p]) >= thr_wet                                   (false if the window leaves the period);
//   stop  per_day: x_s <= thr_dry_start on all of p .. p+wd-1; total: float32(sum x_s[p .. p+wd-1]) <= thr_dry_start;
//   event runs_with_holes(wet, 1, stop, ...) (run_length.py:844-888): 0 if stop, else 1 if wet, else the previous event;
//   start the first position of S_start that begins an event run at least window_not_dry_start + window_wet_start long;
//   end   with y = x after start (NaN up to start), the first position of S_end that begins a run of y <= thr_dry_end at
//         least window_dry_end long (per_day), or ends a window_dry_end window whose sum is <= thr_dry_end (total).
// The first-run rule (`_get_first_run`, argmax != argmin) gives no answer when S holds no candidate, or only candidates.
// Window sums follow `window_stat` of rolling.cu: a float64 sum in time order (NaN if any element is NaN), rounded once
// to float32 (DESIGN.md section 4).
//
// One pass over the period, in time order: stop(p) is known wd - 1 steps after p, so the event automaton runs that
// far behind the reads, with the wet flags of the steps in between in a 64-bit delay line (wd <= XC_RS_MAX_WINDOW).
// The end search runs at the automaton's position and restarts at every event run that begins in S_start until the
// first of them qualifies as the start; its end search is then already under way.  Windows are re-read (L1 / L2 hits
// on the device).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/xclim_b200.h"

#if defined(__CUDACC__)
#define XC_RS_HD __host__ __device__ __forceinline__
#else
#define XC_RS_HD inline
#endif

namespace xc {
namespace rs {

struct Args {
  const float* x;
  int64_t T, C, ldx;
  const int32_t* poff;  // (P + 1) row offsets of the periods
  int32_t P;
  const uint8_t* mask;  // (T) XC_RS_PRE | XC_RS_START | XC_RS_END
  float scale, thr_wet, thr_dry_start, thr_dry_end;
  int32_t window_wet, window_not_dry, window_dry_start, method_dry_start, window_dry_end, method_dry_end;
  int32_t* out_start;   // (P, C) step of the start inside its period, -1 for none
  int32_t* out_end;     // (P, C) step of the end inside its period, -1 for none
};

// Thresholds are Python floats against float32 data: numpy >= 2 compares them in float32 (NEP 50).
inline Args make_args(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* poff, int32_t P,
                      const uint8_t* mask, float scale, double thr_wet, int32_t window_wet, int32_t window_not_dry,
                      double thr_dry_start, int32_t window_dry_start, int32_t method_dry_start, double thr_dry_end,
                      int32_t window_dry_end, int32_t method_dry_end, int32_t* out_start, int32_t* out_end) {
  Args a{};
  a.x = x; a.T = T; a.C = C; a.ldx = ldx; a.poff = poff; a.P = P; a.mask = mask;
  a.scale = scale;
  a.thr_wet = (float)thr_wet; a.thr_dry_start = (float)thr_dry_start; a.thr_dry_end = (float)thr_dry_end;
  a.window_wet = window_wet; a.window_not_dry = window_not_dry;
  a.window_dry_start = window_dry_start; a.method_dry_start = method_dry_start;
  a.window_dry_end = window_dry_end; a.method_dry_end = method_dry_end;
  a.out_start = out_start; a.out_end = out_end;
  return a;
}

// XC_OK, or the status of the C ABI with its message in *msg
inline int32_t check_args(const Args& a, const char** msg) {
  *msg = nullptr;
  if (!a.x || !a.poff || !a.mask || !a.out_start || !a.out_end) *msg = "null pointer argument";
  else if (!(a.T > 0 && a.C > 0 && a.ldx >= a.C && a.P > 0 && a.P <= 65535 && a.T < 2147483647LL)) *msg = "bad shape";
  else if (a.method_dry_start != XC_RS_PER_DAY && a.method_dry_start != XC_RS_TOTAL) *msg = "Unknown method_dry_start.";
  else if (a.method_dry_end != XC_RS_PER_DAY && a.method_dry_end != XC_RS_TOTAL) *msg = "Unknown method_dry_end.";
  else if (a.window_wet < 1 || a.window_dry_start < 1 || a.window_dry_end < 1) *msg = "windows must be >= 1";
  else if (a.window_not_dry < 0) *msg = "window_not_dry_start must be >= 0";
  if (*msg) return XC_ERR_INVALID;
  if (a.window_dry_start > XC_RS_MAX_WINDOW) {
    *msg = "window_dry_start above 64 days is not supported";
    return XC_ERR_UNSUPPORTED;
  }
  return XC_OK;
}

XC_RS_HD float load(const float* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
XC_RS_HD uint8_t load(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// float32 of the float64 sum of v(lo .. hi) in time order (NaN if any element is NaN)
template <class V>
XC_RS_HD float window_sum(const V& v, int lo, int hi) {
  double s = 0.0;
  for (int k = lo; k <= hi; ++k) s += (double)v(k);
  return (float)s;
}

XC_RS_HD void scan(const Args& a, int64_t c, int p) {
  const int t0 = a.poff[p], t1 = a.poff[p + 1];
  const float* col = a.x + c;
  const float scale = a.scale;
  const int64_t ldx = a.ldx;
  const uint8_t* mask = a.mask;
  auto amount = [=](int t) -> float { return load(col + (int64_t)t * ldx) * scale; };
  auto amount_s = [=](int t) -> float { return (load(mask + t) & XC_RS_PRE) ? amount(t) : NAN; };

  const int ww = a.window_wet, wd = a.window_dry_start, we = a.window_dry_end;
  const int D = wd - 1;                                         // delay of stop(q) behind the reads
  const int64_t need = (int64_t)a.window_not_dry + ww;          // event run length of a candidate start
  const bool dry_per_day = a.method_dry_start == XC_RS_PER_DAY, end_per_day = a.method_dry_end == XC_RS_PER_DAY;

  uint64_t wet_line = 0;  // bit k: wet(t - k)
  int dry_run = 0;        // per_day: dry steps of x_s ending at t
  // event automaton at q = t - D
  bool ev = false, run_in_s = false, s_other = false;
  int64_t run_len = 0;
  int run_at = -1, start = -1;
  // end search at q, over y = x after `from`
  int from = -1, end = -1, e_run = 0, e_run_at = -1;
  bool e_run_in_s = false, e_other = false, e_seen = false;

  for (int t = t0; t < t1 + D; ++t) {
    bool wet = false, stop = false;
    if (t < t1) {
      wet = t - ww + 1 >= t0 && window_sum(amount_s, t - ww + 1, t) >= a.thr_wet;
      if (dry_per_day) {
        dry_run = amount_s(t) <= a.thr_dry_start ? dry_run + 1 : 0;
        stop = dry_run >= wd;
      } else {
        stop = t - D >= t0 && window_sum(amount_s, t - D, t) <= a.thr_dry_start;
      }
    }
    wet_line = (wet_line << 1) | (uint64_t)wet;
    const int q = t - D;
    if (q < t0) continue;
    const uint8_t m = load(mask + q);
    const bool in_s = m & XC_RS_START, in_e = m & XC_RS_END;

    // ---- events and candidate starts (rle(index="first") >= need)
    const bool prev = ev;
    ev = !stop && (((wet_line >> D) & 1u) || prev);
    if (ev && !prev) {
      run_at = q;
      run_len = 0;
      run_in_s = in_s;
      if (start < 0 && in_s) {  // a possible start: search for its end from here on
        from = q;
        end = -1;
        e_run = 0;
        e_other = e_seen;       // the S_end steps up to here are NaN in y, hence no candidates
      }
    } else if (in_s) {
      s_other = true;           // not the first step of an event run
    }
    if (ev) {
      if (++run_len == need && run_in_s && start < 0) start = run_at;
    } else if (prev && run_in_s && run_len < need) {
      s_other = true;           // an event run too short
    }

    // ---- end candidates
    if (end_per_day) {
      if (from >= 0 && q > from && amount(q) <= a.thr_dry_end) {
        if (e_run == 0) {
          e_run_at = q;
          e_run_in_s = in_e;
        } else if (in_e) {
          e_other = true;
        }
        if (++e_run == we && e_run_in_s && end < 0) end = e_run_at;
      } else {
        if (in_e || (e_run > 0 && e_run < we && e_run_in_s)) e_other = true;
        e_run = 0;
      }
    } else if (in_e) {
      if (from >= 0 && q - we + 1 > from && window_sum(amount, q - we + 1, q) <= a.thr_dry_end) {
        if (end < 0) end = q;
      } else {
        e_other = true;
      }
    }
    e_seen = e_seen || in_e;
  }
  // runs still open at the period end are cut there
  if (ev && run_in_s && run_len < need) s_other = true;
  if (e_run > 0 && e_run < we && e_run_in_s) e_other = true;

  const bool has_start = start >= 0 && s_other;
  const int64_t o = (int64_t)p * a.C + c;
  a.out_start[o] = has_start ? start - t0 : -1;
  a.out_end[o] = has_start && end >= 0 && e_other ? end - t0 : -1;
}

}  // namespace rs
}  // namespace xc
