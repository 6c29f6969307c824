// Rolling-window primitives: (1) rolling statistic then per-period reduction, (2) spell statistics
// for spells defined by a rolling window (window > 1).
//
// Replaces:
//   indices/generic.py:128-174   select_rolling_resample_op   (da.rolling(time=w).<op>() then resample)
//   indices/_simple.py:485-525   max_n_day_precipitation_amount
//   indices/generic.py:434-540   spell_mask, general path (:519-535) and min/max fast path (:503-518)
//   indices/generic.py:543-585   _spell_length_statistics (window > 1)
//
// Design: a lane owns one cell and walks the time steps of one period; the w values of a
// window are re-read from L1/L2 (the rows were just fetched by the same warp), so DRAM traffic stays
// one read of the input.  These are the low-volume members of the family (the window == 1 fast
// kernels in period_stats.cu carry the headline configurations); operators are runtime switches.
#include "launch_plan.cuh"
#include "runstat.cuh"
#include <limits>
#include <type_traits>
#include <string.h>

namespace xc {
namespace {

// A switch on the uniform operator, not bivariate.cu's branch-free OpMask: with the mask form the
// compute-bound spell_runstat4_kernel runs about 14% slower.
__device__ __forceinline__ bool cmp_rt(int op, float x, float t) {
  switch (op) {
    case XC_OP_GT: return x > t;
    case XC_OP_LT: return x < t;
    case XC_OP_GE: return x >= t;
    case XC_OP_LE: return x <= t;
    case XC_OP_EQ: return x == t;
    default: return x != t;
  }
}

// statistic of x[i .. i+w-1] (NaN if any element is NaN) -- xarray rolling with min_periods == w
__device__ __forceinline__ float window_stat(const float* __restrict__ col, int64_t ldx, int i, int w, int stat) {
  double s = 0.0;
  float mn = INFINITY, mx = -INFINITY;
  bool nan = false;
  for (int k = 0; k < w; ++k) {
    const float v = __ldg(col + (int64_t)(i + k) * ldx);
    nan = nan || (v != v);
    s += (double)v;
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  if (nan) return NAN;
  switch (stat) {
    case XC_STAT_SUM: return (float)s;
    case XC_STAT_MEAN: return (float)(s / (double)w);
    case XC_STAT_MIN: return mn;
    default: return mx;
  }
}

// s += v; true when the float64 add is exact.  r = s + v exactly <=> r - s == v and r - v == s (the
// difference with the larger operand is computed exactly, Fast2Sum), and an infinity fails the test (inf - inf).
__device__ __forceinline__ bool add_exact(double& s, double v) {
  const double r = s + v;
  const bool ok = (r - s == v) & (r - v == s);
  s = r;
  return ok;
}

// Sliding window state for sum / mean windows: float64 sum of the non-NaN values plus the number of NaNs in
// the window.  A running sum (new value in, oldest out) is the window_stat value only while it is exact: an
// infinity leaving the window would leave NaN behind (inf - inf), and a value that absorbed its neighbours
// (the 9.97e36 netCDF fill) would leave their loss behind.  So every update is checked, and a window reached
// through a rounded update is summed again directly, oldest value first -- exactly window_stat's sum.  That
// happens only while the window holds such a value: on ordinary data every update is exact.
struct SlideSum {
  double s;
  int nan;
  bool exact;     // s is the exact sum of the window's non-NaN values
  // the direct sum of x[i .. i+w-1]
  __device__ __forceinline__ void load(const float* __restrict__ col, int64_t ldx, int i, int w) {
    s = 0.0;
    nan = 0;
    exact = true;
    for (int k = 0; k < w; ++k) {
      const float v = __ldg(col + (int64_t)(i + k) * ldx);
      if (v != v) ++nan;
      else exact &= add_exact(s, (double)v);
    }
  }
  // window [i, i+w-1] -> [i+1, i+w]: vin = x[i+w] enters, vout = x[i] leaves
  __device__ __forceinline__ void slide(float vin, float vout, const float* __restrict__ col, int64_t ldx, int i,
                                        int w) {
    bool ok = exact;
    if (vin != vin) ++nan;
    else ok &= add_exact(s, (double)vin);
    if (vout != vout) --nan;
    else ok &= add_exact(s, -(double)vout);
    if (!ok) load(col, ldx, i + 1, w);
  }
  __device__ __forceinline__ float value(int wstat, int w) const {
    return nan ? NAN : (float)(wstat == XC_STAT_MEAN ? s / (double)w : s);
  }
};

constexpr int kChunk = 8;

__global__ void __launch_bounds__(kThreads)
rolling_period_reduce_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                             const int32_t* __restrict__ poff, int32_t w, int32_t wstat, int32_t shift,
                             int32_t stat, float* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c;
  StatAcc acc;
  acc.init(stat);
  // the value labelled t covers x[i .. i+w-1], i = t + shift - w + 1 (shift 0: right-aligned, w/2: centred)
  if (wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN) {
    int t = t0;
    // labels whose window is incomplete at the series start give NaN
    while (t < t1 && t + shift - w + 1 < 0) ++t;
    SlideSum win;
    int i = t + shift - w + 1;          // first complete window of this period
    if (t < t1 && i + w <= (int)T) win.load(col, ldx, i, w);
    while (t < t1 && i + w <= (int)T) {
      acc.take(win.value(wstat, w));
      // slide by up to kChunk steps with all loads issued first
      const int steps = min(kChunk, min(t1 - 1 - t, (int)T - (i + w)));
      if (steps <= 0) break;
      float vin[kChunk], vout[kChunk];
#pragma unroll
      for (int k = 0; k < kChunk; ++k) {
        if (k < steps) {
          vin[k] = ld_stream(col + (int64_t)(i + w + k) * ldx);
          vout[k] = __ldg(col + (int64_t)(i + k) * ldx);
        }
      }
#pragma unroll
      for (int k = 0; k < kChunk; ++k) {
        if (k < steps) {
          win.slide(vin[k], vout[k], col, ldx, i + k, w);
          if (k + 1 < steps) acc.take(win.value(wstat, w));
        }
      }
      t += steps;
      i += steps;
    }
  } else {
    for (int t = t0; t < t1; ++t) {
      const int i = t + shift - w + 1;
      float r = NAN;
      if (i >= 0 && i + w <= (int)T) r = window_stat(col, ldx, i, w, wstat);
      acc.take(r);
    }
  }
  out[(int64_t)p * C + c] = acc.result(stat);
}

// mask[t] = any length-w block [i, i+w-1] containing t, fully inside the series, whose window
// statistic satisfies (stat op thr)   (indices/generic.py:519-535); then run-length statistics of
// the mask per period (window == 1 on the mask, generic.py:562-570).
//
// The block statistics are produced in time order by BlockStream: for sum / mean windows a sliding
// float64 sum (+ NaN counter, SlideSum), two loads per step; for min / max windows the w values are re-read
// (L1 hits).
struct BlockStream {
  const float* col;
  int64_t ldx;
  int T, w, wstat, op;
  float thr;
  int i;          // start of the next block to evaluate
  SlideSum win;   // window [i, i+w-1] when sliding
  bool primed;

  __device__ __forceinline__ void init(int start) {
    i = start;
    primed = false;
  }
  __device__ __forceinline__ bool sliding() const { return block_stream_slides(wstat, w); }
  // qualifies(block starting at i) ; advances to i + 1.  Caller guarantees i + w <= T.
  __device__ __forceinline__ bool next() {
    float r;
    if (sliding()) {
      if (!primed) {
        win.load(col, ldx, i, w);
        primed = true;
      }
      r = win.value(wstat, w);
      if (i + 1 + w <= T)    // slide to i + 1: one new row, one row re-read from L1/L2
        win.slide(__ldg(col + (int64_t)(i + w) * ldx), __ldg(col + (int64_t)i * ldx), col, ldx, i, w);
    } else {
      r = window_stat(col, ldx, i, w, wstat);
    }
    ++i;
    return cmp_rt(op, r, thr);
  }
};

__global__ void __launch_bounds__(kThreads)
spell_runstat_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                     const int32_t* __restrict__ poff, int32_t w, int32_t wstat, int32_t op, float thr,
                     int32_t reducer, int32_t after, float* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  BlockStream bs;
  bs.col = x + c; bs.ldx = ldx; bs.T = (int)T; bs.w = w; bs.wstat = wstat; bs.op = op; bs.thr = thr;
  // the mask at t needs the blocks starting in [t - w + 1, t]; with `after` the mask at t0 - 1 too
  const int first_t = after ? max(0, t0 - 1) : t0;
  bs.init(max(0, first_t - w + 1));
  int last_true = -1;
  auto mask_at = [&](int t) -> bool {
    const int imax = min(t, (int)T - w);
    while (bs.i <= imax) {
      const int ii = bs.i;
      if (bs.next()) last_true = ii;
    }
    return last_true >= 0 && last_true >= t - w + 1;
  };
  PeriodMask pm;
  pm.init();
  if (after && t0 > 0) pm.look_back(mask_at(t0 - 1));
  int32_t cur = 0;
  RunAcc<kRunAny> acc;
  acc.init();
  for (int t = t0; t < t1; ++t) run_step(cur, acc, pm.inside(after, mask_at(t)), 1);
  if (after) {
    for (int t = t1; cur > 0 && t < (int)T; ++t) run_step(cur, acc, PeriodMask::past_end(mask_at(t), cur > 0), 1);
  }
  run_close(cur, acc, 1);
  out[(int64_t)p * C + c] = acc.result(reducer);
}


// ------------------------------------------------------------------------------------------------
// Streaming variants: a thread owns 4 adjacent cells (128-bit loads), walks the rows of one period
// once and keeps the last w rows of its cells in a shared-memory ring [w][kThreads] of float4 (each
// thread only touches its own column: no synchronisation).  Sum / mean windows slide a float64 sum
// (new row in, ring row out; SlideSum's rule: re-summed from the ring after a rounded update); min / max
// windows rescan the ring.  DRAM traffic is one read of the input (+ w-1 halo rows per period) and
// nothing is re-read through L1/L2, so these run at the
// speed of the window == 1 kernels instead of the latency-bound lane-per-cell kernels above, which
// remain as the fall-back for unaligned inputs and windows that do not fit shared memory.
// ------------------------------------------------------------------------------------------------
constexpr int kU = 4;  // rows in flight per thread

// SlideSum for the 4 cells of a thread; a window reached through a rounded update is summed again from the ring
struct Win4 {
  double s[4];
  int nan[4];
  bool exact[4];
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int j = 0; j < 4; ++j) { s[j] = 0.0; nan[j] = 0; exact[j] = true; }
  }
  // appends a row: while priming, s is the direct sum of the rows appended so far
  __device__ __forceinline__ void push(const float4& v) {
    const float a[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (a[j] != a[j]) ++nan[j];
      else exact[j] &= add_exact(s[j], (double)a[j]);
    }
  }
  // vin entered and vout left; the ring holds the new window, its oldest row at `slot`
  __device__ __forceinline__ void slide(const float4& vin, const float4& vout, const float4* __restrict__ ring,
                                        int lane, int w, int slot) {
    const float a[4] = {vin.x, vin.y, vin.z, vin.w};
    const float b[4] = {vout.x, vout.y, vout.z, vout.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      bool ok = exact[j];
      if (a[j] != a[j]) ++nan[j];
      else ok &= add_exact(s[j], (double)a[j]);
      if (b[j] != b[j]) --nan[j];
      else ok &= add_exact(s[j], -(double)b[j]);
      if (!ok) {
        s[j] = 0.0;
        nan[j] = 0;
        exact[j] = true;
        for (int k = 0, r = slot; k < w; ++k, r = (r + 1 == w) ? 0 : r + 1) {
          const float4 v = ring[r * kThreads + lane];
          const float c[4] = {v.x, v.y, v.z, v.w};
          if (c[j] != c[j]) ++nan[j];
          else exact[j] &= add_exact(s[j], (double)c[j]);
        }
      }
    }
  }
};

// window statistic of the 4 cells after the ring holds the w rows ending at the current one
__device__ __forceinline__ void window_stat4(const Win4& win, const float4* __restrict__ ring, int lane, int w,
                                             int wstat, float (&r)[4]) {
  if (wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      r[j] = win.nan[j] ? NAN : (float)(wstat == XC_STAT_MEAN ? win.s[j] / (double)w : win.s[j]);
    return;
  }
  float mn[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
  float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  bool nan[4] = {false, false, false, false};
  for (int k = 0; k < w; ++k) {
    const float4 v = ring[k * kThreads + lane];
    const float a[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      nan[j] = nan[j] || (a[j] != a[j]);
      mn[j] = fminf(mn[j], a[j]);
      mx[j] = fmaxf(mx[j], a[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) r[j] = nan[j] ? NAN : (wstat == XC_STAT_MIN ? mn[j] : mx[j]);
}

// rows [r0, r1) into the ring (and the sliding sums), ring slot advancing from `slot`
__device__ __forceinline__ void prime_ring(const float* __restrict__ col, int64_t ldx, int r0, int r1,
                                           float4* __restrict__ ring, int lane, int w, int& slot, Win4& win) {
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = r0; r < r1; r += kU) {
    float4 v[kU];
#pragma unroll
    for (int k = 0; k < kU; ++k)
      if (r + k < r1) v[k] = ld_stream4(col + (int64_t)(r + k) * ldx);
#pragma unroll
    for (int k = 0; k < kU; ++k) {
      if (r + k < r1) {
        ring[slot * kThreads + lane] = v[k];
        win.push(v[k]);
        slot = (slot + 1 == w) ? 0 : slot + 1;
      }
    }
  }
  ring[slot * kThreads + lane] = zero;  // the slot the first streamed row replaces: dropping it is a no-op
}

__global__ void __launch_bounds__(kThreads)
rolling_period_reduce4_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                              const int32_t* __restrict__ poff, int32_t w, int32_t wstat, int32_t shift,
                              int32_t stat, float* __restrict__ out) {
  extern __shared__ float4 ring4[];
  const int lane = threadIdx.x;
  const int64_t c = ((int64_t)blockIdx.x * kThreads + lane) * 4;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c;
  StatAcc acc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j].init(stat);
  // the value labelled t covers the w rows ending at e = t + shift; incomplete windows give NaN (ignored)
  const int eb = max(t0 + shift, w - 1);
  const int ee = min((int)T - 1, t1 - 1 + shift);
  Win4 win;
  win.clear();
  int slot = 0;
  if (eb <= ee) prime_ring(col, ldx, eb - w + 1, eb, ring4, lane, w, slot, win);
  for (int e = eb; e <= ee; e += kU) {
    float4 v[kU];
#pragma unroll
    for (int k = 0; k < kU; ++k)
      if (e + k <= ee) v[k] = ld_stream4(col + (int64_t)(e + k) * ldx);
#pragma unroll
    for (int k = 0; k < kU; ++k) {
      if (e + k <= ee) {
        const float4 old = ring4[slot * kThreads + lane];
        ring4[slot * kThreads + lane] = v[k];
        slot = (slot + 1 == w) ? 0 : slot + 1;
        if (wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN) win.slide(v[k], old, ring4, lane, w, slot);
        float r[4];
        window_stat4(win, ring4, lane, w, wstat, r);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j].take(r[j]);
      }
    }
  }
  *reinterpret_cast<float4*>(out + (int64_t)p * C + c) =
      make_float4(acc[0].result(stat), acc[1].result(stat), acc[2].result(stat), acc[3].result(stat));
}

// Spell statistics, streaming form.  cond(e) = (statistic of the w rows ending at e) op thr;
// mask[t] = any e in [t, t+w-1] with cond(e)  <=>  (latest e' <= t+w-1 with cond(e')) >= t, so a
// per-cell `last` index is the whole mask state and mask[t] is final once row t+w-1 has been seen.
template <bool AFTER>
__global__ void __launch_bounds__(kThreads)
spell_runstat4_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                      const int32_t* __restrict__ poff, int32_t w, int32_t wstat, int32_t op, float thr,
                      int32_t reducer, float* __restrict__ out) {
  extern __shared__ float4 ring4[];
  const int lane = threadIdx.x;
  const int64_t c = ((int64_t)blockIdx.x * kThreads + lane) * 4;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const int Ti = (int)T;
  const float* col = x + c;
  const int first_t = (AFTER && t0 > 0) ? t0 - 1 : t0;
  int last[4] = {-1, -1, -1, -1};
  int32_t cur[4] = {0, 0, 0, 0};
  PeriodMask pm[4];
  RunAcc<kRunAny> acc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { pm[j].init(); acc[j].init(); }
  // mask value of step t for cell j (t >= first_t, in time order)
  auto feed = [&](int j, int t, bool mk) {
    if (AFTER && t < t0) pm[j].look_back(mk);
    else if (AFTER && t >= t1) run_step(cur[j], acc[j], PeriodMask::past_end(mk, cur[j] > 0), 1);
    else run_step(cur[j], acc[j], pm[j].inside(AFTER, mk), 1);
  };
  auto open_any = [&]() { return (cur[0] | cur[1] | cur[2] | cur[3]) != 0; };

  const int sb = max(first_t, w - 1);                      // first row whose window is evaluated
  const int s_lim = AFTER ? Ti - 1 : min(Ti - 1, t1 - 1 + w - 1);
  Win4 win;
  win.clear();
  int slot = 0;
  if (sb <= s_lim) prime_ring(col, ldx, sb - w + 1, sb, ring4, lane, w, slot, win);
  int s = sb;
  while (s <= s_lim) {
    const int steps = min(kU, s_lim - s + 1);
    float4 v[kU];
#pragma unroll
    for (int k = 0; k < kU; ++k)
      if (k < steps) v[k] = ld_stream4(col + (int64_t)(s + k) * ldx);
#pragma unroll
    for (int k = 0; k < kU; ++k) {
      if (k < steps) {
        const float4 old = ring4[slot * kThreads + lane];
        ring4[slot * kThreads + lane] = v[k];
        slot = (slot + 1 == w) ? 0 : slot + 1;
        if (wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN) win.slide(v[k], old, ring4, lane, w, slot);
        float r[4];
        window_stat4(win, ring4, lane, w, wstat, r);
        const int e = s + k, t = e - w + 1;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (cmp_rt(op, r[j], thr)) last[j] = e;
          if (t >= first_t) feed(j, t, last[j] >= t);
        }
      }
    }
    s += steps;
    if (AFTER && s - w + 1 >= t1 && !open_any()) break;   // every run of this period has ended
  }
  // steps whose later windows would leave the series: no new condition can cover them
  for (int t = max(first_t, s - w + 1); t < Ti; ++t) {
    if (t >= t1 && !(AFTER && open_any())) break;
#pragma unroll
    for (int j = 0; j < 4; ++j) feed(j, t, last[j] >= t);
  }
  float res[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    run_close(cur[j], acc[j], 1);
    res[j] = acc[j].result(reducer);
  }
  *reinterpret_cast<float4*>(out + (int64_t)p * C + c) = make_float4(res[0], res[1], res[2], res[3]);
}


// ------------------------------------------------------------------------------------------------
// Short sum / mean windows (2 <= w <= 8), the common case (dry/wet spells: 3; n-day amounts: 2..7):
// the window lives in REGISTERS as float64 values, the loop is unrolled over the w ring positions so every index is static, and the window
// sum is re-added from the ring at every step in window order (oldest first): no sliding, hence
// no drift and no cancellation residue -- the value is the same direct float64 sum the
// lane-per-cell kernel computes.  One float32->float64 conversion per element (the conversion pipe
// runs at 16/clk/SM) and w-1 float64 adds.
//
// The comparison of the window statistic with the threshold happens on the float64 SUM: the map
// s -> (float)(s) or (float)(s / w) is monotone, so {s : stat(s) op thr} is an interval [lo, hi) of
// float64 sums (or its complement) that the host finds by bisection over the ordered doubles with
// the very same operations -- no per-element division or float64->float32 conversion.
// ------------------------------------------------------------------------------------------------
struct SumRange {
  double lo, hi;        // stat(s) op thr  <=>  ((s >= lo) && (hi_unbounded || s < hi)) != negate
  int hi_unbounded;
  int negate;
  int nan_cond;         // value of (NaN op thr)
};

// branch-free on purpose (bitwise, not short-circuit, operators): two DSETP and a predicate op
__device__ __forceinline__ bool in_range(const SumRange& g, double s) {
  const bool a = (s >= g.lo) & ((g.hi_unbounded != 0) | (s < g.hi));
  return a != (g.negate != 0);
}

constexpr int unroll_for(int W) { return W >= 4 ? W : (W == 3 ? 6 : 4); }

__device__ __noinline__ float mean_of_sum(double s, double w) { return (float)(s / w); }

template <int W, int RED, bool AFTER>
__global__ void __launch_bounds__(kThreads)
spell_sumw_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                  SumRange rng, int32_t reducer, float* __restrict__ out) {
  constexpr int U = unroll_for(W);
  const int64_t c = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * 4;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const int Ti = (int)T;
  const float* col = x + c;
  const int first_t = (AFTER && t0 > 0) ? t0 - 1 : t0;
  double ring[W][4];
#pragma unroll
  for (int k = 0; k < W; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) ring[k][j] = 0.0;
  int last[4] = {-1, -1, -1, -1};
  bool skip[4] = {false, false, false, false};
  // MAX / SUM / COUNT keep run_step's running form; any other reducer closes runs into RunAcc<kRunAny>
  constexpr bool kRunning = RED == XC_RL_MAX || RED == XC_RL_SUM || RED == XC_RL_COUNT;
  int cur[4] = {0, 0, 0, 0};
  RunAcc<kRunning ? RED : kRunAny> acc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j].init();
  // run-length update with the mask value of the next step (cur > 0 <=> a run is open)
  auto update = [&](int j, bool mk) {
    if constexpr (kRunning) {
      run_step<true>(cur[j], acc[j], mk, 1);
    } else if (mk) {
      ++cur[j];
    } else {
      acc[j].add(cur[j], cur[j] > 0);
      cur[j] = 0;
    }
  };
  // The period-edge rule of runstat.cuh (PeriodMask), kept as a copy: with PeriodMask's look_back / inside / past_end
  // in place of the lambdas below, ptxas spills 64 bytes in the W = 5 MAX, SUM and COUNT instances with
  // resample_before_rl=False.
  // inside the period: with resample_before_rl=False a run that was already open at t0 is skipped
  auto feed_inside = [&](int j, bool mk) {
    if (AFTER) {
      skip[j] = skip[j] & mk;
      mk = mk & !skip[j];
    }
    update(j, mk);
  };
  auto feed = [&](int j, int t, bool mk) {
    if (AFTER) {
      if (t < t0) { skip[j] = mk; return; }
      if (t >= t1) {                   // past the period end only an open run is followed
        if (cur[j] != 0) update(j, mk);
        return;
      }
    }
    feed_inside(j, mk);
  };
  auto open_any = [&]() { return (cur[0] | cur[1] | cur[2] | cur[3]) != 0; };

  const int sb = max(first_t, W - 1);                      // first row whose window is evaluated
  const int s_lim = AFTER ? Ti - 1 : min(Ti - 1, t1 - 1 + W - 1);

  // U rows starting at `base`.  STEADY: every row exists, is evaluated, and its step lies inside
  // the period -- no per-row conditions at all.
  auto chunk = [&](auto steady_tag, int base) {
    constexpr bool STEADY = decltype(steady_tag)::value;
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (STEADY || base + u <= s_lim) v[u] = ld_stream4(col + (int64_t)(base + u) * ldx);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int e = base + u;
      if (STEADY || e <= s_lim) {
        const float a[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) ring[u % W][j] = (double)a[j];
        if (STEADY || e >= sb) {
          const int t = e - W + 1;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            double sw = ring[(u + 1) % W][j];              // oldest row of the window first
#pragma unroll
            for (int k = 2; k <= W; ++k) sw += ring[(u + k) % W][j];
            // a NaN in the window makes the sum NaN and in_range(NaN) == negate == (NaN op thr)
            const bool cond = in_range(rng, sw);
            last[j] = cond ? e : last[j];
            if (STEADY) feed_inside(j, last[j] >= t);
            else if (t >= first_t) feed(j, t, last[j] >= t);
          }
        }
      }
    }
  };

  int s = sb;                                              // next row to evaluate (for the tail loop)
  if (sb <= s_lim) {
    for (int base = sb - W + 1; base <= s_lim; base += U) {
      const bool steady = (base - W + 1 >= t0) && (base + U - 1 <= s_lim) && (base + U - W < t1);
      if (steady) chunk(std::true_type{}, base);
      else chunk(std::false_type{}, base);
      s = min(base + U, s_lim + 1);
      if (AFTER && s - W + 1 >= t1 && !open_any()) break;
    }
  }
  for (int t = max(first_t, s - W + 1); t < Ti; ++t) {
    if (t >= t1 && !(AFTER && open_any())) break;
#pragma unroll
    for (int j = 0; j < 4; ++j) feed(j, t, last[j] >= t);
  }
  float res[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if constexpr (!kRunning) acc[j].add(cur[j], cur[j] > 0);   // the run closed by the period / series end
    res[j] = acc[j].result(reducer);
  }
  *reinterpret_cast<float4*>(out + (int64_t)p * C + c) = make_float4(res[0], res[1], res[2], res[3]);
}

// rolling sum / mean of w rows then a per-period statistic.  MODE 0 / 1: max / min of the rolling
// value, tracked on the float64 sums (monotone map, converted once at the end); MODE 2: the other
// statistics convert every value.
template <int W, int MODE>
__global__ void __launch_bounds__(kThreads)
rolling_sumw_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                    int32_t is_mean, int32_t shift, int32_t stat, float* __restrict__ out) {
  constexpr int U = unroll_for(W);
  const int64_t c = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * 4;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c;
  const int eb = max(t0 + shift, W - 1);
  const int ee = min((int)T - 1, t1 - 1 + shift);
  double ring[W][4];
#pragma unroll
  for (int k = 0; k < W; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) ring[k][j] = 0.0;
  double s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0}, m[4];
  int n[4] = {0, 0, 0, 0};
#pragma unroll
  for (int j = 0; j < 4; ++j) m[j] = (MODE == 1) ? INFINITY : -INFINITY;
  auto chunk = [&](auto steady_tag, int base) {
    constexpr bool STEADY = decltype(steady_tag)::value;
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (STEADY || base + u <= ee) v[u] = ld_stream4(col + (int64_t)(base + u) * ldx);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int e = base + u;
      if (STEADY || e <= ee) {
        const float a[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) ring[u % W][j] = (double)a[j];
        if (STEADY || e >= eb) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            double sw = ring[(u + 1) % W][j];
#pragma unroll
            for (int k = 2; k <= W; ++k) sw += ring[(u + k) % W][j];
            const bool valid = (sw == sw);   // a NaN in the window (or inf + -inf) gives a NaN sum: ignored
            n[j] += valid ? 1 : 0;
            if constexpr (MODE == 0) {
              m[j] = (valid & (sw > m[j])) ? sw : m[j];
            } else if constexpr (MODE == 1) {
              m[j] = (valid & (sw < m[j])) ? sw : m[j];
            } else {
              if (valid) {
                const float r = is_mean ? mean_of_sum(sw, (double)W) : (float)sw;
                s[j] += (double)r;
                q[j] += (double)r * (double)r;
              }
            }
          }
        }
      }
    }
  };
  if (eb <= ee) {
    for (int base = eb - W + 1; base <= ee; base += U) {
      if (base >= eb && base + U - 1 <= ee) chunk(std::true_type{}, base);
      else chunk(std::false_type{}, base);
    }
  }
  float res[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    // stat_result()'s formula, kept as a copy: calling it changes this kernel's code.  Every operation rounded, as
    // there: this file is built with -fmad.
    const double nn = (double)n[j];
    switch (stat) {
      case XC_STAT_SUM: res[j] = (float)s[j]; break;
      case XC_STAT_COUNT: res[j] = (float)n[j]; break;
      case XC_STAT_MEAN: res[j] = n[j] ? (float)(s[j] / nn) : NAN; break;
      case XC_STAT_MIN:
      case XC_STAT_MAX: res[j] = n[j] ? (float)(is_mean ? m[j] / (double)W : m[j]) : NAN; break;
      default: {
        if (!n[j]) { res[j] = NAN; break; }
        const double mean = __ddiv_rn(s[j], nn);
        double var = __dsub_rn(__ddiv_rn(q[j], nn), __dmul_rn(mean, mean));
        var = var > 0.0 ? var : 0.0;
        res[j] = (stat == XC_STAT_STD) ? (float)__dsqrt_rn(var) : (float)var;
      }
    }
  }
  *reinterpret_cast<float4*>(out + (int64_t)p * C + c) = make_float4(res[0], res[1], res[2], res[3]);
}

// ---- host side: the interval of float64 sums whose statistic satisfies `op thr` -----------------
inline int64_t dkey(double d) {   // order-preserving map double -> int64 (no NaN)
  int64_t b;
  memcpy(&b, &d, 8);
  return b >= 0 ? b : (int64_t)(0x8000000000000000ull - (uint64_t)b) ;
}
inline double dunkey(int64_t k) {
  int64_t b = k >= 0 ? k : (int64_t)(0x8000000000000000ull - (uint64_t)k);
  double d;
  memcpy(&d, &b, 8);
  return d;
}
inline float sum_stat(double s, int w, bool mean) { return (float)(mean ? s / (double)w : s); }

// smallest double s (in the total order -inf .. +inf) with stat(s) >= thr (strict: > thr); false if none
inline bool first_sum_reaching(float thr, int w, bool mean, bool strict, double* out) {
  auto ok = [&](double s) { const float r = sum_stat(s, w, mean); return strict ? (r > thr) : (r >= thr); };
  int64_t lo = dkey(-INFINITY), hi = dkey(INFINITY);
  if (!ok(dunkey(hi))) return false;
  if (ok(dunkey(lo))) { *out = -INFINITY; return true; }
  while ((uint64_t)hi - (uint64_t)lo > 1) {   // invariant: !ok(lo), ok(hi)
    const int64_t mid = (lo >> 1) + (hi >> 1) + (lo & hi & 1);   // no overflow across the sign change
    if (ok(dunkey(mid))) hi = mid; else lo = mid;
  }
  *out = dunkey(hi);
  return true;
}

inline SumRange make_sum_range(int op, float thr, int w, bool mean) {
  SumRange g;
  g.lo = -INFINITY; g.hi = INFINITY; g.hi_unbounded = 1; g.negate = 0;
  g.nan_cond = (op == XC_OP_NE) ? 1 : 0;
  const double qnan = std::numeric_limits<double>::quiet_NaN();
  if (thr != thr) {               // every comparison with NaN is false, except !=
    g.lo = qnan;                  // s >= NaN is false: empty interval
    g.negate = (op == XC_OP_NE) ? 1 : 0;
    return g;
  }
  double bge = 0, bgt = 0;
  const bool hge = first_sum_reaching(thr, w, mean, false, &bge);
  const bool hgt = first_sum_reaching(thr, w, mean, true, &bgt);
  switch (op) {
    case XC_OP_GT: g.lo = hgt ? bgt : qnan; break;
    case XC_OP_GE: g.lo = hge ? bge : qnan; break;
    case XC_OP_LT: if (hge) { g.hi = bge; g.hi_unbounded = 0; } break;
    case XC_OP_LE: if (hgt) { g.hi = bgt; g.hi_unbounded = 0; } break;
    default:       // EQ: [bge, bgt) ; NE: its complement
      g.lo = hge ? bge : qnan;
      if (hgt) { g.hi = bgt; g.hi_unbounded = 0; }
      g.negate = (op == XC_OP_NE) ? 1 : 0;
  }
  return g;
}

// spell_sumw_kernel<W, RED, AFTER> with the plan's RED (the run-length reducer stays a run-time argument)
template <int W, bool AFTER>
int32_t launch_spell_sumw(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* poff, int32_t P,
                          const SumRange& g, int32_t red, int32_t reducer, float* out, cudaStream_t st) {
  dim3 grid((unsigned)((C / 4 + kThreads - 1) / kThreads), (unsigned)P, 1);
  switch (red) {
    case XC_RL_MAX: spell_sumw_kernel<W, XC_RL_MAX, AFTER><<<grid, kThreads, 0, st>>>(x, T, C, ldx, poff, g, reducer, out); break;
    case XC_RL_SUM: spell_sumw_kernel<W, XC_RL_SUM, AFTER><<<grid, kThreads, 0, st>>>(x, T, C, ldx, poff, g, reducer, out); break;
    case XC_RL_COUNT: spell_sumw_kernel<W, XC_RL_COUNT, AFTER><<<grid, kThreads, 0, st>>>(x, T, C, ldx, poff, g, reducer, out); break;
    default: spell_sumw_kernel<W, kRunAny, AFTER><<<grid, kThreads, 0, st>>>(x, T, C, ldx, poff, g, reducer, out);
  }
  return launch_status("spell_sumw_kernel");
}

// rolling_sumw_kernel<W, MODE> with the plan's MODE
template <int W>
int32_t launch_rolling_sumw(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* poff, int32_t P,
                            int32_t mode, int32_t is_mean, int32_t shift, int32_t stat, float* out, cudaStream_t st) {
  dim3 grid((unsigned)((C / 4 + kThreads - 1) / kThreads), (unsigned)P, 1);
  if (mode == 0)
    rolling_sumw_kernel<W, 0><<<grid, kThreads, 0, st>>>(x, T, C, ldx, poff, is_mean, shift, stat, out);
  else if (mode == 1)
    rolling_sumw_kernel<W, 1><<<grid, kThreads, 0, st>>>(x, T, C, ldx, poff, is_mean, shift, stat, out);
  else
    rolling_sumw_kernel<W, 2><<<grid, kThreads, 0, st>>>(x, T, C, ldx, poff, is_mean, shift, stat, out);
  return launch_status("rolling_sumw_kernel");
}

// f(W) for the window w of a register-kernel plan, W in [kRegisterWMin, kRegisterWMax]
template <int W = kRegisterWMin, typename F>
int32_t dispatch_register_window(int w, F&& f) {
  if constexpr (W > kRegisterWMax) {
    set_error("no register kernel for window %d", w);
    return XC_ERR_INVALID;
  } else {
    return w == W ? f(std::integral_constant<int, W>{}) : dispatch_register_window<W + 1>(w, f);
  }
}


// ------------------------------------------------------------------------------------------------
// spell mask, materialised (SURVEY.md 8f.2: `select_time` on the spell mask, indices/generic.py:557-558)
// ------------------------------------------------------------------------------------------------
// mask[t, c] = NaN where keep[t] == 0 (out of the selected season), else 1 / 0 = day t belongs / does not
// belong to a length-w block whose window statistic satisfies the condition (indices/generic.py:503-535,
// computed on the UNMASKED series: the reference selects after the spell mask is built).  Run statistics of
// this mask with `x > 0` are the reference's per-series path (statistics_run_1d, run_length.py:1408-1437):
// a NaN ends a run, the in-season part of a spell under way on the first in-season day counts with its
// in-season length (tests/test_indices.py:4116-4126 expects 9).  keep[t] == 2 marks a first in-season day
// that is not the first step of its resampling group: with drop_nan_adjacent != 0 a run STARTING there is
// zeroed, which is what the whole-array `rle` does (its `where(shift == 0)` test fails next to a NaN,
// run_length.py:264) -- the two reference paths disagree, the caller chooses.
// A lane owns a cell and walks the series (this is the rarely used seasonal path, not a headline kernel).
__global__ void __launch_bounds__(kThreads)
spell_mask_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, int32_t w, int32_t wstat,
                  int32_t op, float thr, const uint8_t* __restrict__ keep, int32_t drop_nan_adjacent,
                  float* __restrict__ mask) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  BlockStream bs;
  bs.col = x + c;
  bs.ldx = ldx;
  bs.T = (int)T;
  bs.w = w;
  bs.wstat = wstat;
  bs.op = op;
  bs.thr = thr;
  bs.init(0);
  int last = -(1 << 30);      // start of the latest qualifying block
  bool dropping = false;
  for (int t = 0; t < (int)T; ++t) {
    if (t + w <= (int)T && bs.next()) last = t;           // block [t, t + w - 1]
    const bool in = last >= t - w + 1;
    const int k = keep ? (int)keep[t] : 1;
    float v;
    if (k == 0) {
      v = NAN;
      dropping = false;
    } else {
      if (drop_nan_adjacent && k == 2 && in) dropping = true;   // a run starts right after a masked step
      if (!in) dropping = false;
      v = (in && !dropping) ? 1.f : 0.f;
    }
    mask[(int64_t)t * C + c] = v;
  }
}


// select_rolling_resample_op(**indexer) -- indices/generic.py:128-174: the rolling statistic is computed on the
// WHOLE series and `select_time` then keeps the rolled values whose label lies in the selection
// (generic.py:169-174), so the selection is a mask on the LABELS of the windows, not on the input.
// Lane = (cell, period); every kept label re-reads its window (L1 hits).  The seasonal path, not a headline.
__global__ void __launch_bounds__(kThreads)
rolling_period_reduce_sel_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                                 const int32_t* __restrict__ poff, int32_t w, int32_t wstat, int32_t shift,
                                 int32_t stat, const uint8_t* __restrict__ keep, float* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c;
  StatAcc acc;
  acc.init(stat);
  for (int t = t0; t < t1; ++t) {
    if (!keep[t]) continue;
    const int i = t + shift - w + 1;
    if (i < 0 || i + w > (int)T) continue;            // incomplete window: NaN, skipped by the reduction
    acc.take(window_stat(col, ldx, i, w, wstat));
  }
  out[(int64_t)p * C + c] = acc.result(stat);
}

// The rolled series itself (standardized indices, indices/stats.py:831-832): each label's window mean by
// window_stat, a direct float64 sum of its w values, so an infinity stays confined to the windows holding it.
// blockIdx.y walks chunks of kRollChunk labels; the window's other values are L1 / L2 hits.
constexpr int kRollChunk = 32;

__global__ void __launch_bounds__(kThreads)
rolling_mean_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, int32_t w,
                    float* __restrict__ out, int64_t ldo) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int t0 = blockIdx.y * kRollChunk;
  const int t1 = min((int)T, t0 + kRollChunk);
  for (int t = t0; t < t1; ++t)
    out[(int64_t)t * ldo + c] = (t < w - 1) ? NAN : window_stat(x + c, ldx, t - w + 1, w, XC_STAT_MEAN);
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int32_t xc_rolling_mean_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t window, float* out,
                                       int64_t ldo, void* stream) {
  XC_REQUIRE(x && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && ldo >= C && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1, "window must be >= 1");
  XC_REQUIRE((T + kRollChunk - 1) / kRollChunk <= 65535, "series longer than %d steps", 65535 * kRollChunk);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)((T + kRollChunk - 1) / kRollChunk), 1);
  rolling_mean_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(x, T, C, ldx, window, out, ldo);
  return launch_status("rolling_mean_kernel");
}

extern "C" int32_t xc_rolling_period_reduce_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                                const int32_t* period_offsets, int32_t P, int32_t window,
                                                int32_t window_stat, int32_t center, int32_t stat, float* out,
                                                void* stream) {
  XC_REQUIRE(x && period_offsets && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1 && window <= T, "window must be in [1, T]");
  XC_REQUIRE(window_stat == XC_STAT_SUM || window_stat == XC_STAT_MEAN || window_stat == XC_STAT_MIN ||
                 window_stat == XC_STAT_MAX,
             "window statistic must be sum, mean, min or max");
  XC_REQUIRE(stat >= XC_STAT_SUM && stat <= XC_STAT_COUNT, "unknown reduction %d", stat);
  RollPlan pl;
  if (int32_t e = plan_rolling(C, ldx, aligned16(x), aligned16(out), window, window_stat, center, stat, &pl)) return e;
  if (pl.family == kRollingSumw) {
    const int32_t is_mean = (window_stat == XC_STAT_MEAN) ? 1 : 0, shift = center ? window / 2 : 0;
    return dispatch_register_window(pl.window, [&](auto WC) {
      return launch_rolling_sumw<decltype(WC)::value>(x, T, C, ldx, period_offsets, P, pl.arg, is_mean, shift, stat,
                                                      out, (cudaStream_t)stream);
    });
  }
  if (pl.family == kRollingReduce4) {
    const size_t smem = (size_t)window * kThreads * 16;
    if (smem > 48 * 1024)
      XC_CHECK_CUDA(cudaFuncSetAttribute(rolling_period_reduce4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
    dim3 grid4((unsigned)((C / 4 + kThreads - 1) / kThreads), (unsigned)P, 1);
    rolling_period_reduce4_kernel<<<grid4, kThreads, smem, (cudaStream_t)stream>>>(
        x, T, C, ldx, period_offsets, window, window_stat, center ? window / 2 : 0, stat, out);
    return launch_status("rolling_period_reduce4_kernel");
  }
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P, 1);
  rolling_period_reduce_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(
      x, T, C, ldx, period_offsets, window, window_stat, center ? window / 2 : 0, stat, out);
  return launch_status("rolling_period_reduce_kernel");
}

extern "C" int32_t xc_spell_sum_interval(int32_t op, double thr, int32_t window, int32_t window_stat, double* lo,
                                         double* hi, int32_t* out4) {
  XC_REQUIRE(lo && hi && out4, "null pointer argument");
  XC_REQUIRE(op >= XC_OP_GT && op <= XC_OP_NE, "Operation `%d` not recognized.", op);
  XC_REQUIRE(window >= 1 && (window_stat == XC_STAT_SUM || window_stat == XC_STAT_MEAN),
             "window statistic must be sum or mean");
  const SumRange g = make_sum_range(op, (float)thr, window, window_stat == XC_STAT_MEAN);
  *lo = g.lo;
  *hi = g.hi;
  out4[0] = g.hi_unbounded;
  out4[1] = g.negate;
  out4[2] = g.nan_cond;
  out4[3] = 0;
  return XC_OK;
}

extern "C" int32_t xc_spell_runstat_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                        const int32_t* period_offsets, int32_t P, int32_t window,
                                        int32_t window_stat, int32_t op, double thr, int32_t reducer,
                                        int32_t resample_before_rl, float* out, void* stream) {
  XC_REQUIRE(x && period_offsets && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1 && window <= T, "window must be in [1, T]");
  XC_REQUIRE(window_stat == XC_STAT_SUM || window_stat == XC_STAT_MEAN || window_stat == XC_STAT_MIN ||
                 window_stat == XC_STAT_MAX,
             "window reducer must be sum, mean, min or max");
  XC_REQUIRE(op >= XC_OP_GT && op <= XC_OP_NE, "Operation `%d` not recognized.", op);
  XC_REQUIRE(reducer >= XC_RL_MAX && reducer <= XC_RL_STD, "unknown run-length reducer %d", reducer);
  const RollPlan pl = plan_spell(C, ldx, aligned16(x), aligned16(out), window, window_stat, reducer,
                                 resample_before_rl == 0);
  if (pl.family == kSpellSumw) {
    const SumRange g = make_sum_range(op, (float)thr, window, window_stat == XC_STAT_MEAN);
    return dispatch_register_window(pl.window, [&](auto WC) {
      constexpr int W = decltype(WC)::value;
      return pl.after ? launch_spell_sumw<W, true>(x, T, C, ldx, period_offsets, P, g, pl.arg, reducer, out,
                                                   (cudaStream_t)stream)
                      : launch_spell_sumw<W, false>(x, T, C, ldx, period_offsets, P, g, pl.arg, reducer, out,
                                                    (cudaStream_t)stream);
    });
  }
  if (pl.family == kSpellRunstat4) {
    const size_t smem = (size_t)window * kThreads * 16;
    dim3 grid4((unsigned)((C / 4 + kThreads - 1) / kThreads), (unsigned)P, 1);
    auto go = [&](auto AFTC) -> int32_t {
      auto kernel = spell_runstat4_kernel<decltype(AFTC)::value>;
      if (int32_t e = allow_smem(kernel, smem, "cudaFuncSetAttribute(spell_runstat4_kernel)")) return e;
      kernel<<<grid4, kThreads, smem, (cudaStream_t)stream>>>(x, T, C, ldx, period_offsets, window, window_stat, op,
                                                              (float)thr, reducer, out);
      return launch_status("spell_runstat4_kernel");
    };
    return !pl.after ? go(std::false_type{}) : go(std::true_type{});
  }
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P, 1);
  spell_runstat_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(x, T, C, ldx, period_offsets, window,
                                                                    window_stat, op, (float)thr, reducer,
                                                                    pl.after ? 1 : 0, out);
  return launch_status("spell_runstat_kernel");
}

extern "C" int32_t xc_spell_mask_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t window,
                                     int32_t window_stat, int32_t op, double thr, const uint8_t* keep,
                                     int32_t drop_nan_adjacent, float* out_mask, void* stream) {
  XC_REQUIRE(x && out_mask, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1 && window <= T, "window must be in [1, T]");
  XC_REQUIRE(window_stat == XC_STAT_SUM || window_stat == XC_STAT_MEAN || window_stat == XC_STAT_MIN ||
                 window_stat == XC_STAT_MAX,
             "window reducer must be sum, mean, min or max");
  XC_REQUIRE(op >= XC_OP_GT && op <= XC_OP_NE, "Operation `%d` not recognized.", op);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), 1, 1);
  spell_mask_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(x, T, C, ldx, window, window_stat, op, (float)thr,
                                                                 keep, drop_nan_adjacent, out_mask);
  return launch_status("spell_mask_kernel");
}

extern "C" int32_t xc_rolling_period_reduce_sel_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                                    const int32_t* period_offsets, int32_t P, int32_t window,
                                                    int32_t window_stat, int32_t center, int32_t stat,
                                                    const uint8_t* keep, float* out, void* stream) {
  XC_REQUIRE(x && period_offsets && out && keep, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1 && window <= T, "window must be in [1, T]");
  XC_REQUIRE(window_stat == XC_STAT_SUM || window_stat == XC_STAT_MEAN || window_stat == XC_STAT_MIN ||
                 window_stat == XC_STAT_MAX,
             "window statistic must be sum, mean, min or max");
  XC_REQUIRE(stat >= XC_STAT_SUM && stat <= XC_STAT_COUNT, "unknown reduction %d", stat);
  if (center && window % 2 == 0) {
    set_error("centred rolling windows of even length are not supported");
    return XC_ERR_UNSUPPORTED;
  }
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P, 1);
  rolling_period_reduce_sel_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(
      x, T, C, ldx, period_offsets, window, window_stat, center ? window / 2 : 0, stat, keep, out);
  return launch_status("rolling_period_reduce_sel_kernel");
}
