/*
 * xclim_b200 -- C ABI of the H100 (sm_90a) per-grid-cell time-series kernels.
 *
 * This is the drop-in boundary for ONE hot path of Ouranosinc/xclim (reference @ a8cbec8c):
 * the per-cell reductions behind `xclim.indices.run_length`, `xclim.indices.generic`,
 * `xclim.core.calendar.percentile_doy` (+ bootstrap) and sdba empirical quantile mapping.
 * The reference is pure Python (no FFI); a maintainer binds these symbols with `ctypes`
 * (INTEGRATION.md shows the stub).  Each entry point cites the reference interface it
 * replaces as `file:line` relative to /root/reference/src/xclim.
 *
 * Conventions
 *   - All array arguments are DEVICE pointers unless the name ends in `_host`.
 *   - Gridded inputs are `(time, cell)` row-major float32: element (t, c) at x[t*ldx + c],
 *     where `cell` is the flattened `(lat, lon)` index (the reference's (time, lat, lon)
 *     C-contiguous layout has ldx == C == lat*lon).
 *   - `period_offsets` is an int32 device array of P+1 boundaries produced by
 *     `resample(time=freq)`: period p covers time steps [off[p], off[p+1]).
 *   - `doy_index` is an int16 device array of length T holding `time.dt.dayofyear` (1-based).
 *   - Every call is asynchronous on `stream` (a cudaStream_t passed as void*; NULL = legacy
 *     default stream) on the CURRENT device; the library allocates nothing, keeps no global
 *     mutable state and is re-entrant (one host thread or process per GPU).
 *   - Return value: 0 on success, negative XC_ERR_* otherwise; `xc_last_error()` returns a
 *     thread-local message.  Nothing throws across the boundary.
 */
#ifndef XCLIM_B200_H
#define XCLIM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XC_VERSION 100

/* status codes */
#define XC_OK 0
#define XC_ERR_INVALID (-1)  /* bad argument (ValueError in the reference) */
#define XC_ERR_UNSUPPORTED (-2) /* NotImplementedError in the reference */
#define XC_ERR_CUDA (-3)     /* CUDA runtime error, see xc_last_error() */

/* comparison operators: indices/generic.py:255-326 (`binary_ops`, `get_op`, `compare`) */
#define XC_OP_GT 0
#define XC_OP_LT 1
#define XC_OP_GE 2
#define XC_OP_LE 3
#define XC_OP_EQ 4
#define XC_OP_NE 5
/* NaN tests (threshold ignored), accepted by xc_period_count_f32 / xc_period_runstat_f32 only:
 * the `~valid` / `valid` masks of core/missing.py:253-298, 434-450 (MissingWMO's longest NaN run) */
#define XC_OP_ISNAN 6
#define XC_OP_NOTNAN 7

/* run-length reducers over the run lengths >= window attributed to a period:
 * indices/run_length.py:275-335 (`rle_statistics`, `get_rl_stat`), 381-488
 * (`windowed_run_events` == COUNT, `windowed_run_count` == SUM). */
#define XC_RL_MAX 0
#define XC_RL_MIN 1
#define XC_RL_SUM 2
#define XC_RL_COUNT 3
#define XC_RL_MEAN 4
#define XC_RL_STD 5

/* resample reductions: indices/generic.py:83-125 (`select_resample_op`) */
#define XC_STAT_SUM 0
#define XC_STAT_MEAN 1
#define XC_STAT_MIN 2
#define XC_STAT_MAX 3
#define XC_STAT_STD 4
#define XC_STAT_VAR 5
#define XC_STAT_COUNT 6

/* element transforms fused into xc_period_reduce_f32 */
#define XC_TF_NONE 0
#define XC_TF_EXCESS 1  /* (x - thr).clip(0) for >,>= ; (thr - x).clip(0) for <,<= : generic.py:1514-1552 */
#define XC_TF_WHERE 2   /* x where (x op thr) else NaN: generic.py:1278-1320 (`thresholded_statistics`) */

/* per-replacement indices of xc_bootstrap_doy_index_f32 */
#define XC_BOOT_COUNT 0  /* days_over_precip_thresh: indices/_multivariate.py:1174-1233 */
#define XC_BOOT_SPELL 1  /* warm / cold spell duration index: indices/_multivariate.py:69-153, 1719-1795 */
#define XC_BOOT_SUM 2    /* fraction_over_precip_thresh: indices/_multivariate.py:1238-1297 */

int32_t xc_version(void);
const char* xc_last_error(void);

/* Device properties the host side sizes its launches with (no reference counterpart). */
int32_t xc_device_sm_count(int32_t* out_sm_count);

/* ---------------------------------------------------------------------------------------------
 * a1+a2  threshold_count  -- indices/generic.py:329-361 (+ domain_count 364-392 via two calls)
 *   out[p, c] = #{ t in period p : x[t, c] op thr }   (NaN compares False)
 *   thr is a double; cmp_f64 == 0 reproduces numpy>=2 `float32_array op python_float`
 *   (comparison in float32 against float(thr)); cmp_f64 == 1 reproduces a float64 threshold.
 *   valid_count (optional, may be NULL): number of non-NaN steps per period (the fused
 *   MissingAny input, core/missing.py:296-298, 318-322).
 * ------------------------------------------------------------------------------------------- */
int32_t xc_period_count_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                            const int32_t* period_offsets, int32_t P,
                            int32_t op, double thr, int32_t cmp_f64,
                            int32_t* out_count, int32_t* valid_count, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a6-a11  run-length statistics of the condition (x op thr)
 *   replaces  generic._spell_length_statistics (window==1)   indices/generic.py:543-585
 *             run_length.resample_and_rl                      indices/run_length.py:87-132
 *             run_length.rle / rle_statistics / longest_run   indices/run_length.py:223-378
 *             run_length.windowed_run_count / _events         indices/run_length.py:381-488
 *   resample_before_rl != 0: runs are cut at period edges (run_length.py:122-129);
 *   resample_before_rl == 0: runs are found on the whole series and attributed, with their full
 *   length, to the period holding their first element (run_length.py:318, 329-334).
 *   out[p, c] (float32) = reducer over run lengths >= window, 0 when there is none.
 * ------------------------------------------------------------------------------------------- */
int32_t xc_period_runstat_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                              const int32_t* period_offsets, int32_t P,
                              int32_t op, double thr, int32_t cmp_f64,
                              int32_t reducer, int32_t window, int32_t resample_before_rl,
                              float* out, int32_t* valid_count, void* stream);

/* The same statistics (runs cut at period edges) on the mask with holes filled: spells separated
 * by fewer than min_gap non-spell steps are merged -- generic.spell_mask(min_gap > 1)
 * (indices/generic.py:537-538) = run_length.runs_with_holes(m, 1, ~m, min_gap)
 * (indices/run_length.py:844-888), including its rule that a short gap running into the end of
 * the series is bridged while a gap that starts the series is not.  window == 1 masks only. */
int32_t xc_period_runstat_gap_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                  const int32_t* period_offsets, int32_t P,
                                  int32_t op, double thr, int32_t cmp_f64,
                                  int32_t reducer, int32_t window, int32_t min_gap,
                                  float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a6 (bivariate)  run statistics / counts of a condition on two variables:
 *   cond = (x1 op1 thr1) AND|OR (x2 op2 thr2)  -> reducer over run lengths >= window per period.
 *   replaces heat_wave_frequency / _max_length / _total_length (indices/_multivariate.py:646-880),
 *   tx_tn_days_above (:1653-1716; reducer SUM, window 1 == count) and
 *   generic.bivariate_count_occurrences (indices/generic.py:1002-1073; var_any != 0 for "any").
 * ------------------------------------------------------------------------------------------- */
int32_t xc_period_runstat2_f32(const float* x1, const float* x2, int64_t T, int64_t C, int64_t ldx,
                               const int32_t* period_offsets, int32_t P,
                               int32_t op1, double thr1, int32_t op2, double thr2, int32_t var_any,
                               int32_t reducer, int32_t window, int32_t resample_before_rl,
                               float* out, void* stream);

/* a10 (cont.)  quantile reducers ("q90", "q10", ...) of rle_statistics -- indices/run_length.py:320-327
 *   with reducer "quantile": numpy's linear quantile q of the run lengths >= window attributed to the
 *   period, 0 when there is none.  period_offsets_host mirrors period_offsets (run-list sizing). */
int32_t xc_period_run_quantile_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                   const int32_t* period_offsets, const int32_t* period_offsets_host, int32_t P,
                                   int32_t op, double thr, int32_t cmp_f64, double q,
                                   int32_t window, int32_t resample_before_rl, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a11  windowed_max_run_sum of the excess over a threshold -- indices/run_length.py:491-540 on
 *   `(x - thr).clip(0)` (indices/_threshold.py:2064-2073, `hot_spell_max_magnitude`): per period the
 *   largest sum of (x - thr) (op >, >=; thr - x for <, <=) over a run at least `window` long.
 * ------------------------------------------------------------------------------------------- */
int32_t xc_period_run_maxsum_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                 const int32_t* period_offsets, int32_t P,
                                 int32_t op, double thr, int32_t window, int32_t resample_before_rl,
                                 float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a12  first / last run of at least `window` steps of the condition (x op thr), per period
 *   replaces run_length._boundary_run / first_run / last_run (indices/run_length.py:543-740,
 *   general branches with `freq`).  out[p, c] (float32) = index, relative to the period start, of
 *   the first element of the first run (position_last == 0) or of the last element of the last
 *   run (position_last != 0); NaN when there is none.  window == 1 keeps the reference's
 *   argmax == argmin rule (:603-605): an all-True period also gives NaN.
 * ------------------------------------------------------------------------------------------- */
int32_t xc_period_boundary_run_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                   const int32_t* period_offsets, int32_t P,
                                   int32_t op, double thr, int32_t cmp_f64,
                                   int32_t window, int32_t position_last, float* out, void* stream);

/* a12 (cont.)  runs confined to a per-period sub-range: the per-group calls of
 *   run_length.first_run_after_date / last_run_before_date / first_run_before_date /
 *   run_end_after_date (indices/run_length.py:1148-1331) and the two steps of run_length.season
 *   (:998-1110).  Period p is searched on [range_lo[p], range_hi[p]) (absolute steps; range_lo < 0:
 *   the date is not in the group -> NaN); negate != 0 runs on NOT(x op thr) (season end, `~da`);
 *   cell_lo (optional (P, C) float32, relative to the period start, NaN -> 0) raises the lower
 *   bound per cell (`index >= beg.fillna(0)`, :977).  out as xc_period_boundary_run_f32. */
int32_t xc_period_boundary_run_range_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                         const int32_t* period_offsets, const int32_t* range_lo,
                                         const int32_t* range_hi, int32_t P,
                                         int32_t op, double thr, int32_t cmp_f64, int32_t negate,
                                         int32_t window, int32_t position_last,
                                         const float* cell_lo, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a3  per-period reductions -- indices/generic.py:83-125 (`select_resample_op`), 1255-1320
 *   (`statistics`, `thresholded_statistics`), 1514-1552 (`cumulative_difference`); _simple.py:113
 *   NaN steps are skipped (xarray skipna); an all-NaN period gives NaN (0 for SUM, COUNT).
 *   Accumulation is in float64, results are rounded once to float32.
 * ------------------------------------------------------------------------------------------- */
int32_t xc_period_reduce_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                             const int32_t* period_offsets, int32_t P,
                             int32_t stat, int32_t transform, int32_t op, double thr,
                             float* out, int32_t* valid_count, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a4  rolling window then per-period reduction -- indices/generic.py:128-174
 *   (`select_rolling_resample_op`), _simple.py:485-525 (`max_n_day_precipitation_amount`).
 *   window_stat in {SUM, MEAN, MIN, MAX}; right-aligned (center == 0) or centred window,
 *   min_periods == window (NaN for incomplete windows or windows holding a NaN); then `stat`.
 * ------------------------------------------------------------------------------------------- */
int32_t xc_rolling_period_reduce_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                     const int32_t* period_offsets, int32_t P,
                                     int32_t window, int32_t window_stat, int32_t center,
                                     int32_t stat, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a5+a6  spell statistics for spells defined by a rolling window (window > 1)
 *   replaces generic.spell_mask (indices/generic.py:434-540: a step is in a spell iff it belongs
 *   to at least one block of `window` consecutive steps, fully inside the series, whose
 *   window_stat (sum/mean/min/max, NaN if the block holds a NaN) satisfies `op thr`) followed by
 *   generic._spell_length_statistics (:543-585: run statistics of that mask per period with
 *   window 1).  thr is compared in float32 (Python-float threshold).  out (P, C) float32.
 * ------------------------------------------------------------------------------------------- */
int32_t xc_spell_runstat_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                             const int32_t* period_offsets, int32_t P,
                             int32_t window, int32_t window_stat, int32_t op, double thr,
                             int32_t reducer, int32_t resample_before_rl, float* out, void* stream);

/* The same with `select_time` applied to the ROLLED series -- indices/generic.py:169-174
 * (`select_resample_op(rolled, op=op, freq=freq, **indexer)`): only the windows whose label t has
 * keep[t] != 0 (device uint8[T]) enter the per-period reduction. */
int32_t xc_rolling_period_reduce_sel_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                         const int32_t* period_offsets, int32_t P, int32_t window,
                                         int32_t window_stat, int32_t center, int32_t stat,
                                         const uint8_t* keep, float* out, void* stream);

/* The spell mask itself, with `select_time` applied to it -- indices/generic.py:503-535 + 557-558
 * (`is_in_spell = select_time(spell_mask(...), **indexer)`): out_mask (T, C) float32 = NaN where
 * keep[t] == 0, else 1 / 0 (day t is / is not covered by a qualifying length-`window` block of the
 * UNMASKED series).  keep (device uint8[T], NULL = keep all): 0 out of season, 1 in season, 2 first
 * in-season day after a masked one inside a resampling group; drop_nan_adjacent != 0 zeroes the runs that
 * start on a `2` day (the whole-array `rle` of run_length.py:264), 0 counts them with their in-season
 * length (the per-series path, pinned by tests/test_indices.py:4116-4126).  Feed the mask to
 * xc_period_runstat_f32 with op `>` 0. */
int32_t xc_spell_mask_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t window,
                          int32_t window_stat, int32_t op, double thr, const uint8_t* keep,
                          int32_t drop_nan_adjacent, float* out_mask, void* stream);

/* Host-side helper of the entry point above (no device work; exported so that it can be tested
 * without a GPU): for sum / mean windows the kernels compare the float64 window SUM s instead of
 * the float32 statistic r(s) = (float)(s) or (float)(s / window).  r is monotone in s, hence
 *   r(s) op (float)thr   <=>   ((s >= lo) && (hi_unbounded || s < hi)) != negate
 * for the interval this function finds by bisection over the ordered doubles (window_stat is
 * XC_STAT_SUM or XC_STAT_MEAN).  out4 = {hi_unbounded, negate, value of (NaN op thr), 0}. */
int32_t xc_spell_sum_interval(int32_t op, double thr, int32_t window, int32_t window_stat,
                              double* lo, double* hi, int32_t* out4);

/* ---------------------------------------------------------------------------------------------
 * a14+a15  percentile_doy -- core/calendar.py:395-494 with the quantile of
 *   core/utils.py:279-557 (`calc_perc` -> `_nan_quantile`, Hyndman-Fan alpha/beta).
 *   x: (T, C) float32 base-period series (device).  doy_index_host / year_index_host: HOST int16
 *   arrays (T) with the 1-based day-of-year and the 0-based year ordinal of every step (tiny
 *   calendar metadata, read synchronously during the call); n_doy = max day-of-year present;
 *   n_years = number of distinct years; window must be odd.
 *   out: (n_per, n_doy, C) float64 (device), i.e. the reference's (lat, lon, dayofyear,
 *   percentiles) table stored doy-major so that it is coalesced along cells.  The 366 -> 1..366
 *   re-interpolation of core/calendar.py:484-485 is xc_doy_interp_f64 (separate, tiny).
 *   Percentiles whose order statistics lie more than 64 ranks from both ends of the sample (the
 *   median of 30 x 5 values ...) run through a slower exact selection kernel (samples of up to
 *   768 values per day; larger ones are rejected with XC_ERR_UNSUPPORTED).
 *   workspace: device scratch of xc_percentile_doy_workspace_bytes() bytes.
 * ------------------------------------------------------------------------------------------- */
int64_t xc_percentile_doy_workspace_bytes(int64_t T, int64_t C, int32_t n_doy, int32_t n_years,
                                          int32_t window, int32_t n_per);
int32_t xc_percentile_doy_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                              const int16_t* doy_index_host, const int16_t* year_index_host,
                              int32_t n_doy, int32_t n_years, int32_t window,
                              const double* percentiles_host, int32_t n_per,
                              double alpha, double beta,
                              double* out, void* workspace, int64_t workspace_bytes, void* stream);

/* The same with a virtual-row map (bootstrap on calendars with leap years, core/bootstrapping.py:
 * 235-282): the series keeps its time axis (doy / year labels) but the VALUE of step t is read
 * from row vrow_host[t] (HOST int32[T]; -1 = missing, i.e. NaN).  Replacing the block of one year
 * by the (calendar-converted) block of another year is such a map, so no copy of the input is
 * made.  Workspace: xc_percentile_doy_workspace_bytes. */
int32_t xc_percentile_doy_vrow_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                   const int16_t* doy_index_host, const int16_t* year_index_host,
                                   const int32_t* vrow_host, int32_t n_doy, int32_t n_years,
                                   int32_t window, const double* percentiles_host, int32_t n_per,
                                   double alpha, double beta, double* out, void* workspace,
                                   int64_t workspace_bytes, void* stream);

/* Test hook: same contract as xc_percentile_doy_f32 for ONE percentile, but always through the
 * generic (any-calendar) kernel, so the fast uniform-year kernel can be checked against it. */
int32_t xc_percentile_doy_generic_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                      const int16_t* doy_index_host, const int16_t* year_index_host,
                                      int32_t n_doy, int32_t n_years, int32_t window, double percentile,
                                      double alpha, double beta, double* out, void* workspace,
                                      int64_t workspace_bytes, void* stream);

/* core/calendar.py:690-726 (`_interpolate_doy_calendar`): table (n_src, C) float64 on doys
 * linspace(doy_min, doy_max, n_src) -> (doy_max - doy_min + 1, C) by linear interpolation
 * (NaN entries along doy are first filled by linear interpolation of their neighbours). */
int32_t xc_doy_interp_f64(const double* table, int32_t n_src, int64_t C,
                          int32_t doy_min, int32_t doy_max, double* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a16+a2  percentile-threshold count -- indices/_multivariate.py:1583-1590 (`tx90p` & family),
 *   core/calendar.py:763-790 (`resample_doy` as an index into the table instead of a
 *   materialised (lat, lon, time) float64 array), generic.py:357-361.
 *   out[p, c] = #{ t in p : (double)x[t, c] op table[doy_index[t]-1, c] }  (float64 compare)
 * ------------------------------------------------------------------------------------------- */
int32_t xc_doy_threshold_count_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                   const int32_t* period_offsets, int32_t P,
                                   const int16_t* doy_index, const double* table, int32_t n_doy,
                                   int32_t op, int32_t* out_count, int32_t* valid_count,
                                   void* stream);

/* Same count for the common layout "n_years whole years of year_len steps starting at first_row,
 * day-of-year == position in the year" (noleap / 360_day with freq YS): out[y, c] for y < n_years.
 * Year-blocked so that each table row is read once per 3 years; needs C, ldx % 4 == 0 and 16-byte
 * aligned buffers (use xc_doy_threshold_count_f32 otherwise). */
int32_t xc_doy_threshold_count_years_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                         int64_t first_row, int32_t n_years, int32_t year_len,
                                         const double* table, int32_t op,
                                         int32_t* out_count, int32_t* valid_count, void* stream);

/* ---------------------------------------------------------------------------------------------
 * d1  the remaining ETCCDI day-of-year percentile indices.  Every comparison against a table is in
 *   float64 (the reference's `resample_doy` array), the threshold of step t being
 *   table[(doy_index[t] - 1) * C + c] as for xc_doy_threshold_count_f32.
 * ------------------------------------------------------------------------------------------- */
/* Run statistic of `x op table[doy]` per period, as xc_period_runstat_f32 (reducer, window,
 * resample_before_rl, valid_count): warm_spell_duration_index / cold_spell_duration_index
 * (indices/_multivariate.py:69-153, 1719-1795: rl.windowed_run_count == XC_RL_SUM).  op is one of
 * > < >= <=. */
int32_t xc_doy_runstat_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                           const int32_t* period_offsets, int32_t P,
                           const int16_t* doy_index, const double* table, int32_t n_doy,
                           int32_t op, int32_t reducer, int32_t window, int32_t resample_before_rl,
                           float* out, int32_t* valid_count, void* stream);

/* The two sums of fraction_over_precip_thresh (indices/_multivariate.py:1238-1297) from one read of x:
 *   out_sum_thr[p, c] = sum of x[t, c] over t in p with (double)x op thr[row(t) * thr_rstride + c],
 *   out_sum_wet[p, c] = sum of x[t, c] over t in p with x op (float)wet,
 * row(t) = doy_index[t] - 1, or t when doy_index is NULL (thr_rstride = 0: one threshold per cell).
 * Sums are float64 in time order, rounded once to float32.  op is > or >=. */
int32_t xc_period_sums_thr_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                               const int32_t* period_offsets, int32_t P, const int16_t* doy_index,
                               const double* thr, int64_t thr_rstride, int32_t op, double wet,
                               float* out_sum_thr, float* out_sum_wet, void* stream);

/* Days with (x1 op1 table1[doy]) AND (x2 op2 table2[doy]) per period (float32 counts): the compound
 * percentile days cold_and_dry_days ... cold_and_wet_days (indices/_multivariate.py:162-416).
 * x1, x2 share (T, C, ldx); both tables are (n_doy, C); op1, op2 are > < >= <=. */
int32_t xc_doy_count2_f32(const float* x1, const float* x2, int64_t T, int64_t C, int64_t ldx,
                          const int32_t* period_offsets, int32_t P, const int16_t* doy_index,
                          const double* table1, const double* table2, int32_t n_doy,
                          int32_t op1, int32_t op2, float* out, void* stream);

/* Per-period statistic `stat` (XC_STAT_*, NaN skipped) of d[t] = hi[t] - lo[t] in float32:
 * daily_temperature_range (indices/_multivariate.py:514-557).  variability != 0: the mean of
 * |d[t] - d[t-1]| over the steps t >= 1 of the period (the first one reaches into the previous
 * period), daily_temperature_range_variability (:561-598); stat must then be XC_STAT_MEAN. */
int32_t xc_period_range_stat_f32(const float* lo, const float* hi, int64_t T, int64_t C, int64_t ldx,
                                 const int32_t* period_offsets, int32_t P, int32_t stat,
                                 int32_t variability, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a17  percentile bootstrap (Zhang 2005) -- core/bootstrapping.py:81-211, 235-282
 *   x: (T, C) studied series; the base (climatology) period is the n_base_years equal-length
 *   year blocks of year_len steps starting at row base_start (noleap / 360_day calendars,
 *   core/bootstrapping.py:264-265; 365<->366 block conversion is not supported).
 *   step_period: device int32[n_base_years*year_len], output period index of every base step
 *   (periods nest in years: freq YS/QS/MS...).  For every period p holding steps of in-base
 *   year y:
 *     out[p, c] = mean over base years s != y of #{ t in p : (double)x[t] op P^(y<-s)[doy(t)] }
 *   where P^(y<-s) = percentile_doy(window, percentile, alpha, beta) of the base series with
 *   block y replaced by block s.  out is (P, C) float64 and is written for ALL p (periods without
 *   base steps get 0: the caller fills them with xc_doy_threshold_count_f32, bootstrapping.py:205-207).
 *   count_scratch: device int32 (P, C).
 * ------------------------------------------------------------------------------------------- */
int32_t xc_bootstrap_doy_count_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                   int64_t base_start, int32_t n_base_years, int32_t year_len,
                                   const int32_t* step_period, int32_t P,
                                   int32_t window, double percentile, double alpha, double beta,
                                   int32_t op, int32_t* count_scratch, double* out, void* stream);

/* The same bootstrap for the indices whose value depends on the ORDER of the exceedance days or on the values
 * over the threshold -- `percentile_bootstrap` on warm_spell_duration_index, cold_spell_duration_index,
 * days_over_precip_thresh and fraction_over_precip_thresh (indices/_multivariate.py:69-153, 1174-1297, 1719-1795;
 * core/bootstrapping.py:81-211, 235-282).  For every in-base year y and base year s != y the bootstrap kernel
 * writes year y's exceedance mask against max(P^(y<-s), floor) (a NaN percentile takes the floor:
 * `pr_per.where(pr_per > thresh, thresh)`, :1222, 1288; floor = -inf: no floor, a NaN percentile is never
 * exceeded), then one lane per (cell, y) computes the index on year y's own slice for each s and averages:
 *   XC_BOOT_COUNT: out float64 (P, C), mean over s of the days over the threshold;
 *   XC_BOOT_SPELL: out float64 (P, C), mean over s of rl.windowed_run_count(mask, run_window) per period
 *                  (resample_before_rl as in xc_doy_runstat_f32; runs end at the edges of year y);
 *   XC_BOOT_SUM:   out float32 (P, C), mean over s of float32(float64 time-order sum of x over the mask days)
 *                  / wet_total[p, c] (float32 (P, C), row stride C): the float64 sum of the non-NaN float32
 *                  fractions in s order over their number, rounded once to float32; NaN when all are NaN.
 * Only periods holding base steps are written.  floor is only accepted with > / >=.
 * step_period must keep every period inside one base year (the periods nest in the years: one lane per (cell,
 * year) writes a period's result); a period spanning two years is not detected and gives undefined results.
 * scratch: device memory of scratch_bytes bytes, 16-byte aligned.  The cells are processed in tiles of as many
 * cells as it holds masks for (xc_bootstrap_doy_index_scratch_bytes(N, L, C) bytes: all of them); a tile smaller
 * than the C and than 128 cells is XC_ERR_INVALID.  On return the scratch holds the last tile's masks,
 * uint32 [(pair * ceil(L / 32) + d / 32) * n + c], pair = y (N - 1) + (s < y ? s : s - 1), n its cells. */
int64_t xc_bootstrap_doy_index_scratch_bytes(int32_t n_base_years, int32_t year_len, int64_t C);
int32_t xc_bootstrap_doy_index_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                   int64_t base_start, int32_t n_base_years, int32_t year_len,
                                   const int32_t* step_period, int32_t P,
                                   int32_t window, double percentile, double alpha, double beta, int32_t op,
                                   int32_t reducer, int32_t run_window, int32_t resample_before_rl, double floor,
                                   const float* wet_total, void* scratch, int64_t scratch_bytes, void* out,
                                   void* stream);

/* ---------------------------------------------------------------------------------------------
 * a20  empirical quantile mapping -- xsdba.EmpiricalQuantileMapping (third-party, re-exported
 *   by sdba.py:11; call sites tests/test_xsdba.py:21-34, 143-150).  group="time".
 *   train : af, hist_q (nq, C) float32 from ref, hist (T, C); kind 0 = "+", 1 = "*".
 *   adjust: scen (T, C) from sim (T, C); interp 0 = nearest, 1 = linear; constant extrapolation.
 * ------------------------------------------------------------------------------------------- */
int64_t xc_eqm_train_workspace_bytes(int64_t T, int64_t C, int32_t nq);
int32_t xc_eqm_train_f32(const float* ref, const float* hist, int64_t T, int64_t C, int64_t ldx,
                         int32_t nq, int32_t kind, float* af, float* hist_q,
                         void* workspace, int64_t workspace_bytes, void* stream);
int32_t xc_eqm_adjust_f32(const float* sim, int64_t T, int64_t C, int64_t ldx,
                          const float* af, const float* hist_q, int32_t nq,
                          int32_t kind, int32_t interp, float* scen, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a20 (cont.)  quantile delta mapping -- xsdba.QuantileDeltaMapping (third-party, re-exported by
 *   sdba.py:11; its train step is EmpiricalQuantileMapping.train, i.e. xc_eqm_train_f32).
 *   group="time", extrapolation="constant".  Per cell of sim (T, C):
 *     sim_q = percentage rank of sim within the cell's whole series (average ranks of ties over the
 *             n valid values, p = r / n, then (mx * (p - mn)) / (mx - mn) with mn / mx the min / max
 *             of p; float64; NaN where sim is NaN or the cell has fewer than two distinct values);
 *     scen  = sim (+|*) interp(sim_q; nodes -> af) in float32, af entries that are NaN dropped,
 *             interp 0 = nearest (ties to the lower node), 1 = linear, constant end factors.
 *   nodes: device float32[nq], the quantile nodes of af (equally_spaced_nodes(nq) as float32).
 *   af: (nq, C) float32 with leading dimension C.  sim_q: (T, C) float64 or NULL.
 *   workspace: device scratch; any size >= xc_qdm_adjust_workspace_bytes(T, 32) works (the cells are
 *   processed in chunks that fit), xc_qdm_adjust_workspace_bytes(T, C) processes all cells at once.
 *   T <= 32768 (longer series return XC_ERR_UNSUPPORTED).
 * ------------------------------------------------------------------------------------------- */
int64_t xc_qdm_adjust_workspace_bytes(int64_t T, int64_t C);
int32_t xc_qdm_adjust_f32(const float* sim, int64_t T, int64_t C, int64_t ldx,
                          const float* af, const float* nodes, int32_t nq, int32_t kind, int32_t interp,
                          float* scen, double* sim_q, void* workspace, int64_t workspace_bytes,
                          void* stream);

/* ---------------------------------------------------------------------------------------------
 * a20 (cont.)  detrended quantile mapping -- xsdba.DetrendedQuantileMapping (third-party,
 *   re-exported by sdba.py:11; xsdba's dqm_train / dqm_adjust with PolyDetrend), group="time",
 *   extrapolation="constant"; and the polynomial trend of xclim.indices.generic.detrend
 *   (indices/generic.py:1711-1736: polyfit, then polyval).  kind 0 = "+", 1 = "*"; (+) is + or *,
 *   inv(m) is -m or float32(1 / m).
 *   train, per cell of ref, hist (T, C):
 *     m_ref, m_hist = NaN-skipping means (float64 sums over n, rounded once: xc_period_reduce_f32,
 *       one period, XC_STAT_MEAN); scaling[c] = m_ref - m_hist or m_ref / m_hist (float32);
 *     af, hist_q (nq, C) = xc_eqm_train_f32 of refn = float32(ref (+) inv(m_ref)) and histn (likewise),
 *       computed without a normalised copy of ref / hist.
 *     workspace: device scratch of at least xc_dqm_train_workspace_bytes(T, C, nq).  T <= 32768.
 *   trend of a series y with degree D in {0, 1, 2}: the least-squares polynomial over the valid steps
 *     in the basis u_t = (2t - (T - 1)) / max(T - 1, 1), float64; the degree is lowered to n - 1 for
 *     n <= D valid steps; all NaN for n = 0 or any infinite valid value.  coef (D + 1, C) float64,
 *     row k = the coefficient of u^k; tau_t = ((c2 u + c1) u + c0) without fused multiply-adds.
 *     xc_poly_fit_f32 fits y = x, or y = float32(x (+) scaling[c]) when scaling is not NULL.
 *   adjust, per cell of sim (T, C), coef = xc_poly_fit_f32(sim, kind, scaling):
 *     y = float32(sim (+) scaling); d = y - tau or y * (1 / tau) (float64);
 *     f = interp(d; hist_q -> af) over the entries where neither is NaN (interp 0 = nearest, ties to
 *       the lower node; 1 = linear, scipy interp1d's two-weight form), constant end factors, float32;
 *     scen = float32((d (+) f) (+) tau) with the inner operations in float64.
 *     nq in [2, 200]; no limit on T.
 *   detrend: out (T, C) float64 = x - tau, with coef = xc_poly_fit_f32(x, scaling = NULL); no limit on T.
 * ------------------------------------------------------------------------------------------- */
int64_t xc_dqm_train_workspace_bytes(int64_t T, int64_t C, int32_t nq);
int32_t xc_dqm_train_f32(const float* ref, const float* hist, int64_t T, int64_t C, int64_t ldx,
                         int32_t nq, int32_t kind, float* af, float* hist_q, float* scaling,
                         void* workspace, int64_t workspace_bytes, void* stream);
int32_t xc_poly_fit_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t degree, int32_t kind,
                        const float* scaling, double* coef, void* stream);
int32_t xc_dqm_adjust_f32(const float* sim, int64_t T, int64_t C, int64_t ldx, const float* af,
                          const float* hist_q, const float* scaling, const double* coef, int32_t nq,
                          int32_t kind, int32_t interp, int32_t degree, float* scen, void* stream);
int32_t xc_detrend_apply_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const double* coef,
                             int32_t degree, double* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Synthetic inputs (BASELINE.json configs; SURVEY.md section 8d).  Stateless counter-based
 * generators: value(t, global_cell) depends only on (seed, t, global_cell), so a lat tile
 * generated on any rank equals the same slab of the global grid.
 *   kind 0: pr in mm/d (10-day wet/dry regimes, exponential amounts, rare NaN blocks)
 *   kind 1: tasmax in K (latitudinal gradient, annual cycle, daily + weekly anomalies)
 * ------------------------------------------------------------------------------------------- */
int32_t xc_synth_f32(float* out, int64_t T, int64_t C, int64_t ldx, int64_t cell_offset,
                     int64_t cells_per_lat, int64_t n_lat_global, int32_t year_len,
                     int32_t kind, uint64_t seed, void* stream);

/* select_time(da, **indexer) with drop=False -- core/calendar.py:1259-1376: out[t, c] = keep[t] ? x[t, c] : NaN
 * (keep: device uint8[T] built on the host from season / month / doy_bounds / date_bounds). */
int32_t xc_mask_steps_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const uint8_t* keep,
                          float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Host-buffer entry points (the end-to-end path: host -> device copies inside the call).
 *   x_host: (T, C) float32 in (pinned or pageable) host memory; the call streams year-sized
 *   slabs through the caller's device workspace with double buffering, launches the same
 *   kernels per slab and copies the small outputs back.  Synchronous: returns when out_host is
 *   complete.  workspace_bytes >= xc_host_stream_workspace_bytes(...).
 * ------------------------------------------------------------------------------------------- */
int64_t xc_host_stream_workspace_bytes(int64_t T, int64_t C, const int32_t* period_offsets_host,
                                       int32_t P);
int32_t xc_period_runstat_f32_host(const float* x_host, int64_t T, int64_t C,
                                   const int32_t* period_offsets_host, int32_t P,
                                   int32_t op, double thr, int32_t cmp_f64,
                                   int32_t reducer, int32_t window,
                                   float* out_host, int32_t* valid_count_host,
                                   void* workspace, int64_t workspace_bytes);

/* threshold_count with an ARRAY threshold -- indices/generic.py:301-361 (`compare(da, op, threshold)` with a
 * DataArray threshold): out[p, c] = #{ t in period p : (double)x[t, c] op thr[t * thr_tstride + c] }, thr float64
 * (numpy promotes float32 data against a float64 array to float64); thr_tstride = 0: one threshold per cell. */
int32_t xc_period_count_arr_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                const int32_t* period_offsets, int32_t P, int32_t op,
                                const double* thr, int64_t thr_tstride, int32_t* out_count, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused multi-output pass (batch of indicators over ONE variable and ONE resampling frequency):
 * core/indicator.py:884-886 runs the indicators one after the other, each re-reading its input; here
 * every count / run-length / reduction output that shares (x, period_offsets) comes out of a single
 * streaming pass (SURVEY.md section 8d: "unique inputs once each").
 *   Conditions are normalised on the host to  sgn * x > thr  (x >= t  <=>  x > pred(t), x < t  <=>
 *   -x > -t, ...; indices/generic.py:301-326); runs are cut at the period edges
 *   (resample_before_rl=True, indices/run_length.py:122-129).
 *   cond[i]: n_true (threshold_count, generic.py:329-361) and the longest run (rle_statistics "max";
 *            a longest run shorter than `wmax` is reported as 0: `max_l.where(max_l >= window, 0)`,
 *            indices/_threshold.py:311)
 *   runs[k]: total length (kind 0, windowed_run_count) or number (kind 1, windowed_run_events) of the runs
 *            of condition k / 2 that are at least `window` long (run_length.py:381-488): the first
 *            n_runs / 2 conditions own two run outputs each (slot -1: unused), so that the kernel
 *            needs no indirection; `cond` must equal k / 2
 *   msum[0]: largest run sum of sgn * (x - thr0) over the runs of condition 0 at least `window` long
 *            (windowed_max_run_sum, run_length.py:491-540; hot_spell_max_magnitude); `cond` must be 0
 *   sums[k]: mode 0: sum of (off_sgn * (x - off)).clip(0) (cumulative_difference, generic.py:1514-1552);
 *            mode 1: sum of x where sgn * x > thr (thresholded_statistics "sum", generic.py:1278-1320)
 *   plain:   sum / mean / min / max of x (select_resample_op, generic.py:83-125)
 *   Every `slot` is an index into `out` (slot s occupies out[s*P*C .. (s+1)*P*C), 4-byte elements: int32
 *   for n_true, float32 otherwise) or -1 when that output is not wanted.  n_runs is even.  Needs C % 4 == 0,
 *   ldx % 4 == 0, 16-byte aligned buffers and T < 2^24 (counters and run lengths are float32).
 * ------------------------------------------------------------------------------------------- */
#define XC_MULTI_MAX_COND 6
#define XC_MULTI_MAX_RUNS 4
#define XC_MULTI_MAX_MSUM 1
#define XC_MULTI_MAX_SUMS 3
typedef struct { float sgn, thr; int32_t wmax, slot_n, slot_max; } XcMultiCond;
typedef struct { int32_t cond, window, kind, slot; } XcMultiRun;
typedef struct { int32_t cond, window; float sgn, thr0; int32_t slot; } XcMultiMaxSum;
typedef struct { float sgn, thr, off_sgn, off; int32_t mode, slot; } XcMultiSum;
typedef struct {
  int32_t n_cond, n_runs, n_msum, n_sums;
  XcMultiCond cond[XC_MULTI_MAX_COND];
  XcMultiRun runs[XC_MULTI_MAX_RUNS];
  XcMultiMaxSum msum[XC_MULTI_MAX_MSUM];
  XcMultiSum sums[XC_MULTI_MAX_SUMS];
  int32_t slot_sum, slot_mean, slot_min, slot_max;
} XcMultiPlan;
int32_t xc_period_multi_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                            const int32_t* period_offsets, int32_t P, const XcMultiPlan* plan_host,
                            void* out, int32_t n_slots, void* stream);

/* Percentile table layout change: (n_per, n_doy, C) doy-major (the kernels' coalesced layout) ->
 * (C, n_doy, n_per), the reference's `(*space, dayofyear, percentiles)` order of
 * core/calendar.py:479-483 (`.transpose(..., "dayofyear", "percentiles")`), on the device. */
int32_t xc_table_cell_major_f64(const double* table, int32_t n_per, int32_t n_doy, int64_t C,
                                double* out, void* stream);

/* Slab copy between a strided host box and device memory (either direction), asynchronous on
 * `stream`: `height` rows of `width_bytes`, row r at src + r*src_pitch -> dst + r*dst_pitch.
 * This is the unwrap step of the end-to-end path (core/indicator.py:884-886 hands host arrays to
 * the index function): a lat tile `x[:, r0:r1, :]` of a (time, lat, lon) host array is one such box
 * (width = rows*lon*4 bytes, height = time).  Pinned host memory is copied by the DMA engines
 * without staging; pageable memory is accepted.  to_device != 0: host -> device, else device -> host. */
int32_t xc_copy_box_async(void* dst, int64_t dst_pitch, const void* src, int64_t src_pitch,
                          int64_t width_bytes, int64_t height, int32_t to_device, void* stream);
/* 1 when host_ptr lies in page-locked (pinned / registered) host memory, 0 otherwise (pageable memory,
 * memory-mapped files: the slab streamer stages those through its own pinned buffers). */
int32_t xc_host_pinned(const void* host_ptr);

/* ---------------------------------------------------------------------------------------------
 * f4  Canadian Forest Fire Weather Index System -- indices/fire/_cffwis.py
 *   Replaces the day loop `_fire_weather_calc` (:680-873; the gufunc core of `fire_weather_ufunc`
 *   :879-1151, behind `cffwis_indices` :1273-1402, `drought_code` :1415-1500, `duff_moisture_code`
 *   :1513-1594) with its numba step functions (`_fine_fuel_moisture_code` :246-319,
 *   `_duff_moisture_code` :322-393, `_drought_code` :396-446, `_overwintering_drought_code` :549-583),
 *   the numpy indices (`initial_spread_index` :449-469, `build_up_index` :472-501,
 *   `fire_weather_index` :504-528, `daily_severity_rating` :531-546) and the season masks
 *   (`_fire_season` :590-677).  One lane walks one cell through time; every requested output is
 *   written in the same pass.
 *   Inputs (T, C) float32 with leading dimension ldx, units as `fire_weather_ufunc` takes them:
 *   tas degC, pr mm/day, hurs %, ws km/h, snd m (NULL where the requested codes / modes do not
 *   need them).  season_mask_in: (T, C) uint8, season_mode == XC_FWI_SEASON_MASK only.
 *   month: device int8[T] (1..12).  lat: device float64[C] (degrees north).
 *   dc0 / dmc0 / ffmc0 / winter_pr0: device float32[C] or NULL (= NaN, NaN, NaN, 0).
 *   Outputs: any of DC..DSR (T, C) float32, season_mask_out (T, C) uint8, winter_pr_out float32[C]
 *   may be NULL; codes an index depends on are computed whether or not they are stored, as the
 *   reference adds them to `indexes` (:1046-1057).  Arithmetic as the reference's for float32
 *   inputs: the three codes in float64 (sqrt of the wind speed and log of the previous DMC in
 *   float32, as numba types them), stored and carried as float32; ISI / BUI / FWI / DSR in float32.
 *   Limits: temp_condition_days, snow_condition_days <= 32, snow_cover_days <= 128.
 * ------------------------------------------------------------------------------------------- */
#define XC_FWI_SEASON_ALWAYS 0   /* season_method=None: no start-ups or shut-downs */
#define XC_FWI_SEASON_MASK   1   /* season_mask given */
#define XC_FWI_SEASON_WF93   2
#define XC_FWI_SEASON_LA08   3
#define XC_FWI_SEASON_GFWED  4
#define XC_FWI_DRY_NONE       0
#define XC_FWI_DRY_CFS        1
#define XC_FWI_DRY_GFWED      2
#define XC_FWI_DRY_GFWED_SNOW 3  /* "GFWED" with snow depth given (:1085-1088) */
typedef struct {
  int32_t season_mode, overwintering, dry_start, initial_start_up;
  int32_t temp_condition_days, snow_condition_days, snow_cover_days;
  float temp_start_thresh, temp_end_thresh, snow_thresh, prec_thresh, snow_min_mean_depth;
  float dc_start, dmc_start, ffmc_start, dc_dry_factor, dmc_dry_factor;
  double snow_min_cover_frac, carry_over_fraction, wetting_efficiency_fraction, min_dc;
  /* unit conversion of the five series on load, value = raw * in_scale[i] + in_offset[i] in float32 (one
   * rounding each, no fused multiply-add), i = tas, pr, hurs, ws, snd: what `convert_units_to` does to the
   * arrays in `cffwis_indices` (:1369-1374), e.g. K -> degC {1, -273.15}, kg m-2 s-1 -> mm/day {86400, 0}. */
  float in_scale[5], in_offset[5];
} XcFwiParams;
int32_t xc_fwi_f32(const float* tas, const float* pr, const float* hurs, const float* ws, const float* snd,
                   const uint8_t* season_mask_in, const int8_t* month, const double* lat,
                   const float* dc0, const float* dmc0, const float* ffmc0, const float* winter_pr0,
                   int64_t T, int64_t C, int64_t ldx, const XcFwiParams* params_host,
                   float* DC, float* DMC, float* FFMC, float* ISI, float* BUI, float* FWI, float* DSR,
                   uint8_t* season_mask_out, float* winter_pr_out, void* stream);

/* The element-wise members of the same module on float32 arrays of n values (device pointers):
 *   XC_FWI_EW_ISI  out = initial_spread_index(a = ws [km/h], b = ffmc)            :449-469
 *   XC_FWI_EW_BUI  out = build_up_index(a = dmc, b = dc)                          :472-501
 *   XC_FWI_EW_FWI  out = fire_weather_index(a = isi, b = bui)                     :504-528
 *   XC_FWI_EW_DSR  out = daily_severity_rating(a = fwi)                           :531-546
 *   XC_FWI_EW_OWDC out = overwintering_drought_code(a = last_dc, b = winter_pr [mm], p0 = carry-over
 *                  fraction, p1 = wetting efficiency fraction, p2 = min_dc)       :549-583, 1165-1250
 * float32 arithmetic for the first four (numpy on float32 arrays), float64 for the last (numba), as the
 * reference. */
#define XC_FWI_EW_ISI  0
#define XC_FWI_EW_BUI  1
#define XC_FWI_EW_FWI  2
#define XC_FWI_EW_DSR  3
#define XC_FWI_EW_OWDC 4
int32_t xc_fwi_elementwise_f32(int32_t kind, const float* a, const float* b, int64_t n,
                               double p0, double p1, double p2, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * s1  Standardized indices (SPI, SPEI) -- indices/stats.py
 *   Replaces the rolling step of `preprocess_standardized_index` (:831-832), the per-(cell, group) fit of
 *   `standardized_index_fit_params` (:944-953: `fit` -> `_fitfunc_1d` :45-112 -> `_fit_start` :576-684 and,
 *   for ML, scipy's gamma_gen.fit / lognorm_gen.fit with a fixed loc) and the transform of
 *   `standardized_index` (:1155-1191: rv_continuous.cdf, the zero-inflation algebra, norm.ppf, clip).
 * ------------------------------------------------------------------------------------------- */
/* out[t] = mean of x[t - window + 1 .. t] (float64 window sum, then float32(s / window)); NaN for the first
 * window - 1 steps and for any window that holds a NaN: `rolling(time=window).mean(skipna=False)`.  out has
 * leading dimension ldo (it may not alias x). */
int32_t xc_rolling_mean_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t window, float* out,
                            int64_t ldo, void* stream);

#define XC_SI_GAMMA   0
#define XC_SI_FISK    1
#define XC_SI_LOGNORM 2
#define XC_SI_APP     0
#define XC_SI_ML      1   /* with a fixed loc only (gamma, lognorm) */
/* status word bits, OR-ed over all (cell, group) samples */
#define XC_SI_STATUS_FITDATA          1   /* ML: a value <= floc (scipy FitDataError) */
#define XC_SI_STATUS_ROOT_NAN         2   /* gamma ML: brentq met a NaN at a bracket end (constant samples) */
#define XC_SI_STATUS_ROOT_SIGN        4   /* gamma ML: brentq bracket ends of one sign */
#define XC_SI_STATUS_LOGNORM_FALLBACK 8   /* lognorm ML: zero spread; scipy runs its generic optimiser */

/* Bytes of the fit workspace: one float32 per cell and value of the largest group (max_n values). */
int64_t xc_si_fit_workspace_bytes(int64_t C, int32_t max_n);
/* Fit every (group, cell): the sample of group g is x[steps[k], c] for k in [group_offsets[g],
 * group_offsets[g+1]) (device int32 arrays, steps in time order), its finite values -- zeros left out when
 * zero_inflated -- fitted with `dist` by `method` with loc fixed at floc.  Outputs (device): params (G, 3, C)
 * float64 in scipy order (shape, loc, scale), NaN where the sample has <= 1 value or a parameter is NaN;
 * n_zeros / n_notnull (G, C) int32 (values == 0, values not NaN; NULL when not zero_inflated); *status
 * (device int32, OR-ed, caller zeroes it) gets XC_SI_STATUS_* bits.  max_n >= the largest group. */
int32_t xc_si_fit_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* group_offsets,
                      const int32_t* steps, int32_t G, int32_t max_n, int32_t dist, int32_t method,
                      int32_t zero_inflated, double floc, double* params, int32_t* n_zeros, int32_t* n_notnull,
                      int32_t* status, void* workspace, int64_t workspace_bytes, void* stream);
/* out[t, c] (float64, leading dimension ldo) = the standardized index of x[t, c] under the parameters of
 * group group_of_step[t] (device int16, -1 = NaN): params (G, 3, C) float64, counts (G, C) int32 (zero-inflated
 * only, else NULL), interp = the zero-rank interpolation factor, (alpha, beta) = the zeros' plotting
 * position. */
int32_t xc_si_apply_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const int16_t* group_of_step,
                        int32_t G, const double* params, const int32_t* n_zeros, const int32_t* n_notnull,
                        int32_t dist, int32_t zero_inflated, double interp, double alpha, double beta, double* out,
                        int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * s2  Frequency analysis -- indices/stats.py
 *   Replaces the per-cell scipy fit of `fit` (:115-218: `_fitfunc_1d` :45-112 with `_fit_start` :576-610,
 *   method ML, then scipy's norm_gen.fit / gumbel_r_gen.fit / rv_continuous.fit) and the per-cell scipy ppf /
 *   isf / cdf of `parametric_quantile` (:221-289) and `parametric_cdf` (:294-360), which `fa` (:429-475) and
 *   `frequency_analysis` (:478-548) call.
 * ------------------------------------------------------------------------------------------- */
#define XC_EV_NORM       0   /* params (loc, scale) */
#define XC_EV_GUMBEL_R   1   /* params (loc, scale) */
#define XC_EV_GENEXTREME 2   /* params (c, loc, scale), scipy's sign of c */
#define XC_EV_PPF 0
#define XC_EV_ISF 1
#define XC_EV_CDF 2
/* status word bits, OR-ed over all cells */
#define XC_EV_STATUS_NOT_CONVERGED 1   /* the Newton iterations did not converge (the cell is NaN) */
#define XC_EV_STATUS_UNBOUNDED     2   /* no maximum of the likelihood (NaN): genextreme ran into c -> 1, or
                                          gumbel_r / genextreme on a sample of one repeated value */
#define XC_EV_STATUS_ROOT_NAN      4   /* gumbel_r: the scale equation is NaN at a bracket end (scipy raises) */
#define XC_EV_STATUS_ROOT_SIGN     8   /* gumbel_r: no sign change on [0, inf] (scipy raises) */

/* Bytes of the fit workspace: one float32 per cell and step. */
int64_t xc_ev_fit_workspace_bytes(int64_t T, int64_t C);
/* Fit `dist` by maximum likelihood to the finite values of each column x[t * ldx + c], t < T (device float32;
 * NaN and +-inf dropped as np.ma.masked_invalid does).  params (device float64, (2 | 3, C)): scipy's order,
 * NaN for a column with <= 1 finite value or any NaN parameter.  norm is scipy's closed form bit for bit,
 * gumbel_r the root of scipy's scale equation to a few ulp, genextreme the optimum of the likelihood (Newton in
 * (c, loc, log scale) from xclim's start).  *status (device int32, OR-ed, caller zeroes it) gets
 * XC_EV_STATUS_* bits. */
int32_t xc_ev_fit_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t dist, double* params,
                      int32_t* status, void* workspace, int64_t workspace_bytes, void* stream);
/* out[j * C + c] (device float64, (nq, C)) = scipy's `dist.ppf(q[j], *p)`, `dist.isf(q[j], *p)` or
 * `dist.cdf(q[j], *p)` (kind XC_EV_*) with p the column c of params ((2 | 3, C) device float64); q device
 * float64 (nq <= 65535).  rv_continuous's argument checks: NaN for scale <= 0, a non-finite shape, a NaN loc or
 * a probability outside [0, 1]. */
int32_t xc_ev_transform_f64(const double* params, int64_t C, int32_t dist, int32_t kind, const double* q,
                            int32_t nq, double* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a1  Spatial analogues -- analog.py
 *   Replaces the per-cell metric call of `spatial_analogs` (:87-97, xr.apply_ufunc(vectorize=True)) with
 *   `_metric_overhead` (:154-170) and the metrics `seuclidean` (:181-213), `nearest_neighbor` (:216-251),
 *   `zech_aslan` (:254-319), `szekely_rizzo` (:322-385), `kolmogorov_smirnov` (:433-495), `kldiv` (:498-587)
 *   and `mahalanobis` (:590-628).  Everything is float64 from the float32 samples (DESIGN.md section 4).
 * ------------------------------------------------------------------------------------------- */
#define XC_AN_SEUCLIDEAN         0   /* consts (K, d): the target's var(ddof=1) */
#define XC_AN_NEAREST_NEIGHBOR   1
#define XC_AN_ZECH_ASLAN         2   /* param: dmin */
#define XC_AN_SZEKELY_RIZZO      3   /* param: standardize (0 or 1) */
#define XC_AN_KOLMOGOROV_SMIRNOV 4
#define XC_AN_KLDIV              5   /* param: k, 1 <= k <= XC_AN_KLDIV_MAX_K; d <= 10 */
#define XC_AN_MAHALANOBIS        6   /* consts (K, d, d): the inverse covariance VI */
#define XC_AN_MAX_D        16
#define XC_AN_KLDIV_MAX_K  16
/* status word bits, OR-ed over all (target, cell) pairs: the reference raises ValueError for the whole call */
#define XC_AN_STATUS_NOT_FINITE 1   /* nearest_neighbor / kldiv: cKDTree's "data must be finite, check for nan
                                       or inf values" (a non-finite standardized value, or +-inf for kldiv) */
#define XC_AN_STATUS_CHKFINITE  2   /* seuclidean: scipy.linalg.norm's "array must not contain infs or NaNs" */
/* out[t * C + c] (device float64, (K, C)) = metric(target t, candidate cell c).  target: device float32 (K, n, d)
 * contiguous; cand: device float32 (m, d, C) at cand[(s * d + k) * ldc + c], ldc >= C.  NaN anywhere in either
 * sample gives NaN (:154-156).  consts: device float64 per target for seuclidean and mahalanobis (NULL
 * otherwise).  *status (device int32, caller zeroes it) gets XC_AN_STATUS_* bits.  Returns XC_ERR_INVALID for
 * bad shapes, an unknown method or a sample too large for one CTA's shared memory. */
int32_t xc_analog_f32(const float* target, int64_t n, int64_t K, const float* cand, int64_t m, int64_t C,
                      int64_t ldc, int64_t d, int32_t method, double param, const double* consts, double* out,
                      int32_t* status, void* stream);

/* ---------------------------------------------------------------------------------------------
 * e1  Ensemble statistics across realizations -- ensembles/_base.py, ensembles/_robustness.py
 *   The ensemble is an (R, N) matrix of N independent columns, x[r * ldr + n] (device float32, ldr >= N: a lat
 *   tile of a wider buffer is a column range with the buffer's member stride).  1 <= R <= XC_ENS_MAX_MEMBERS.
 * ------------------------------------------------------------------------------------------- */
#define XC_ENS_MAX_MEMBERS 128
/* The percentiles (host array of n_per <= 32 values in [0, 100]) of each column's non-NaN values, by the
 * Hyndman-Fan (alpha, beta) plotting position: `ensemble_percentiles` (_base.py:329-342) = `calc_perc`
 * (core/utils.py:279-323) along realization, `_nan_quantile` (:494-557) bit for bit, then the
 * `min_members` mask (_base.py:356-357): NaN where fewer than min_members values are not NaN.  out is (n_per, N)
 * float64 for R >= 2 and float32 for R == 1 (the np.take branch, :515-517). */
int32_t xc_ens_percentiles_f32(const float* x, int64_t R, int64_t N, int64_t ldr, const double* percentiles,
                               int32_t n_per, double alpha, double beta, int32_t min_members, void* out,
                               void* stream);
/* Mean, standard deviation (ddof 0), minimum and maximum of each column's non-NaN values, NaN where fewer than
 * min_members (and no) values are not NaN: `ensemble_mean_std_max_min` (_base.py:178-206).  weights == NULL:
 * mean / std float32 (N), float64 sums in member order rounded once; weights (device float64, R): xarray's
 * Weighted.mean / .std, float64 (N), NaN where the weights of the valid members sum to 0.  vmin / vmax float32. */
int32_t xc_ens_moments_f32(const float* x, int64_t R, int64_t N, int64_t ldr, const double* weights,
                           int32_t min_members, void* mean, void* std, float* vmin, float* vmax, void* stream);
/* `robustness_fractions` (_robustness.py:74-333) per cell: fut (R, Tf, C) at fut[r * ldf_r + t * ldf_t + c],
 * ref (R, Tr, C) likewise or NULL (fut then holds deltas, Tf = 1).  A member is valid when none of its fut and
 * ref values is NaN (MissingAny); its delta is the difference of the float64 NaN-omitting means.  `changed`:
 *   XC_ENS_TEST_NONE   always                                 (:229-232)
 *   XC_ENS_TEST_ABS    |delta| > param                        (:237)
 *   XC_ENS_TEST_REL    |delta / mean(ref)| > param            (:240)
 *   XC_ENS_TEST_TTEST  p < param, ttest_1samp(fut, mean(ref)) (:518-549)
 *   XC_ENS_TEST_WELCH  p < param, Welch's t-test              (:552-581)
 *   XC_ENS_TEST_IPCC   |delta| > sqrt(2/20) 1.645 sigma        (:636-661, without ref_pi), sigma the std of the
 *                      residuals of the float64 least-squares line through the member's annual means of ref,
 *                      ref_annual (R, P, C) at ref_annual[r * lda_r + p * C + c] (float32, from xc_period_reduce_f32
 *                      with YS periods), against ys_time[P] (device float64: the YS timestamps, e.g. in days)
 * with float64 p-values (ensemble_core.cuh).  ref_annual / ys_time are NULL for the other tests.  fractions (7, C) float64: changed, positive, changed_positive,
 * negative, changed_negative, valid, agree, as :257-271 with weights (device float64, R, or NULL for ones) and
 * strict_sign, NaN filled with 0 (:319).  pvals (R, C) float32 (t-tests only, or NULL). */
#define XC_ENS_TEST_NONE  0
#define XC_ENS_TEST_ABS   1
#define XC_ENS_TEST_REL   2
#define XC_ENS_TEST_TTEST 3
#define XC_ENS_TEST_WELCH 4
#define XC_ENS_TEST_IPCC  5
int32_t xc_ens_robustness_f32(const float* fut, int64_t Tf, int64_t ldf_r, int64_t ldf_t, const float* ref,
                              int64_t Tr, int64_t ldr_r, int64_t ldr_t, const float* ref_annual, int64_t P,
                              int64_t lda_r, const double* ys_time, int64_t R, int64_t C,
                              const double* weights, int32_t test, double param, int32_t strict_sign,
                              double* fractions, float* pvals, void* stream);

/* ---------------------------------------------------------------------------------------------
 * p1  Potential evapotranspiration and the water budget -- indices/converters.py
 *   Replaces `potential_evapotranspiration` (:1890-2152) and `water_budget` (:2652-2739) on daily inputs.
 *   The solar terms (extraterrestrial radiation, day length: indices/helpers.py:95-525) depend on (day,
 *   latitude) only; the host tabulates them once per (row, distinct latitude) in float64 and the kernels read
 *   table[row * L + lat_index[c]].  Each input is loaded as float32, mapped by its affine unit conversion
 *   (x * in_scale + in_offset, in float32) and the formula is evaluated in float64, rounded once to float32.
 *   Output unit: kg m-2 s-1 (the reference's amount2rate + hydro conversion, :2149-2151).
 * ------------------------------------------------------------------------------------------- */
#define XC_PET_BR65   0   /* tasmin, tasmax [degF]; table: radiation [cal cm-2 d-1]          :2000-2009 */
#define XC_PET_HG85   1   /* tasmin, tasmax, tas (optional) [degC]; table: 0.408 * ra [MJ m-2 d-1] :2011-2027 */
#define XC_PET_MB05   2   /* tas, or tasmin and tasmax [degC]; table: radiation (1367 W m-2) [J m-2 d-1]
                                                                                          :2060-2080 */
#define XC_PET_ALLEN98 3  /* tasmin, tasmax [degC], hurs [1], rsds, rsus, rlds, rlus [W m-2], sfcWind [m s-1];
                             no table                                                       :2116-2144 */
#define XC_PET_TW48   4   /* monthly: tas, or tasmin and tasmax [degC]; table: mean day length / 12 :2082-2114 */
#define XC_PET_DA02   5   /* monthly: tasmin, tasmax, tas (optional) [degC], pr [mm/month]; table: 0.408 * the
                             monthly sum of ra [MJ m-2 d-1]                                 :2029-2058 */
#define XC_PET_GIVEN  6   /* daily water budget from a given evspsblpot [kg m-2 s-1]; no table  :2732-2733 */
/* input slots of XcPetParams / the inputs array */
#define XC_PET_IN_TASMIN 0
#define XC_PET_IN_TASMAX 1
#define XC_PET_IN_TAS    2
#define XC_PET_IN_HURS   3
#define XC_PET_IN_RSDS   4
#define XC_PET_IN_RSUS   5
#define XC_PET_IN_RLDS   6
#define XC_PET_IN_RLUS   7
#define XC_PET_IN_WIND   8
#define XC_PET_IN_PR     9   /* the precipitation of DA02 [mm/month], or of the fused water budget [kg m-2 s-1] */
#define XC_PET_IN_EVSPSBLPOT 10
#define XC_PET_N_IN     11
typedef struct {
  int32_t method;          /* XC_PET_* */
  int32_t water_budget;    /* 1: out = pr - pet (pr in slot XC_PET_IN_PR, kg m-2 s-1), 0: out = pet */
  float in_scale[XC_PET_N_IN], in_offset[XC_PET_N_IN];
  double peta, petb;       /* MB05 coefficients (:1903-1904) */
  double wind_num, wind_den;  /* allen98: sfcWind at 2 m = sfcWind * wind_num / wind_den, the log law of
                                 helpers.py:809-849 from 10 m (log(67.8 * 2 - 5.42), log(67.8 * 10 - 5.42)) */
} XcPetParams;
/* Daily methods (BR65, HG85, MB05, allen98, GIVEN).  inputs: host array of XC_PET_N_IN device float32 pointers,
 * NULL where unused, each (T, C) at x[t * ldx + c], ldx >= C.  table: device float64 (T, L); lat_index: device
 * int32 (C) in [0, L) (allen98, GIVEN: both may be NULL).  out: device float32 (T, C) at out[t * ldx + c]. */
int32_t xc_pet_daily_f32(const float* const* inputs, int64_t T, int64_t C, int64_t ldx, const double* table,
                         int64_t L, const int32_t* lat_index, const XcPetParams* params_host, float* out,
                         void* stream);
/* Monthly methods (TW48, DA02) from daily inputs.  moff: device int32 (M + 1) row offsets of the M calendar
 * months the series touches; yoff: device int32 (Y + 1) month offsets of the years (YS groups) those months
 * fall in (TW48's annual heat index; a group of more than 12 months gives NaN months); mdays: device float64 (M) days of each complete month.  table: device
 * float64 (M, L).  Monthly means are skipna (an all-NaN month is NaN).  out: device float32 (M, C),
 * out[m * C + c].  The fused water budget (TW48 only) subtracts from pr's monthly mean. */
int32_t xc_pet_monthly_f32(const float* const* inputs, int64_t T, int64_t C, int64_t ldx, const int32_t* moff,
                           int64_t M, const int32_t* yoff, int64_t Y, const double* mdays, const double* table,
                           int64_t L, const int32_t* lat_index, const XcPetParams* params_host, float* out,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * r1  rain season (Sivakumar 1998) -- indices/_agro.py:790-980 `rain_season`, per period of freq.
 *   x: (T, C) daily precipitation at x[t * ldx + c], ldx >= C, turned into amounts by one float32
 *   multiply by `scale` (rate2amount to mm).  mask: device uint8 (T) shared by all cells:
 *   XC_RS_PRE  inside the onset prefilter (date_min_start .. the last day of the step's period),
 *   XC_RS_START inside [date_min_start, date_max_start], XC_RS_END inside [date_min_end, date_max_end];
 *   every period must hold at least one step of each of the last two (the caller checks it).
 *   Thresholds are in mm and compared in float32; methods are XC_RS_PER_DAY or XC_RS_TOTAL.
 *   out_start, out_end: device int32 (P, C) at out[p * C + c], the step of the season's start and end
 *   inside the period, -1 where there is none.  window_dry_start <= XC_RS_MAX_WINDOW, else
 *   XC_ERR_UNSUPPORTED.  Semantics in xclim_b200/csrc/rain_season_core.cuh and DESIGN.md section 4.
 * ------------------------------------------------------------------------------------------- */
#define XC_RS_PER_DAY 0
#define XC_RS_TOTAL   1
#define XC_RS_PRE     1
#define XC_RS_START   2
#define XC_RS_END     4
#define XC_RS_MAX_WINDOW 64
int32_t xc_rain_season_f32(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* period_offsets,
                           int32_t P, const uint8_t* mask, float scale, double thresh_wet_start,
                           int32_t window_wet_start, int32_t window_not_dry_start, double thresh_dry_start,
                           int32_t window_dry_start, int32_t method_dry_start, double thresh_dry_end,
                           int32_t window_dry_end, int32_t method_dry_end, int32_t* out_start, int32_t* out_end,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * c1  chill portions (Dynamic Model) and chill units (Utah Model) -- indices/_agro.py:1436-1534
 *   `chill_portions`, :1537-1592 `chill_units`, per period of freq, on the hourly temperature of
 *   `make_hourly_temperature` (indices/helpers.py:1059-1123).
 *   xc_chill_daily_f32: tasmin, tasmax (T, C) daily at x[t * ldx + c], ldx >= C; the 24 hours of each day
 *   are made in registers from weights (T, L, XC_CHILL_ROW) float64, the row of cell c being
 *   lat_index[c] (converters.hourly_weights).  xc_chill_hourly: an explicit hourly series (H, C), float32
 *   or float64 (x_f64), 24 steps per day from 00:00 (the last day may be partial: 24 (T - 1) < H <= 24 T).
 *   period_offsets: (P + 1) day offsets.  day_mask: device uint8 (T), nonzero = selected, or null for
 *   every day; unselected days are skipped (select_time(drop=True) for the portions, NaN for the units).
 *   An hourly value v is v * k_scale + k_offset in K for the portions and v * c_scale + c_offset in degC
 *   for the units.  what: XC_CHILL_PORTIONS | XC_CHILL_UNITS, plus XC_CHILL_POSITIVE_ONLY for the units.
 *   out_cp, out_cu: device float64 (P, C) at out[p * C + c]; out_valid: int32 (P, C) selected non-NaN
 *   hours, or null.  xc_hourly_temperature_f32 writes the hourly series (24 T, C) float64 at
 *   out[h * C + c].  Semantics in xclim_b200/csrc/chill_core.cuh and DESIGN.md section 4.
 * ------------------------------------------------------------------------------------------- */
#define XC_CHILL_ROW 28
#define XC_CHILL_PORTIONS 1
#define XC_CHILL_UNITS 2
#define XC_CHILL_POSITIVE_ONLY 4
int32_t xc_chill_daily_f32(const float* tasmin, const float* tasmax, int64_t T, int64_t C, int64_t ldx,
                           const double* weights, int32_t L, const int32_t* lat_index,
                           const int32_t* period_offsets, int32_t P, const uint8_t* day_mask, double k_scale,
                           double k_offset, double c_scale, double c_offset, int32_t what, double* out_cp,
                           double* out_cu, int32_t* out_valid, void* stream);
int32_t xc_chill_hourly(const void* x, int32_t x_f64, int64_t H, int64_t C, int64_t ldx,
                        const int32_t* period_offsets, int32_t P, const uint8_t* day_mask, double k_scale,
                        double k_offset, double c_scale, double c_offset, int32_t what, double* out_cp,
                        double* out_cu, int32_t* out_valid, void* stream);
int32_t xc_hourly_temperature_f32(const float* tasmin, const float* tasmax, int64_t T, int64_t C, int64_t ldx,
                                  const double* weights, int32_t L, const int32_t* lat_index, double* out,
                                  void* stream);

#ifdef __cplusplus
}
#endif
#endif /* XCLIM_B200_H */
