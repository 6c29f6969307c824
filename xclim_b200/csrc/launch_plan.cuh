// Launch plans: which template instance a launcher runs, on which day range, with how many chunks and how much
// dynamic shared memory.  Pure host functions of the call's shape (no CUDA runtime call, no environment read: the
// launchers pass XCLIM_B200_NO_TMA / XCLIM_B200_BOOT_V1 and the device's SM count in), so that the launchers and
// the host build of tests/csrc/dispatch_host.cu execute the same decision.  On a rejected call a plan sets the
// error text and returns the status of the entry point.
#pragma once
#include <stdio.h>

#include <vector>

#include "quantile.cuh"

namespace xc {

constexpr int kThreads = 128;              // cells per CTA of the day-of-year, bootstrap, rolling and period kernels
constexpr int kSelThreads = 64;            // cells per CTA of the percentile selection kernel
constexpr int kTmaCells = kThreads;        // cells per CTA of the TMA-fed window-5 kernel
constexpr int kBT = 32;                    // threads per CTA of bootstrap5_kernel: one warp
constexpr int kSelMaxSamples = 768;        // samples per cell the selection kernel holds in shared memory
constexpr size_t kDayListSmemCap = 200 * 1024;   // the ring kernels' day lists
constexpr size_t kBootSmemCap = 227 * 1024;      // bootstrap_kernel: the H100's per-block opt-in maximum
constexpr size_t kRingSmemCap = 160 * 1024;      // the four-cells-per-thread rolling rings
constexpr int kSlideAbove = 6;             // BlockStream slides sum / mean windows longer than this
constexpr int kBootExactAbove = 32;        // more base years: bootstrap_kernel drops its rank shortcuts

// Day split of the day-of-year kernels: blockIdx.y walks `chunks` chunks of `per` consecutive days.  Enough
// chunks that the cblocks cell blocks give ctas_per_sm CTAs on each of the `sms` SMs, but at least min_per days
// per chunk (each chunk pays a halo of extra days), rounded up to whole pairs of days when `pairs` and to a
// multiple of `align` days (every chunk starts on a multiple of `align`).  The split never changes a result.
struct DaySplit {
  int chunks, per;
};
inline DaySplit split_days(int nd, int64_t cblocks, int ctas_per_sm, int min_per, bool pairs, int align, int sms) {
  int chunks = (int)(((int64_t)sms * ctas_per_sm + cblocks - 1) / cblocks);
  if (chunks < 1) chunks = 1;
  int per = (nd + chunks - 1) / chunks;
  if (per < min_per) per = min_per;
  if (pairs) per = (per + 1) & ~1;
  per = (per + align - 1) / align * align;
  if (per > nd) per = nd;
  return {(nd + per - 1) / per, per};
}

// ---- percentile_doy ---------------------------------------------------------------------------------------
// Every instance xc_percentile_doy_f32 can launch.  The launcher instantiates each one with the K (list length;
// w5t: years - 16) and TABLE of its entry in kPdoy, the plan sizes its shared memory from the same entry.
enum PdoyKernel : int32_t {
  kGeneric4, kGeneric8, kGeneric16, kGeneric32, kGeneric64, kSelect,
  kUniform8, kUniform8T, kUniform16, kUniform16T, kUniform32, kUniform32T,
  kW5p8, kW5p8T, kW5p16, kW5p16T, kW5t14, kW5t15, kW5t16, kPdoyKernels
};
struct PdoyInstance {
  const char* name;
  int k;
  bool table;   // reads the (year, doy) position tables
};
constexpr PdoyInstance kPdoy[kPdoyKernels] = {
    {"generic<4>", 4, true}, {"generic<8>", 8, true}, {"generic<16>", 16, true}, {"generic<32>", 32, true},
    {"generic<64>", 64, true}, {"select", 0, true},
    {"uniform<8, false>", 8, false}, {"uniform<8, true>", 8, true}, {"uniform<16, false>", 16, false},
    {"uniform<16, true>", 16, true}, {"uniform<32, false>", 32, false}, {"uniform<32, true>", 32, true},
    {"w5p<8, false>", 8, false}, {"w5p<8, true>", 8, true}, {"w5p<16, false>", 16, false},
    {"w5p<16, true>", 16, true}, {"w5t<14>", 14, false}, {"w5t<15>", 15, false}, {"w5t<16>", 16, false}};

// One launch: percentile ip on days [a, b), cblocks x chunks CTAs of `per` days each.
struct PdoyLaunch {
  int32_t kernel, ip, a, b, chunks, per;
  int64_t cblocks;
  size_t smem;       // dynamic shared memory
  QuantSpec spec;
};

inline int64_t cell_blocks(int64_t C, int threads) { return (C + threads - 1) / threads; }

// generic kernel with the shortest list that holds `need` (<= 64) order statistics
inline PdoyLaunch pdoy_generic(int need, int ip, int a, int b, int64_t C, int sms) {
  int k = kGeneric4;
  while (kPdoy[k].k < need) ++k;
  const DaySplit sp = split_days(b - a, cell_blocks(C, kThreads), 8, 1, false, 1, sms);
  return {k, ip, a, b, sp.chunks, sp.per, cell_blocks(C, kThreads), 0, {}};
}

// Day-list kernel for `need` (<= 32) order statistics and window W: the paired kernel for window 5 and need <= 16,
// else the ring kernel; `table`: through the (year, doy) table, else on uniform years.
inline PdoyLaunch pdoy_day_lists(int need, int W, int ip, int a, int b, int64_t C, bool table, int sms) {
  const int64_t cb = cell_blocks(C, kThreads);
  const int t = table ? 1 : 0;
  if (W == 5 && need <= 16) {
    const int k = (need <= 8 ? kW5p8 : kW5p16) + t, K = kPdoy[k].k;
    const DaySplit sp = split_days(b - a, cb, 16, 40, true, 1, sms);   // 4 extra day lists per chunk, whole pairs
    // 4 lists + 4 counts per lane, plus the 32-row staging column of the cp.async prefetch
    const size_t smem = (size_t)4 * (K + 1) * kThreads * 4 + (K == 16 && !table ? (size_t)32 * kThreads * 4 : 0);
    return {k, ip, a, b, sp.chunks, sp.per, cb, smem, {}};
  }
  const int k = (need <= 8 ? kUniform8 : need <= 16 ? kUniform16 : kUniform32) + t;
  // at least 8 W days per chunk keeps the halo overhead (W-1 extra day lists per chunk) small
  const DaySplit sp = split_days(b - a, cb, 12, 8 * W, false, 1, sms);
  return {k, ip, a, b, sp.chunks, sp.per, cb, (size_t)(W - 1) * (kPdoy[k].k + 1) * kThreads * 4, {}};
}

// (year, doy) -> step table: pos[y * n_doy + d - 1] = the step of day-of-year d of year y, -1 where there is
// none.  Returns the first step whose indexes are out of range, or -1.
inline int64_t build_pos_table(int64_t T, const int16_t* doy, const int16_t* year, int32_t n_doy, int32_t n_years,
                               std::vector<int32_t>& pos) {
  pos.assign((size_t)n_doy * n_years, -1);
  for (int64_t t = 0; t < T; ++t) {
    const int d = doy[t], y = year[t];
    if (d < 1 || d > n_doy || y < 0 || y >= n_years) return t;
    pos[(size_t)y * n_doy + (d - 1)] = (int32_t)t;
  }
  return -1;
}

struct PdoyPlan {
  std::vector<int32_t> pos;          // the (year, doy) -> step table
  std::vector<PdoyLaunch> launches;
};

// The launches of xc_percentile_doy_f32 (has_vrow: _vrow_f32) for a series of T steps in rows of ldx floats from
// a base pointer that is (aligned16) or is not 16-byte aligned; no_tma: XCLIM_B200_NO_TMA is set.
inline int32_t plan_percentile_doy(int64_t T, const int16_t* doy, const int16_t* year, bool has_vrow, int32_t n_doy,
                                   int32_t n_years, int32_t window, const double* percentiles, int32_t n_per,
                                   double alpha, double beta, int64_t C, int64_t ldx, bool aligned16, bool no_tma,
                                   int sms, PdoyPlan* plan) {
  if (window % 2 == 0) {
    set_error("even `window` (xarray's center=True convention for even windows) is not supported");
    return XC_ERR_UNSUPPORTED;
  }
  const int h = window / 2;
  std::vector<int32_t>& pos = plan->pos;
  const int64_t bad = build_pos_table(T, doy, year, n_doy, n_years, pos);
  XC_REQUIRE(bad < 0, "doy/year index out of range at step %lld", (long long)bad);
  // uniform-year fast path: step t is day t % n_doy of year t / n_doy
  bool uniform = !has_vrow && T == (int64_t)pos.size();
  for (size_t k = 0; uniform && k < pos.size(); ++k) uniform = (pos[k] == (int32_t)k);

  // interior days whose windows never leave the year: [h, L_int - h) with L_int the shortest full year
  const int L_int = (n_doy == 366) ? 365 : n_doy;
  std::vector<PdoyLaunch>& out = plan->launches;
  out.clear();
  for (int ip = 0; ip < n_per; ++ip) {
    const double per = percentiles[ip];
    XC_REQUIRE(per >= 0.0 && per <= 100.0, "percentiles must be in [0, 100], got %g", per);
    QuantSpec spec;
    const int need = plan_quantile(per, alpha, beta, n_years * window, &spec);
    if (need < 0) {
      set_error("percentile %g with alpha=%g beta=%g: plotting positions outside [0, 1] are not supported", per,
                alpha, beta);
      return XC_ERR_UNSUPPORTED;
    }
    const size_t first = out.size();
    if (need > 64) {
      // order statistics far from both ends of the sample (e.g. the median): selection kernel
      const int nmax = n_years * window;
      if (nmax > kSelMaxSamples) {
        set_error("percentile %g of up to %d samples: the selection kernel holds at most 768 samples per cell", per,
                  nmax);
        return XC_ERR_UNSUPPORTED;
      }
      const int64_t cb = cell_blocks(C, kSelThreads);
      const DaySplit sp = split_days(n_doy, cb, 8, 1, false, 1, sms);
      out.push_back({kSelect, ip, 0, n_doy, sp.chunks, sp.per, cb, (size_t)nmax * kSelThreads * 4, {}});
    } else {
      const int kk = need <= 8 ? 8 : need <= 16 ? 16 : 32;
      const size_t smem_need = (size_t)(window - 1) * (kk + 1) * kThreads * 4;
      const bool fast_ok = window >= 3 && need <= 32 && smem_need <= kDayListSmemCap && (L_int - 2 * h) >= 8;
      if (uniform && fast_ok) {
        // TMA: 30..32 years, global strides of whole 16 bytes from an aligned base, a whole box of days
        const bool tma = window == 5 && need > 8 && need <= 16 && !no_tma && n_years >= 30 && n_years <= 32 &&
                         ldx % 4 == 0 && aligned16 && T == (int64_t)n_doy * n_years && n_doy >= 8 &&
                         C <= 2147483647LL - kTmaCells;
        if (tma) {
          const int k = kW5t14 + (n_years - 30), N = 16 + kPdoy[k].k;
          const int64_t cb = cell_blocks(C, kTmaCells);
          const DaySplit sp = split_days(n_doy, cb, 12, 40, true, 1, sms);   // 4 extra day lists, whole pairs
          const size_t smem = (size_t)2 * N * kTmaCells * 4 + (size_t)4 * (16 + 1) * kThreads * 4 + 64;
          out.push_back({k, ip, 0, n_doy, sp.chunks, sp.per, cb, smem, {}});
        } else {
          out.push_back(pdoy_day_lists(need, window, ip, 0, n_doy, C, false, sms));
        }
      } else {
        // Days whose samples decompose into per-day lists: the window must stay inside the year
        // ([h, L_int - h)) and no window centre may fall outside the series (the h days before the first
        // step's day-of-year and after the last step's: their neighbours exist but their centres do not).
        std::vector<char> fast_day((size_t)n_doy, 0);
        if (fast_ok) {
          for (int d = h; d < L_int - h; ++d) fast_day[d] = 1;
          const int s0 = doy[0] - 1, e1 = doy[T - 1] - 1;
          for (int d = s0 - h; d < s0; ++d)
            if (d >= 0) fast_day[d] = 0;
          for (int d = e1 + 1; d <= e1 + h; ++d)
            if (d < n_doy) fast_day[d] = 0;
        }
        for (int a = 0; a < n_doy;) {
          int b = a;
          const bool fast = fast_day[a] != 0;
          while (b < n_doy && (fast_day[b] != 0) == fast) ++b;
          out.push_back(fast && (b - a) >= 8 ? pdoy_day_lists(need, window, ip, a, b, C, true, sms)
                                             : pdoy_generic(need, ip, a, b, C, sms));
          a = b;
        }
      }
    }
    for (size_t i = first; i < out.size(); ++i) out[i].spec = spec;
  }
  return XC_OK;
}

// ---- bootstrap exceedance kernels -------------------------------------------------------------------------
// bootstrap5_kernel, then bootstrap_kernel<KA, KB>: kept order statistics KB, list length KA >= KB + window
enum BootKernel : int32_t { kBoot5, kBoot16x8, kBoot32x16, kBoot32x32, kBootKernels };
struct BootInstance {
  const char* name;
  int ka, kb;
};
constexpr BootInstance kBoot[kBootKernels] = {{"bootstrap5", 0, 8}, {"16x8", 16, 8}, {"32x16", 32, 16},
                                              {"32x32", 32, 32}};

struct BootPlan {
  int32_t kernel;
  int64_t cblocks;
  DaySplit split;
  size_t smem;
  QuantSpec spec;
};

// The exceedance kernel for N base years of L days, the same choice for per-period counts and (mask) per-pair
// masks, whose day chunks start on multiples of 32 days; boot_v1: XCLIM_B200_BOOT_V1 is set.
inline int32_t plan_bootstrap(int32_t N, int32_t L, int32_t window, double percentile, double alpha, double beta,
                              bool mask, bool boot_v1, int64_t C, int sms, BootPlan* p) {
  const int need = plan_quantile(percentile, alpha, beta, N * window, &p->spec);
  const int align = mask ? 32 : 1;
  if (need > 0 && need <= kBoot[kBoot5].kb && window == 5 && N <= 16 && L > 8 && !boot_v1) {
    p->kernel = kBoot5;
    p->cblocks = cell_blocks(C, kBT);
    p->split = split_days(L, p->cblocks, 12, 20, false, align, sms);
    p->smem = ((size_t)8 * N + 16) * kBT * 4;
    return XC_OK;
  }
  p->kernel = kBoot16x8;
  while (p->kernel < kBootKernels && !(need > 0 && need <= kBoot[p->kernel].kb && need + window <= kBoot[p->kernel].ka))
    ++p->kernel;
  if (p->kernel == kBootKernels) {
    set_error("bootstrap: percentile %g of %d samples needs %d order statistics (+%d removals); at most 32 are kept",
              percentile, N * window, need, window);
    return XC_ERR_UNSUPPORTED;
  }
  p->cblocks = cell_blocks(C, kThreads);
  p->split = split_days(L, p->cblocks, 6, 4 * window, false, align, sms);
  p->smem = ((size_t)(window - 1) * (kBoot[p->kernel].ka + 1) + (size_t)window * N) * kThreads * 4;
  if (p->smem > kBootSmemCap) {
    set_error("bootstrap: %d base years x window %d need %zu bytes of shared memory per block", N, window, p->smem);
    return XC_ERR_UNSUPPORTED;
  }
  return XC_OK;
}

// ---- rolling windows and spells ---------------------------------------------------------------------------
enum RollFamily : int32_t {
  kSpellSumw, kRollingSumw, kSpellRunstat4, kRollingReduce4, kSpellRunstat, kRollingReduce, kSpellMask, kRollFamilies
};
constexpr const char* kRollFamily[kRollFamilies] = {"spell_sumw", "rolling_sumw", "spell_runstat4",
                                                    "rolling_period_reduce4", "spell_runstat",
                                                    "rolling_period_reduce", "spell_mask"};
constexpr int kRegisterWMin = 2, kRegisterWMax = 8;   // the windows of spell_sumw / rolling_sumw

// BlockStream: short windows are cheaper to re-read (L1 hits) than to slide with float64 adds
__host__ __device__ inline bool block_stream_slides(int wstat, int w) {
  return (wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN) && w > kSlideAbove;
}
// whether an instance of `family` keeps a running float64 window sum: the register kernels re-add each window
inline bool roll_slides(int family, int window, int wstat) {
  if (family == kSpellSumw || family == kRollingSumw) return false;
  if (family == kSpellRunstat || family == kSpellMask) return block_stream_slides(wstat, window);
  return wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN;
}
// the streaming kernels need 16-byte aligned rows and a ring that fits shared memory
inline bool can_stream4(int64_t C, int64_t ldx, bool aligned_x, bool aligned_out, int32_t w) {
  return (C % 4 == 0) && (ldx % 4 == 0) && aligned_x && aligned_out && (size_t)w * kThreads * 16 <= kRingSmemCap;
}

// The instance: family<window, arg, after>.  `arg`: spell_sumw's RED (MAX / SUM / COUNT keep their running form,
// the other reducers kRunAny = -1) or rolling_sumw's MODE (0 max, 1 min, 2 the other statistics); `after`: spell
// statistics after the resampling.
struct RollPlan {
  int32_t family, window, arg;
  bool after;
};

inline RollPlan plan_spell(int64_t C, int64_t ldx, bool aligned_x, bool aligned_out, int32_t window, int32_t wstat,
                           int32_t reducer, bool after) {
  const bool s4 = can_stream4(C, ldx, aligned_x, aligned_out, window);
  if (s4 && (wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN) && window >= kRegisterWMin && window <= kRegisterWMax)
    return {kSpellSumw, window, reducer == XC_RL_MAX || reducer == XC_RL_SUM || reducer == XC_RL_COUNT ? reducer : -1,
            after};
  return {s4 ? kSpellRunstat4 : kSpellRunstat, window, 0, after};
}

inline int32_t plan_rolling(int64_t C, int64_t ldx, bool aligned_x, bool aligned_out, int32_t window, int32_t wstat,
                            int32_t center, int32_t stat, RollPlan* p) {
  if (center && window % 2 == 0) {
    set_error("centred rolling windows of even length are not supported");
    return XC_ERR_UNSUPPORTED;
  }
  const bool s4 = can_stream4(C, ldx, aligned_x, aligned_out, window);
  if (s4 && (wstat == XC_STAT_SUM || wstat == XC_STAT_MEAN) && window >= kRegisterWMin && window <= kRegisterWMax)
    *p = {kRollingSumw, window, stat == XC_STAT_MAX ? 0 : stat == XC_STAT_MIN ? 1 : 2, false};
  else
    *p = {s4 ? kRollingReduce4 : kRollingReduce, window, 0, false};
  return XC_OK;
}

// "spell_sumw<5, 2, false>", "rolling_sumw<3, 1>", "spell_runstat4<true>", "rolling_period_reduce", ...
inline void roll_instance_name(const RollPlan& p, char* buf, size_t n) {
  const char* f = kRollFamily[p.family];
  const char* after = p.after ? "true" : "false";
  if (p.family == kSpellSumw) snprintf(buf, n, "%s<%d, %d, %s>", f, p.window, p.arg, after);
  else if (p.family == kRollingSumw) snprintf(buf, n, "%s<%d, %d>", f, p.window, p.arg);
  else if (p.family == kSpellRunstat4) snprintf(buf, n, "%s<%s>", f, after);
  else snprintf(buf, n, "%s", f);
}

// ---- the fused multi-output pass --------------------------------------------------------------------------
// Checks `pl` and neutralises its entries beyond the declared counts (the rounded-up instantiation computes and
// drops them).  Output buffers are checked by the entry point.
inline int32_t check_multi_plan(XcMultiPlan& pl, int32_t n_slots) {
  XC_REQUIRE(pl.n_cond >= 0 && pl.n_cond <= XC_MULTI_MAX_COND && pl.n_runs >= 0 && pl.n_runs <= XC_MULTI_MAX_RUNS &&
                 pl.n_runs % 2 == 0 && pl.n_msum >= 0 && pl.n_msum <= XC_MULTI_MAX_MSUM && pl.n_sums >= 0 &&
                 pl.n_sums <= XC_MULTI_MAX_SUMS,
             "plan holds at most %d conditions, %d run outputs (an even number), %d run sums and %d conditional sums",
             XC_MULTI_MAX_COND, XC_MULTI_MAX_RUNS, XC_MULTI_MAX_MSUM, XC_MULTI_MAX_SUMS);
  XC_REQUIRE(pl.n_runs / 2 <= pl.n_cond && (pl.n_msum == 0 || pl.n_cond > 0), "run outputs need their condition");
  auto slot_ok = [&](int32_t sl) { return sl >= -1 && sl < n_slots; };
  bool ok = slot_ok(pl.slot_sum) && slot_ok(pl.slot_mean) && slot_ok(pl.slot_min) && slot_ok(pl.slot_max);
  for (int j = 0; j < XC_MULTI_MAX_COND; ++j) {
    if (j >= pl.n_cond) { pl.cond[j].slot_n = pl.cond[j].slot_max = -1; pl.cond[j].wmax = 1; pl.cond[j].sgn = 0.f; pl.cond[j].thr = 0.f; }
    ok = ok && slot_ok(pl.cond[j].slot_n) && slot_ok(pl.cond[j].slot_max);
  }
  for (int k = 0; k < XC_MULTI_MAX_RUNS; ++k) {
    if (k >= pl.n_runs) { pl.runs[k].slot = -1; pl.runs[k].cond = k / 2; pl.runs[k].window = 1; pl.runs[k].kind = 0; }
    ok = ok && slot_ok(pl.runs[k].slot) && pl.runs[k].window >= 1 && (pl.runs[k].kind == 0 || pl.runs[k].kind == 1) &&
         pl.runs[k].cond == k / 2;
  }
  for (int k = 0; k < XC_MULTI_MAX_MSUM; ++k) {
    if (k >= pl.n_msum) { pl.msum[k].slot = -1; pl.msum[k].cond = 0; pl.msum[k].window = 1; }
    ok = ok && slot_ok(pl.msum[k].slot) && pl.msum[k].window >= 1 && pl.msum[k].cond == 0;
  }
  for (int k = 0; k < XC_MULTI_MAX_SUMS; ++k) {
    if (k >= pl.n_sums) { pl.sums[k].slot = -1; pl.sums[k].mode = 0; }
    ok = ok && slot_ok(pl.sums[k].slot) && (pl.sums[k].mode == 0 || pl.sums[k].mode == 1);
  }
  XC_REQUIRE(ok, "plan: output slot outside [-1, n_slots), window < 1 or run output not at its condition's place");
  return XC_OK;
}

// period_multi_kernel<NC, NCR, NM, NS, VEC, UNROLL> for a checked plan's counts: the counts rounded up to the
// instantiated shapes.  4 cells per thread only pays for the lightest passes (measured: conditional sums are bound
// by the float32 -> float64 conversions on the XU pipe, more conditions by registers).
struct MultiShape {
  int nc, ncr, nm, ns, vec, unroll;
};
constexpr MultiShape multi_shape(int n_cond, int n_runs, int n_msum, int n_sums) {
  const int nc = n_cond == 0 ? 0 : (n_cond <= 2 ? 2 : (n_cond <= 4 ? 4 : 6));
  const int ncr = n_runs / 2, ns = n_sums == 0 ? 0 : 3;
  const bool light = ncr == 0 && n_msum == 0 && ns == 0 && nc <= 2;
  return {nc, ncr, n_msum, ns, light ? 4 : 2, light ? 8 : 12};
}

}  // namespace xc
