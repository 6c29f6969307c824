// TEST INFRASTRUCTURE: a HOST build of the launch plans (xclim_b200/csrc/launch_plan.cuh) that the launchers of
// percentile_doy, the bootstrap, the rolling windows / spells and the fused multi-output pass execute, so that
// the tests name the kernel instance a call runs by asking the launchers' own code.  Bound by
// tests/dispatch_host_build.py.  Nothing in xclim_b200/ loads this library.
#include <stdarg.h>

#include "../../xclim_b200/csrc/launch_plan.cuh"

using namespace xc;

static char g_error[512];

void xc::set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof g_error, fmt, ap);
  va_end(ap);
}

extern "C" const char* dispatch_error() { return g_error; }

// name k of the percentile_doy instances (list 0), bootstrap kernels (1) and rolling families (2); "" past the end
extern "C" const char* dispatch_name(int32_t list, int32_t k) {
  if (list == 0) return k < kPdoyKernels ? kPdoy[k].name : "";
  if (list == 1) return k < kBootKernels ? kBoot[k].name : "";
  return k < kRollFamilies ? kRollFamily[k] : "";
}

extern "C" void dispatch_split_days(int32_t nd, int64_t cblocks, int32_t ctas_per_sm, int32_t min_per, int32_t pairs,
                                    int32_t align, int32_t sms, int32_t* out) {
  const DaySplit sp = split_days(nd, cblocks, ctas_per_sm, min_per, pairs != 0, align, sms);
  out[0] = sp.chunks;
  out[1] = sp.per;
}

extern "C" int32_t dispatch_plan_quantile(double per, double alpha, double beta, int32_t n_max, int32_t* top) {
  QuantSpec spec;
  const int need = plan_quantile(per, alpha, beta, n_max, &spec);
  *top = need < 0 ? 0 : spec.top;
  return need;
}

// launches as rows of 7 int64: kernel, ip, a, b, chunks, per, smem; *n: their number (up to cap rows)
extern "C" int32_t dispatch_pdoy(int64_t T, const int16_t* doy, const int16_t* year, int32_t has_vrow, int32_t n_doy,
                                 int32_t n_years, int32_t window, const double* pers, int32_t n_per, double alpha,
                                 double beta, int64_t C, int64_t ldx, int32_t aligned16, int32_t no_tma, int32_t sms,
                                 int64_t* out, int32_t cap, int32_t* n) {
  PdoyPlan plan;
  const int32_t e = plan_percentile_doy(T, doy, year, has_vrow != 0, n_doy, n_years, window, pers, n_per, alpha, beta,
                                        C, ldx, aligned16 != 0, no_tma != 0, sms, &plan);
  *n = e ? 0 : (int32_t)plan.launches.size();
  for (int32_t i = 0; i < *n && i < cap; ++i) {
    const PdoyLaunch& ln = plan.launches[i];
    const int64_t row[7] = {ln.kernel, ln.ip, ln.a, ln.b, ln.chunks, ln.per, (int64_t)ln.smem};
    for (int k = 0; k < 7; ++k) out[7 * i + k] = row[k];
  }
  return e;
}

extern "C" int32_t dispatch_boot_exact_above() { return kBootExactAbove; }

// out: kernel, chunks, per, smem
extern "C" int32_t dispatch_bootstrap(int32_t N, int32_t L, int32_t window, double percentile, double alpha,
                                      double beta, int32_t mask, int32_t boot_v1, int64_t C, int32_t sms,
                                      int64_t* out) {
  BootPlan p;
  const int32_t e = plan_bootstrap(N, L, window, percentile, alpha, beta, mask != 0, boot_v1 != 0, C, sms, &p);
  const int64_t row[4] = {p.kernel, p.split.chunks, p.split.per, (int64_t)p.smem};
  for (int k = 0; k < 4 && !e; ++k) out[k] = row[k];
  return e;
}

extern "C" int32_t dispatch_can_stream4(int64_t C, int64_t ldx, int32_t aligned_x, int32_t aligned_out, int32_t w) {
  return can_stream4(C, ldx, aligned_x != 0, aligned_out != 0, w) ? 1 : 0;
}
extern "C" int32_t dispatch_roll_slides(int32_t family, int32_t window, int32_t wstat) {
  return roll_slides(family, window, wstat) ? 1 : 0;
}

// the instance names of xc_spell_runstat_f32 (center < 0: `stat` is the run-length reducer) and
// xc_rolling_period_reduce_f32
extern "C" int32_t dispatch_rolling(int64_t C, int64_t ldx, int32_t aligned_x, int32_t window, int32_t wstat,
                                    int32_t center, int32_t stat, int32_t resample_before_rl, char* name, int32_t n) {
  RollPlan p;
  int32_t e = XC_OK;
  if (center < 0) p = plan_spell(C, ldx, aligned_x != 0, true, window, wstat, stat, resample_before_rl == 0);
  else e = plan_rolling(C, ldx, aligned_x != 0, true, window, wstat, center, stat, &p);
  if (!e) roll_instance_name(p, name, (size_t)n);
  return e;
}

// checks (and normalises) *plan as xc_period_multi_f32 does
extern "C" int32_t dispatch_multi_check(XcMultiPlan* plan, int32_t n_slots) { return check_multi_plan(*plan, n_slots); }

// out: NC, NCR, NM, NS, VEC, UNROLL
extern "C" void dispatch_multi_shape(int32_t n_cond, int32_t n_runs, int32_t n_msum, int32_t n_sums, int32_t* out) {
  const MultiShape s = multi_shape(n_cond, n_runs, n_msum, n_sums);
  const int32_t v[6] = {s.nc, s.ncr, s.nm, s.ns, s.vec, s.unroll};
  for (int k = 0; k < 6; ++k) out[k] = v[k];
}
