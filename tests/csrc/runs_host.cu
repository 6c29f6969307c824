// TEST INFRASTRUCTURE: a HOST build of the period-edge run rule (xc::PeriodMask) and the run-length reducers
// (xc::run_step, xc::run_close, xc::RunAcc in xclim_b200/csrc/runstat.cuh), which every run-length kernel applies on
// the device.  tests/test_runs_host.py drives them in the kernels' order and checks them against the oracle's
// resample_and_rl.  Nothing in xclim_b200/ loads this library.
#include "../../xclim_b200/csrc/runstat.cuh"

// mask: (T, C) of 0 / 1.  out: (P, C) reducer values.  seen: (P, T, C), zeroed by the caller: the mask each period
// sees (its own steps, and with `after` every later step, as a thread does while a neighbouring cell's run is open).
template <bool RUNNING, int RED>
static void drive(const uint8_t* mask, int T, int C, const int32_t* poff, int P, bool after, int window, int reducer,
                  float* out, uint8_t* seen) {
  for (int p = 0; p < P; ++p) {
    const int t0 = poff[p], t1 = poff[p + 1];
    uint8_t* sp = seen + (int64_t)p * T * C;
    for (int c = 0; c < C; ++c) {
      xc::PeriodMask pm;
      pm.init();
      int32_t cur = 0;
      xc::RunAcc<RED> acc;
      acc.init();
      if (after && t0 > 0) pm.look_back(mask[(t0 - 1) * C + c] != 0);
      for (int t = t0; t < t1; ++t) {
        const bool m = pm.inside(after, mask[t * C + c] != 0);
        sp[t * C + c] = m;
        xc::run_step<RUNNING>(cur, acc, m, window);
      }
      for (int t = t1; after && t < T; ++t) {
        const bool m = xc::PeriodMask::past_end(mask[t * C + c] != 0, cur > 0);
        sp[t * C + c] = m;
        xc::run_step<RUNNING>(cur, acc, m, window);
      }
      xc::run_close<RUNNING>(cur, acc, window);
      out[p * C + c] = acc.result(reducer);
    }
  }
}

// form 0: RunAcc<reducer>; 1: RunAcc<kRunAny> with the reducer chosen at run time; 2: the window-1 running forms of
// max, sum and count.  Returns -1 for a combination the kernels never instantiate.
extern "C" int32_t runs_host(const uint8_t* mask, int32_t T, int32_t C, const int32_t* poff, int32_t P, int32_t after,
                             int32_t reducer, int32_t window, int32_t form, float* out, uint8_t* seen) {
  const bool a = after != 0;
  if (form == 1) {
    drive<false, xc::kRunAny>(mask, T, C, poff, P, a, window, reducer, out, seen);
    return 0;
  }
  if (form == 2) {
    if (window != 1) return -1;
    switch (reducer) {
      case XC_RL_MAX: drive<true, XC_RL_MAX>(mask, T, C, poff, P, a, 1, reducer, out, seen); return 0;
      case XC_RL_SUM: drive<true, XC_RL_SUM>(mask, T, C, poff, P, a, 1, reducer, out, seen); return 0;
      case XC_RL_COUNT: drive<true, XC_RL_COUNT>(mask, T, C, poff, P, a, 1, reducer, out, seen); return 0;
    }
    return -1;
  }
  switch (reducer) {
    case XC_RL_MAX: drive<false, XC_RL_MAX>(mask, T, C, poff, P, a, window, reducer, out, seen); return 0;
    case XC_RL_MIN: drive<false, XC_RL_MIN>(mask, T, C, poff, P, a, window, reducer, out, seen); return 0;
    case XC_RL_SUM: drive<false, XC_RL_SUM>(mask, T, C, poff, P, a, window, reducer, out, seen); return 0;
    case XC_RL_COUNT: drive<false, XC_RL_COUNT>(mask, T, C, poff, P, a, window, reducer, out, seen); return 0;
    case XC_RL_MEAN: drive<false, XC_RL_MEAN>(mask, T, C, poff, P, a, window, reducer, out, seen); return 0;
    case XC_RL_STD: drive<false, XC_RL_STD>(mask, T, C, poff, P, a, window, reducer, out, seen); return 0;
  }
  return -1;
}
