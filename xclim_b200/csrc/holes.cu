// Spell statistics with holes: spells separated by fewer than `min_gap` non-spell steps are merged.
//
// Replaces generic.spell_mask(..., min_gap > 1) (indices/generic.py:537-538) =
// rl.runs_with_holes(is_in_spell, 1, ~is_in_spell, min_gap) (indices/run_length.py:844-888) followed by
// generic._spell_length_statistics (:557-585) with resample_before_rl=True, for window == 1 masks
// (is_in_spell = x op thr).  What runs_with_holes does to the mask m, restated per gap (a maximal
// run of False of length G):
//   * G >= min_gap                      : the whole gap stays 0 (its first G-min_gap+1 steps are stop
//                                         points, the rest forward-fill those zeros);
//   * G <  min_gap, preceded by a True  : the gap is bridged (forward-filled 1s) -- INCLUDING a short
//                                         gap that runs into the end of the series (no stop point
//                                         can form there);
//   * a gap that starts the series      : stays 0 (nothing to forward-fill).
// The statistics are taken per period on the bridged mask, runs cut at the period edges.
//
// A lane owns one (cell, period): it looks back at most min_gap-1 steps before the period to learn
// whether a gap open at the period start can still be bridged, walks the period keeping the in-period
// steps of the unresolved gap pending, and looks ahead at most min_gap-1 steps past the period end
// to resolve a gap that is still open there.
#include "runstat.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;

template <int OP>
__global__ void __launch_bounds__(kThreads)
period_runstat_gap_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                          const int32_t* __restrict__ poff, float thr, int32_t window, int32_t min_gap,
                          int32_t reducer, float* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const int Ti = (int)T;
  const float* col = x + c;
  auto m_at = [&](int t) -> bool { return cmp<OP>(ld_stream(col + (int64_t)t * ldx), thr); };

  // falses since the last True before t0, saturated at min_gap ("cannot be bridged any more")
  int since = 0;
  {
    int t = t0 - 1;
    while (t >= 0 && since < min_gap && !m_at(t)) { ++since; --t; }
    if (t < 0) since = min_gap;  // the series starts inside this gap (or at t0): never bridged
  }
  int cur = 0, pend = 0;
  RunAcc<kRunAny> acc;
  acc.init();
  for (int t = t0; t < t1; ++t) {
    if (m_at(t)) {
      if (since < min_gap) cur += pend;  // the gap just closed was short: its steps count as spell steps
      cur += 1;
      since = 0;
      pend = 0;
    } else {
      if (since < min_gap) {
        ++since;
        if (since < min_gap) {
          ++pend;                         // still bridgeable
        } else {                          // the gap reached min_gap: the run ended before it
          acc.add(cur, cur >= window);
          cur = 0;
          pend = 0;
        }
      }
    }
  }
  if (pend > 0) {  // a short gap is open at the period end: look ahead for its verdict
    int s2 = since, t = t1;
    bool bridged;
    for (;;) {
      if (t >= Ti) { bridged = true; break; }   // it runs into the end of the series
      if (m_at(t)) { bridged = true; break; }
      if (++s2 >= min_gap) { bridged = false; break; }
      ++t;
    }
    if (bridged) cur += pend;
  }
  acc.add(cur, cur >= window);
  out[(int64_t)p * C + c] = acc.result(reducer);
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int32_t xc_period_runstat_gap_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                             const int32_t* period_offsets, int32_t P, int32_t op, double thr,
                                             int32_t cmp_f64, int32_t reducer, int32_t window, int32_t min_gap,
                                             float* out, void* stream) {
  XC_REQUIRE(x && period_offsets && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1, "window must be >= 1, got %d", window);
  XC_REQUIRE(min_gap >= 1, "min_gap must be >= 1, got %d", min_gap);
  XC_REQUIRE(reducer >= XC_RL_MAX && reducer <= XC_RL_STD, "unknown run-length reducer %d", reducer);
  const float t32 = fold_threshold(op, thr, cmp_f64);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P, 1);
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_op_nan(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    period_runstat_gap_kernel<OP><<<grid, kThreads, 0, st>>>(x, T, C, ldx, period_offsets, t32, window, min_gap,
                                                             reducer, out);
    return launch_status("period_runstat_gap_kernel");
  });
}
