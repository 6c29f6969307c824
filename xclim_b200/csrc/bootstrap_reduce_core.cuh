// Reduction of the per-(year, replacement year) exceedance masks of the percentile bootstrap to the index of each
// in-base year: the spell duration indices, days over a precipitation percentile and the fraction of precipitation on
// those days (core/bootstrapping.py:182-203 with indices/_multivariate.py:69-153, 1174-1297, 1719-1795).
//
// The masks come from the MASK mode of the bootstrap kernels (bootstrap.cu): bit d of word (pair, d / 32) is set when
// day d of in-base year y beats P^(y<-s)(d), pair = y (N - 1) + (s < y ? s : s - 1).  The reference computes the index
// on year y's own slice of the series, so runs end at the year's edges.  __host__ __device__ so that a host build can
// test it (tests/csrc/bootstrap_reduce_host.cu).
#pragma once

#include "runstat.cuh"

namespace xc {

// bit d of one pair's mask, reading each word once
template <typename Word>
struct MaskBits {
  Word word;
  int pair, wi;
  uint32_t v;
  XC_RS_HD bool at(int d) {
    if ((d >> 5) != wi) {
      wi = d >> 5;
      v = word(pair, wi);
    }
    return (v >> (d & 31)) & 1u;
  }
};

// Every output period of in-base year y (step_period sp[0 .. L), non-decreasing: the periods nest in the year) over
// the N - 1 replacements s != y in s order.  word(pair, w): mask word; xval(d): x of day d of year y (SUM);
// wet(p): float32 wet-day total of period p (SUM); store_int(p, sum over s) for COUNT / SPELL;
// store_frac(p, float64 sum of the non-NaN float32 fractions in s order, their number) for SUM.
//   COUNT: days with the bit set.
//   SPELL: windowed_run_count, the days in runs of at least `window` set bits, with the period-edge rule of
//          PeriodMask (`after` = !resample_before_rl: a run belongs to the period of its first day and is cut
//          at the end of the year only).
//   SUM:   the float64 sum of x over the set days, in time order, rounded once to float32 and divided in
//          float32 by the wet total.
template <int RED, typename Word, typename XVal, typename Wet, typename StoreInt, typename StoreFrac>
XC_RS_HD void boot_reduce_year(int N, int L, int y, const int32_t* sp, int window, bool after, Word word, XVal xval,
                               Wet wet, StoreInt store_int, StoreFrac store_frac) {
  for (int d0 = 0; d0 < L;) {
    const int p = sp[d0];
    int d1 = d0 + 1;
    while (d1 < L && sp[d1] == p) ++d1;
    long long isum = 0;
    double fsum = 0.0;
    int nf = 0;
    for (int s = 0; s < N; ++s) {
      if (s == y) continue;
      MaskBits<Word> b{word, y * (N - 1) + (s < y ? s : s - 1), -1, 0u};
      if constexpr (RED == XC_BOOT_COUNT) {
        int n = 0;
        for (int d = d0; d < d1; ++d) n += b.at(d) ? 1 : 0;
        isum += n;
      } else if constexpr (RED == XC_BOOT_SPELL) {
        RunAcc<XC_RL_SUM> acc;
        acc.init();
        int32_t cur = 0;
        PeriodMask pm;
        pm.init();
        if (after && d0 > 0) pm.look_back(b.at(d0 - 1));
        for (int d = d0; d < d1; ++d) run_step(cur, acc, pm.inside(after, b.at(d)), window);
        if (after)
          for (int d = d1; cur > 0 && d < L; ++d) run_step(cur, acc, PeriodMask::past_end(b.at(d), cur > 0), window);
        run_close(cur, acc, window);
        isum += acc.a;
      } else {
        double sm = 0.0;
        for (int d = d0; d < d1; ++d)
          if (b.at(d)) sm += (double)xval(d);
        const float f = (float)sm / wet(p);
        if (f == f) {
          fsum += (double)f;
          ++nf;
        }
      }
    }
    if constexpr (RED == XC_BOOT_SUM)
      store_frac(p, fsum, nf);
    else
      store_int(p, isum);
    d0 = d1;
  }
}

// mean over the replacements: integers as sum / (N - 1) in float64 (numpy's mean of integers); fractions as the
// float64 mean of the non-NaN terms rounded once to float32, NaN when every term is NaN
XC_RS_HD double boot_int_mean(long long isum, int N) { return (double)isum / (double)(N - 1); }
XC_RS_HD float boot_frac_mean(double fsum, int nf) { return nf ? (float)(fsum / (double)nf) : NAN; }

}  // namespace xc
