// Percentile bootstrap (Zhang et al. 2005) of a day-of-year percentile exceedance count.
//
// Replaces core/bootstrapping.py:81-211 (`bootstrap_func`) + 235-282 (`build_bootstrap_year_da`):
// for every in-base year y and every other base year s the reference rebuilds the base series with
// block y overwritten by block s, recomputes percentile_doy on it (N*(N-1) full evaluations, each a
// rolling-construct + sort of the whole base period) and counts year y's exceedances against it.
//
// Here (uniform year length L, base = N blocks of L steps):
//   S(d)      = base sample of day d (W*N values, as in percentile_doy)
//   R_y(d)    = the <= W values of S(d) that sit in block y   (circular days d-h..d+h of year y)
//   I_s(d)    = the values of block s at the same positions
//   M(y,s,d)  = S(d) - R_y(d) + I_s(d)      -- the sample of day d in the altered series
// so P^(y<-s)(d) is a quantile of "the sorted top list of S(d), minus <= W values, plus <= W values":
// per (cell, day) the sorted extremes of S(d) are built ONCE (same register/shared-memory machinery
// as percentile_doy), per year the <= W removals are applied once, and per (y, s) pair only W
// insertions into a short list and one lerp remain.  Counts are accumulated per output period with
// integer atomics and divided by N-1 at the end (mean over the N-1 altered series,
// core/bootstrapping.py:203; numpy's int64 mean is exactly sum/(N-1) in float64).
#include <stdlib.h>

#include <type_traits>
#include <vector>

#include "common.cuh"
#include "quantile.cuh"
#include "sortnet.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;
#define XC_NEG_INF (__int_as_float(0xff800000))

template <int K>
__device__ __forceinline__ void insert_desc(float (&lst)[K], float v) {
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float hi = fmaxf(lst[k], v);
    v = fminf(lst[k], v);
    lst[k] = hi;
  }
}

// remove ONE instance of value r from the sorted list (no-op when absent; NaN never matches)
template <int K>
__device__ __forceinline__ void remove_one(float (&a)[K], float r) {
  bool found = false;
#pragma unroll
  for (int i = 0; i < K - 1; ++i) {
    found = found || (a[i] == r);
    a[i] = found ? a[i + 1] : a[i];
  }
  found = found || (a[K - 1] == r);
  a[K - 1] = found ? XC_NEG_INF : a[K - 1];
}

// Shared-memory layout per lane (column `lane` of every row):
//   sring [W-1][KA]  sorted (selection-side, masked) extremes of the W-1 previous day lists
//   scnt  [W-1]      their valid counts
//   raw   [W][N]     raw block values x[base + b*L + dd] of the W days of the current window
template <int KA, int KB, int OP>
__global__ void __launch_bounds__(kThreads)
bootstrap_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, int64_t base_start, int32_t N, int32_t L,
                 int32_t W, QuantSpec spec, const int32_t* __restrict__ step_period, int32_t doys_per_chunk,
                 int32_t* __restrict__ counts) {
  extern __shared__ float smem[];
  const int H = W / 2, R = W - 1;
  const int lane = threadIdx.x;
  float* sring = smem;
  int* scnt = reinterpret_cast<int*>(smem + (size_t)R * KA * kThreads);
  float* raw = smem + (size_t)R * (KA + 1) * kThreads;
  const int64_t c = (int64_t)blockIdx.x * kThreads + lane;
  if (c >= C) return;
  const int d0 = blockIdx.y * doys_per_chunk;
  const int d1 = min(L, d0 + doys_per_chunk);
  if (d0 >= d1) return;
  const unsigned wmask = __activemask();  // lanes of this warp that own a cell
  const bool top = spec.top != 0;
  const float sgn = top ? 1.f : -1.f;
  const float* xb = x + base_start * ldx + c;

  // Loads day e (may be < 0 or >= L: the window wraps into the neighbouring year), stores the raw
  // block values into raw slot `rs`, returns the sorted masked top-KA list + valid count.
  auto load_day = [&](int e, int rs, float (&lst)[KA], int& n) {
    const int dd = e < 0 ? e + L : (e >= L ? e - L : e);
    // block b contributes to S(.) through a step i of year b+1 (e < 0) / b-1 (e >= L) / b
    const int blo = (e >= L) ? 1 : 0;
    const int bhi = (e < 0) ? N - 1 : N;
    n = 0;
    bool first = true;
    for (int b0 = 0; b0 < N; b0 += KA) {
      float v[KA];
#pragma unroll
      for (int k = 0; k < KA; ++k) {
        const int b = b0 + k;
        float r = XC_NEG_INF;
        if (b < N) {
          const float xv = ld_stream(xb + ((int64_t)b * L + dd) * ldx);
          raw[((size_t)rs * N + b) * kThreads + lane] = xv;
          const bool ok = (b >= blo) && (b < bhi) && (xv == xv);
          n += ok ? 1 : 0;
          r = ok ? sgn * xv : XC_NEG_INF;
        }
        v[k] = r;
      }
      sort_desc<KA>(v);
      if (first) {
#pragma unroll
        for (int k = 0; k < KA; ++k) lst[k] = v[k];
        first = false;
      } else {
        merge_top_desc<KA>(lst, v);
      }
    }
  };

  float ynew[KA];
  int nnew;
  // prologue: days e = d0-H .. d0+H-1 ; sorted slot = (e - (d0-H)) mod R, raw slot = (e - (d0-H)) mod W
  for (int s = 0; s < R; ++s) {
    load_day(d0 - H + s, s % W, ynew, nnew);
#pragma unroll
    for (int k = 0; k < KA; ++k) sring[((size_t)s * KA + k) * kThreads + lane] = ynew[k];
    scnt[s * kThreads + lane] = nnew;
  }
  int oldest = 0;     // sorted-ring slot of day d-H
  int raw_first = 0;  // raw-ring slot of day d-H
  for (int d = d0; d < d1; ++d) {
    const int raw_new = (raw_first + W - 1) % W;
    load_day(d + H, raw_new, ynew, nnew);
    float tl[KA];
#pragma unroll
    for (int k = 0; k < KA; ++k) tl[k] = ynew[k];
    int nbase = nnew;
#pragma unroll 1
    for (int s = 0; s < R; ++s) {
      const float* slot = sring + (size_t)s * KA * kThreads + lane;
#pragma unroll
      for (int k = 0; k < KA; ++k) tl[k] = fmaxf(tl[k], slot[(size_t)(KA - 1 - k) * kThreads]);
      bitonic_finish_desc<KA>(tl);
      nbase += scnt[s * kThreads + lane];
    }
    // ---- every in-base year y: first a cheap, conservative test on ranks.  With M = S - R_y + I_s,
    // ge(M) = #{m >= x} lies in [geA, geA + W] (geA from S - R_y alone) and the two order statistics the
    // quantile interpolates sit at list indexes k1 and k1 + 1:  ge(M) <= k1 for every s  =>  x beats the
    // threshold for every s (count N-1);  gt(M) >= k1 + 2 for every s  =>  never.  Only the years whose
    // value lies within ~W ranks of the threshold ("in band", ~10 %) go through the exact per-(y, s)
    // evaluation, and each lane walks ITS OWN list of such years, so a warp iterates max-over-lanes
    // list length (~5) instead of N times.
    const int raw_mid = (raw_first + H) % W;
    unsigned band = 0u;
#pragma unroll 1
    for (int y = 0; y < N; ++y) {
      const float xq = raw[((size_t)raw_mid * N + y) * kThreads + lane];
      if (!(xq == xq)) continue;  // NaN never satisfies the comparison
      const float xs = sgn * xq;
      int geT = 0, gtT = 0;
#pragma unroll
      for (int k = 0; k < KA; ++k) {
        geT += (tl[k] >= xs) ? 1 : 0;
        gtT += (tl[k] > xs) ? 1 : 0;
      }
      int geR = 0, gtR = 0, nr = 0;
#pragma unroll 1
      for (int k = 0; k < W; ++k) {
        const int e = d - H + k;
        const bool valid = (e < 0) ? (y + 1 < N) : ((e >= L) ? (y >= 1) : true);
        if (!valid) continue;
        const float r = raw[((size_t)((raw_first + k) % W) * N + y) * kThreads + lane];
        if (r == r) {
          ++nr;
          geR += (sgn * r >= xs) ? 1 : 0;
          gtR += (sgn * r > xs) ? 1 : 0;
        }
      }
      // values below the kept list: geT saturates at KA, which is far beyond any k1 + 2 (KA >= KB + W)
      const int geA = geT - geR, gtA = (gtT == KA) ? KA : gtT - gtR;
      const int na = nbase - nr;
      const QuantIdx q0 = quant_index(na, spec), q1 = quant_index(na + W, spec);
      const bool ok0 = (na >= 2) && (q0.vi < (double)na - 1.0) && (q0.vi >= 0.0);
      const bool ok1 = (q1.vi < (double)(na + W) - 1.0) && (q1.vi >= 0.0);
      const int k1min = top ? (na - 2 - q0.ilo) : q0.ilo;
      const int k1max = top ? (na + W - 2 - q1.ilo) : q1.ilo;
      bool decided = false;
      if (ok0 && ok1 && N <= 32) {
        if (gtA >= k1max + 2) {
          decided = true;                       // never beats the threshold
        } else if (geT < KA && geA + W <= k1min) {
          decided = true;                       // beats it for every other year s
          atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, N - 1);
        }
      }
      if (!decided) band |= (N <= 32) ? (1u << y) : 0u;
    }
    // exact evaluation of the in-band years (all years when N > 32)
    int y_all = 0;
    while (true) {
      int y = -1;
      if (N <= 32) {
        if (band) { y = __ffs(band) - 1; band &= band - 1u; }
      } else if (y_all < N) {
        y = y_all++;
        const float xq0 = raw[((size_t)raw_mid * N + y) * kThreads + lane];
        if (!(xq0 == xq0)) y = -2;  // skip, but keep looping
      }
      if (!__any_sync(wmask, y != -1)) break;
      if (y < 0) continue;
      float a[KA];
#pragma unroll
      for (int k = 0; k < KA; ++k) a[k] = tl[k];
      int na = nbase;
      unsigned vmask = 0;  // window offsets whose position in block y belongs to S(d)
#pragma unroll 1
      for (int k = 0; k < W; ++k) {
        const int e = d - H + k;
        const bool valid = (e < 0) ? (y + 1 < N) : ((e >= L) ? (y >= 1) : true);
        if (!valid) continue;
        vmask |= 1u << k;
        const float r = raw[((size_t)((raw_first + k) % W) * N + y) * kThreads + lane];
        if (r == r) {
          remove_one<KA>(a, sgn * r);
          na -= 1;
        }
      }
      const float xq = raw[((size_t)raw_mid * N + y) * kThreads + lane];
      int cnt = 0;
#pragma unroll 1
      for (int s = 0; s < N; ++s) {
        if (s == y) continue;
        float bl[KB];
#pragma unroll
        for (int k = 0; k < KB; ++k) bl[k] = a[k];
        int nm = na;
#pragma unroll 1
        for (int k = 0; k < W; ++k) {
          if (!((vmask >> k) & 1u)) continue;
          const float v = raw[((size_t)((raw_first + k) % W) * N + s) * kThreads + lane];
          const bool ok = (v == v);
          nm += ok ? 1 : 0;
          insert_desc<KB>(bl, ok ? sgn * v : XC_NEG_INF);
        }
        const double p = finalize_quantile<KB>(bl, nm, spec);
        cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
      }
      if (cnt) atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, cnt);
    }
    // rotate the rings
#pragma unroll
    for (int k = 0; k < KA; ++k) sring[((size_t)oldest * KA + k) * kThreads + lane] = ynew[k];
    scnt[oldest * kThreads + lane] = nnew;
    oldest = (oldest + 1 == R) ? 0 : oldest + 1;
    raw_first = (raw_first + 1 == W) ? 0 : raw_first + 1;
  }
}


// ------------------------------------------------------------------------------------------------
// Window-5 kernel (KA = 16 kept extremes, quantile within the top 8): the same decomposition as
// bootstrap_kernel, with the exact per-(y, s) step turned into a RANK UPDATE instead of a rebuild.
//
// For an in-band year y the altered sample is M = A_y + I_s with A_y = S - R_y (sorted top list, built
// once per y) and I_s the five window values of year s.  The two order statistics the quantile
// interpolates are ranks k1+1 and k1+2 of a union of two sorted lists, i.e.
//     u_hi = max( a[k1],   min(a[k1-1], i1), min(a[k1-2], i2), ..., min(a[k1-5], i5) )
//     u_lo = max( a[k1+1], min(a[k1],   i1), min(a[k1-1], i2), ..., min(a[k1-4], i5) )
// (the max-min formula for the r-th largest of a union; a[<0] = +inf): 20 min/max on a sorted I_s, no
// insertion, no per-s list copy -- against ~150 instructions per (y, s) of the insert-and-finalize path.
// And only the OWNER years need it: when the largest window value of year s is <= a[k1+1] the union's two
// ranks are a[k1], a[k1+1] themselves, one threshold P0 shared by all such s (at most k1+1 years own a
// value above a[k1+1]).
// Classification of the years is two-staged: two compares against day-constant list entries settle
// "never" / "always" for most years (x below rank k1max+7 of S never beats a threshold; x above rank
// floor(k1min/2)+1 always does, because every value of year s that is >= x is itself a member of A_y,
// so #{I_s >= x} <= #{A_y >= x}); the rest go through the exact rank test of bootstrap_kernel.
// Irregular items (a NaN among the inserted values, windows reaching into the neighbouring year, plotting
// positions outside the sample) take the insert-and-finalize path of bootstrap_kernel verbatim, so the
// results stay bit-identical to it.
// Shared memory per lane: raw [5][N], the three largest window values of every year [3][N], scratch [KA]
// (544 bytes for N = 15: the sorted day lists are rebuilt from the raw ring instead of being kept, which
// trades 7 % more instructions for 50 % more resident warps in a latency-bound kernel).  N <= 16.
// ------------------------------------------------------------------------------------------------
#ifndef XC_BOOT_THREADS
#define XC_BOOT_THREADS 32
#endif
constexpr int kBT = XC_BOOT_THREADS;
constexpr float kPosInf = __builtin_huge_valf();

__device__ __forceinline__ void sort5_desc(float& a, float& b, float& c, float& d, float& e) {
  // 9-comparator network
  ce_desc(a, b); ce_desc(d, e); ce_desc(c, e); ce_desc(c, d); ce_desc(a, d);
  ce_desc(a, c); ce_desc(b, e); ce_desc(b, d); ce_desc(b, c);
}

// remove ONE instance of r from the sorted (descending) list: everything not above r moves up one slot.
// r is a member of the sample the list is the top of, so either it is in the list (one instance goes) or it
// lies below it (a[k] > r for every k: nothing moves).  Entries beyond rank K - #removals become inexact,
// like remove_one's; 2 K independent instructions instead of a K-long dependent chain.
template <int K>
__device__ __forceinline__ void remove_shift(float (&a)[K], float r) {
#pragma unroll
  for (int k = 0; k < K - 1; ++k) a[k] = (a[k] > r) ? a[k] : a[k + 1];
  a[K - 1] = (a[K - 1] > r) ? a[K - 1] : XC_NEG_INF;
}

// entry idx of a register list through a 4-level select tree (depth 4 instead of a 15-long chain)
__device__ __forceinline__ float pick16(const float (&l)[16], int idx) {
  float t8[8], t4[4];
#pragma unroll
  for (int i = 0; i < 8; ++i) t8[i] = (idx & 1) ? l[2 * i + 1] : l[2 * i];
#pragma unroll
  for (int i = 0; i < 4; ++i) t4[i] = (idx & 2) ? t8[2 * i + 1] : t8[2 * i];
  const float u0 = (idx & 4) ? t4[1] : t4[0], u1 = (idx & 4) ? t4[3] : t4[2];
  return (idx & 8) ? u1 : u0;
}

template <int OP>
__global__ void __launch_bounds__(kBT)
bootstrap5_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, int64_t base_start, int32_t N, int32_t L,
                  QuantSpec spec, const int32_t* __restrict__ step_period, int32_t doys_per_chunk,
                  int32_t* __restrict__ counts) {
  constexpr int KA = 16, KB = 8, W = 5, H = 2;
  extern __shared__ float smem[];
  const int lane = threadIdx.x;
  float* raw = smem;                                                       // [W][N][kBT] selection-side values
  float* stop = raw + (size_t)W * N * kBT;                                 // [3][N][kBT] three largest window values
  float* sa = stop + (size_t)3 * N * kBT;                                  // [KA][kBT] scratch (A_y)
  const int64_t c = (int64_t)blockIdx.x * kBT + lane;
  if (c >= C) return;
  const int d0 = blockIdx.y * doys_per_chunk;
  const int d1 = min(L, d0 + doys_per_chunk);
  if (d0 >= d1) return;
  const unsigned wmask = __activemask();
  const bool top = spec.top != 0;
  const float sgn = top ? 1.f : -1.f;
  const float* xb = x + base_start * ldx + c;
  const int64_t ystride = (int64_t)L * ldx;

  // day e (may reach into the neighbouring year) -> registers; stored to the raw ring one iteration later,
  // so that the load latency hides behind a whole day of work
  float pre[KA];
  auto issue_day = [&](int e) {
    const int dd = e < 0 ? e + L : (e >= L ? e - L : e);
    const float* p = xb + (int64_t)dd * ldx;
#pragma unroll
    for (int k = 0; k < KA; ++k) {
      pre[k] = (k < N) ? ld_stream(p) : 0.f;
      p += ystride;
    }
  };
  auto store_day = [&](int rs) {
#pragma unroll
    for (int k = 0; k < KA; ++k)
      if (k < N) raw[((size_t)rs * N + k) * kBT + lane] = sgn * pre[k];   // exact (sgn = +-1); NaN stays NaN
  };
  auto k1_of = [&](int n, bool& ok) {
    const QuantIdx q = quant_index(n, spec);
    ok = (n >= 2) && (q.vi < (double)n - 1.0) && (q.vi >= 0.0);
    return top ? (n - 2 - q.ilo) : q.ilo;
  };

  // sorted (descending, masked) list of the day in raw slot `rs` -- day e of the calendar year
  auto sort_day = [&](int e, int rs, float (&v)[KA], int& n) {
    const int blo = (e >= L) ? 1 : 0;
    const int bhi = (e < 0) ? N - 1 : N;
    const float* col = raw + ((size_t)rs * N) * kBT + lane;
    n = 0;
#pragma unroll
    for (int b = 0; b < KA; ++b) {
      const float r = (b < N) ? col[(size_t)b * kBT] : XC_NEG_INF;
      const bool ok = (b >= blo) && (b < bhi) && (r == r);
      n += ok ? 1 : 0;
      v[b] = ok ? r : XC_NEG_INF;
    }
    sort_desc<KA>(v);
  };
  // prologue: days d0-2 .. d0+1 into raw slots 0..3 and, sorted, into the four register lists; day d0+2 in flight.
  // The older day lists live in REGISTERS (64 of them) between days: only the entering day is sorted per
  // iteration (re-sorting all five from the raw ring cost 18 % of the instructions).
  float y0[KA], y1[KA], y2[KA], y3[KA];
  int n0, n1, n2, n3;
  for (int k = 0; k < W - 1; ++k) {
    issue_day(d0 - H + k);
    store_day(k);
  }
  sort_day(d0 - 2, 0, y0, n0);
  sort_day(d0 - 1, 1, y1, n1);
  sort_day(d0, 2, y2, n2);
  sort_day(d0 + 1, 3, y3, n3);
  issue_day(d0 + H);
  int raw_first = 0;
  for (int d = d0; d < d1; ++d) {
    store_day((raw_first + W - 1) % W);
    if (d + 1 < d1) issue_day(d + 1 + H);
    // ---- sorted extremes of the base sample S(d): four kept day lists + the entering one
    float tl[KA], ynew[KA];
    int nnew;
    sort_day(d + H, (raw_first + W - 1) % W, ynew, nnew);
#pragma unroll
    for (int b = 0; b < KA; ++b) tl[b] = y0[b];
    merge_top_desc<KA>(tl, y1);
    merge_top_desc<KA>(tl, y2);
    merge_top_desc<KA>(tl, y3);
    merge_top_desc<KA>(tl, ynew);
    const int nbase = n0 + n1 + n2 + n3 + nnew;
#pragma unroll
    for (int b = 0; b < KA; ++b) { y0[b] = y1[b]; y1[b] = y2[b]; y2[b] = y3[b]; y3[b] = ynew[b]; }
    n0 = n1; n1 = n2; n2 = n3; n3 = nnew;
    const bool interior = (d >= H) && (d + H < L);   // the window stays inside the year: every position valid
    // ---- day constants: list ranks of the interpolated order statistics over every possible count
    // na in [nbase - W, nbase] of A_y (k1 is non-decreasing in n), cf. the per-year test below
    bool okA, okB, okC;
    const int k1lo = k1_of(nbase - W, okA);            // smallest k1min over the years
    const int k1hi = k1_of(nbase + W, okB);            // largest k1max
    const int k1reg = k1_of(nbase, okC);               // regular item: na + W = nbase
    const bool day_ok = okA && okB && (nbase - W >= 2);
    // never: gtA >= k1max + 2  <=  gtT - W >= k1hi + 2  <=  xs < tl[k1hi + W + 1]
    // always: geT < KA and geA + slack <= k1min  <=  geT <= idx with 2 idx <= k1lo (interior) / idx + W <= k1lo
    const int i_never = k1hi + W + 1;
    const int i_always = interior ? (k1lo >> 1) : (k1lo - W);
    const float thr_never = (day_ok && i_never < KA) ? pick16(tl, i_never) : XC_NEG_INF;   // xs < -inf: never true
    const float thr_always = (day_ok && i_always >= 0 && i_always < KA) ? pick16(tl, i_always) : kPosInf;
    // ---- per year: three largest window values (selection side) and NaN flag; cheap classification
    const int raw_mid = (raw_first + H) % W;
    unsigned nanmask = 0u, maybe = 0u;
#pragma unroll 3
    for (int y = 0; y < N; ++y) {
      float m = XC_NEG_INF, m2 = XC_NEG_INF, m3 = XC_NEG_INF;
      bool bad = false;
#pragma unroll
      for (int k = 0; k < W; ++k) {
        const float r = raw[((size_t)k * N + y) * kBT + lane];
        bad = bad || !(r == r);
        m3 = fmaxf(m3, fminf(m2, r));     // fmaxf / fminf ignore a NaN operand (years with a NaN go the slow way)
        m2 = fmaxf(m2, fminf(m, r));
        m = fmaxf(m, r);
      }
      stop[((size_t)0 * N + y) * kBT + lane] = m;
      stop[((size_t)1 * N + y) * kBT + lane] = m2;
      stop[((size_t)2 * N + y) * kBT + lane] = m3;
      nanmask |= bad ? (1u << y) : 0u;
      const float xs = raw[((size_t)raw_mid * N + y) * kBT + lane];
      if (xs == xs) {
        if (xs > thr_always) {
          atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, N - 1);
        } else if (!(xs < thr_never)) {
          maybe |= 1u << y;
        }
      }
    }
    // ---- exact rank test of the undecided years
    unsigned band = 0u;
    while (true) {
      int y = -1;
      if (maybe) { y = __ffs(maybe) - 1; maybe &= maybe - 1u; }
      if (!__any_sync(wmask, y != -1)) break;
      if (y < 0) continue;
      const float xs = raw[((size_t)raw_mid * N + y) * kBT + lane];
      int geR = 0, gtR = 0, nr = 0;
#pragma unroll
      for (int k = 0; k < W; ++k) {
        const int e = d - H + k;
        const bool valid = (e < 0) ? (y + 1 < N) : ((e >= L) ? (y >= 1) : true);
        const float r = raw[((size_t)((raw_first + k) % W) * N + y) * kBT + lane];
        if (valid && r == r) {
          ++nr;
          geR += (r >= xs) ? 1 : 0;
          gtR += (r > xs) ? 1 : 0;
        }
      }
      const int na = nbase - nr;
      bool ok0 = okA, ok1 = okC;               // nr == W (no missing value of year y): the day constants
      int k1min = k1lo, k1max = k1reg;
      if (nr != W) {
        k1min = k1_of(na, ok0);
        k1max = k1_of(na + W, ok1);
      }
      ok0 = ok0 && (na >= 2);
      // bootstrap_kernel's test on geT = #{tl >= xs}, gtT = #{tl > xs} (tl sorted, counts saturate at KA):
      //   never : gtA >= k1max + 2, gtA = (gtT == KA) ? KA : gtT - gtR   <=>  gtT >= min(KA, k1max + 2 + gtR)
      //                                                               <=>  xs < tl[min(KA, k1max + 2 + gtR) - 1]
      //   always: geT < KA and geA + slack <= k1min, geA = geT - geR, slack = interior ? min(W, geA) : W
      //           <=>  geA <= gmax := interior ? max(k1min - W, k1min >> 1) : k1min - W   (geA >= 0)
      //           <=>  geT <= min(KA - 1, gmax + geR)  <=>  xs > tl[min(KA - 1, gmax + geR)]
      bool decided = false;
      if (ok0 && ok1) {
        const int jn = min(KA, k1max + 2 + gtR) - 1;
        const int gmax = interior ? max(k1min - W, k1min >> 1) : (k1min - W);
        const int ja = min(KA - 1, gmax + geR);
        const float tn = pick16(tl, jn < 0 ? 0 : jn), ta = pick16(tl, ja < 0 ? 0 : ja);
        if (jn >= 0 && xs < tn) {
          decided = true;
        } else if (gmax >= 0 && xs > ta) {
          decided = true;
          atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, N - 1);
        }
      }
      if (!decided) band |= (1u << y);
    }
    // ---- exact evaluation of the in-band years
    while (true) {
      int y = -1;
      if (band) { y = __ffs(band) - 1; band &= band - 1u; }
      if (!__any_sync(wmask, y != -1)) break;
      if (y < 0) continue;
      float a[KA];
#pragma unroll
      for (int k = 0; k < KA; ++k) a[k] = tl[k];
      int na = nbase;
      unsigned vmask = 0;
#pragma unroll
      for (int k = 0; k < W; ++k) {
        const int e = d - H + k;
        const bool valid = (e < 0) ? (y + 1 < N) : ((e >= L) ? (y >= 1) : true);
        const float r = raw[((size_t)((raw_first + k) % W) * N + y) * kBT + lane];
        if (valid) {
          vmask |= 1u << k;
          if (r == r) {
            remove_shift<KA>(a, r);
            na -= 1;
          }
        }
      }
      const float xq = sgn * raw[((size_t)raw_mid * N + y) * kBT + lane];   // the data value itself
      // regular item: all five positions valid, the quantile of na + 5 values interpolates list ranks
      // k1+1, k1+2 with k1 + 1 <= KA - 1 - W (those ranks of A_y are exact after the removals)
      const int nm0 = na + W;
      bool okm;
      const int k1 = (nm0 == nbase) ? k1reg : k1_of(nm0, okm);
      if (nm0 == nbase) okm = okC;
      const bool regular = interior && okm && k1 >= 0 && (k1 + 1 <= KA - 1 - W);
      const QuantIdx qm = quant_index(nm0, spec);
      float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f, b4 = 0.f, b5 = 0.f, b6 = 0.f;
      const unsigned all = (N >= 32) ? ~0u : ((1u << N) - 1u);
      unsigned slow = all & ~(1u << y);          // years evaluated by insert-and-finalize
      int cnt = 0;
      if (regular) {
#pragma unroll
        for (int k = 0; k < KA; ++k) sa[(size_t)k * kBT + lane] = a[k];
        auto at = [&](int idx) { return idx >= 0 ? sa[(size_t)idx * kBT + lane] : kPosInf; };
        b0 = at(k1 + 1); b1 = at(k1); b2 = at(k1 - 1); b3 = at(k1 - 2);
        b4 = at(k1 - 3); b5 = at(k1 - 4); b6 = at(k1 - 5);
        // years whose largest window value is <= a[k1+1] leave the two ranks at a[k1], a[k1+1]
        const double p0 = top ? quant_lerp(b0, b1, qm) : quant_lerp(-b1, -b0, qm);
        const int t0 = cmpd<OP>((double)xq, p0) ? 1 : 0;
        unsigned owners = 0u, deep = 0u;
#pragma unroll 5
        for (int s = 0; s < N; ++s) {
          owners |= (stop[((size_t)0 * N + s) * kBT + lane] > b0) ? (1u << s) : 0u;
          deep |= (stop[((size_t)2 * N + s) * kBT + lane] > b0) ? (1u << s) : 0u;   // three or more values above a[k1+1]
        }
        const unsigned others = all & ~(1u << y) & ~nanmask;
        cnt = t0 * __popc(others & ~owners);
        unsigned todo = others & owners & ~deep;
        unsigned full = others & deep;
        slow = all & ~(1u << y) & nanmask;
        while (todo) {     // at most two values of year s above a[k1+1]: every other term min(a[.], i_j) <= a[k1+1]
          const int s = __ffs(todo) - 1;
          todo &= todo - 1u;
          const float i1 = stop[((size_t)0 * N + s) * kBT + lane], i2 = stop[((size_t)1 * N + s) * kBT + lane];
          const float uhi = fmaxf(b1, fmaxf(fminf(b2, i1), fminf(b3, i2)));
          const float ulo = fmaxf(b0, fmaxf(fminf(b1, i1), fminf(b2, i2)));
          const double p = top ? quant_lerp(ulo, uhi, qm) : quant_lerp(-uhi, -ulo, qm);
          cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
        }
        while (full) {     // rare: the whole sorted window
          const int s = __ffs(full) - 1;
          full &= full - 1u;
          float j1 = raw[((size_t)0 * N + s) * kBT + lane], j2 = raw[((size_t)1 * N + s) * kBT + lane],
                j3 = raw[((size_t)2 * N + s) * kBT + lane], j4 = raw[((size_t)3 * N + s) * kBT + lane],
                j5 = raw[((size_t)4 * N + s) * kBT + lane];
          sort5_desc(j1, j2, j3, j4, j5);
          const float uhi = fmaxf(fmaxf(fmaxf(b1, fminf(b2, j1)), fmaxf(fminf(b3, j2), fminf(b4, j3))),
                                  fmaxf(fminf(b5, j4), fminf(b6, j5)));
          const float ulo = fmaxf(fmaxf(fmaxf(b0, fminf(b1, j1)), fmaxf(fminf(b2, j2), fminf(b3, j3))),
                                  fmaxf(fminf(b4, j4), fminf(b5, j5)));
          const double p = top ? quant_lerp(ulo, uhi, qm) : quant_lerp(-uhi, -ulo, qm);
          cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
        }
      }
      while (slow) {   // insert-and-finalize (bootstrap_kernel's exact step)
        const int s = __ffs(slow) - 1;
        slow &= slow - 1u;
        float bl[KB];
#pragma unroll
        for (int k = 0; k < KB; ++k) bl[k] = a[k];
        int nm = na;
#pragma unroll 1
        for (int k = 0; k < W; ++k) {
          if (!((vmask >> k) & 1u)) continue;
          const float v = raw[((size_t)((raw_first + k) % W) * N + s) * kBT + lane];
          const bool ok = (v == v);
          nm += ok ? 1 : 0;
          insert_desc<KB>(bl, ok ? v : XC_NEG_INF);
        }
        const double p = finalize_quantile<KB>(bl, nm, spec);
        cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
      }
      if (cnt) atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, cnt);
    }
    raw_first = (raw_first + 1 == W) ? 0 : raw_first + 1;
  }
}

int32_t launch_bootstrap5(int32_t op, const float* x, int64_t C, int64_t ldx, int64_t base_start, int32_t N, int32_t L,
                          const QuantSpec& spec, const int32_t* step_period, int32_t* counts, cudaStream_t st) {
  const int64_t cblocks = (C + kBT - 1) / kBT;
  int chunks = (int)((sm_count() * 12 + cblocks - 1) / cblocks);
  chunks = chunks < 1 ? 1 : chunks;
  int per = (L + chunks - 1) / chunks;
  if (per < 20) per = 20;
  if (per > L) per = L;
  chunks = (L + per - 1) / per;
  const size_t smem = ((size_t)8 * N + 16) * kBT * 4;
  if (smem > 227 * 1024) return 1;
  dim3 grid((unsigned)cblocks, (unsigned)chunks, 1);
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    if (smem > 48 * 1024) {
      cudaError_t e = cudaFuncSetAttribute(bootstrap5_kernel<OP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(bootstrap5_kernel)");
    }
    bootstrap5_kernel<OP><<<grid, kBT, smem, st>>>(x, C, ldx, base_start, N, L, spec, step_period, per, counts);
    return launch_status("bootstrap5_kernel");
  });
}

__global__ void __launch_bounds__(256)
bootstrap_finish_kernel(const int32_t* __restrict__ counts, int64_t n, double denom, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (double)counts[i] / denom;
}

template <int KA, int KB>
int32_t launch_bootstrap(int32_t op, const float* x, int64_t C, int64_t ldx, int64_t base_start, int32_t N,
                         int32_t L, int32_t W, const QuantSpec& spec, const int32_t* step_period, int32_t* counts,
                         cudaStream_t st) {
  const int64_t cblocks = (C + kThreads - 1) / kThreads;
  int chunks = (int)((sm_count() * 6 + cblocks - 1) / cblocks);
  chunks = chunks < 1 ? 1 : chunks;
  int per = (L + chunks - 1) / chunks;
  if (per < 4 * W) per = 4 * W;
  if (per > L) per = L;
  chunks = (L + per - 1) / per;
  const size_t smem = ((size_t)(W - 1) * (KA + 1) + (size_t)W * N) * kThreads * 4;
  if (smem > 227 * 1024) {
    set_error("bootstrap: %d base years x window %d need %zu bytes of shared memory per block", N, W, smem);
    return XC_ERR_UNSUPPORTED;
  }
  dim3 grid((unsigned)cblocks, (unsigned)chunks, 1);
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    if (smem > 48 * 1024) {
      cudaError_t e = cudaFuncSetAttribute(bootstrap_kernel<KA, KB, OP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem);
      if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(bootstrap_kernel)");
    }
    bootstrap_kernel<KA, KB, OP><<<grid, kThreads, smem, st>>>(x, C, ldx, base_start, N, L, W, spec, step_period, per,
                                                               counts);
    return launch_status("bootstrap_kernel");
  });
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int32_t xc_bootstrap_doy_count_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int64_t base_start,
                                              int32_t n_base_years, int32_t year_len, const int32_t* step_period,
                                              int32_t P, int32_t window, double percentile, double alpha,
                                              double beta, int32_t op, int32_t* count_scratch, double* out,
                                              void* stream) {
  XC_REQUIRE(x && step_period && count_scratch && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0, "bad shape");
  XC_REQUIRE(n_base_years >= 2 && year_len >= 1, "bootstrap needs at least two base years");
  XC_REQUIRE(base_start >= 0 && base_start + (int64_t)n_base_years * year_len <= T, "base period outside the series");
  XC_REQUIRE(window >= 1 && window % 2 == 1 && window <= 31 && window <= year_len, "window must be odd and <= 31");
  XC_REQUIRE(op == XC_OP_GT || op == XC_OP_GE || op == XC_OP_LT || op == XC_OP_LE,
             "Operation `%d` not permitted for indice.", op);
  cudaStream_t st = (cudaStream_t)stream;
  QuantSpec spec;
  const int need = plan_quantile(percentile, alpha, beta, n_base_years * window, &spec);
  XC_CHECK_CUDA(cudaMemsetAsync(count_scratch, 0, (size_t)P * C * 4, st));
  int32_t e = 1;
  if (need > 0 && need <= 8 && window == 5 && n_base_years <= 16 && year_len > 8 && !getenv("XCLIM_B200_BOOT_V1"))
    e = launch_bootstrap5(op, x, C, ldx, base_start, n_base_years, year_len, spec, step_period, count_scratch, st);
  if (e != 1) {
  } else if (need > 0 && need <= 8 && need + window <= 16)
    e = launch_bootstrap<16, 8>(op, x, C, ldx, base_start, n_base_years, year_len, window, spec, step_period,
                                count_scratch, st);
  else if (need > 0 && need <= 16 && need + window <= 32)
    e = launch_bootstrap<32, 16>(op, x, C, ldx, base_start, n_base_years, year_len, window, spec, step_period,
                                 count_scratch, st);
  else if (need > 0 && need + window <= 32)
    e = launch_bootstrap<32, 32>(op, x, C, ldx, base_start, n_base_years, year_len, window, spec, step_period,
                                 count_scratch, st);
  else {
    set_error("bootstrap: percentile %g of %d samples needs %d order statistics (+%d removals); at most 32 are kept",
              percentile, n_base_years * window, need, window);
    return XC_ERR_UNSUPPORTED;
  }
  if (e) return e;
  const int64_t n = (int64_t)P * C;
  bootstrap_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(count_scratch, n, (double)(n_base_years - 1),
                                                                      out);
  return launch_status("bootstrap_finish_kernel");
}
