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
//
// The same kernels in MASK mode keep the (y, s) identity instead: they set bit d of year y's mask word for pair
// (y, s) when day d beats P^(y<-s)(d), and bootstrap_reduce_kernel turns the masks into the spell and sum indices
// (bootstrap_reduce_core.cuh).  Their day chunks start on multiples of 32 days, so that each mask word has one
// writing thread and a plain read-modify-write after the memset needs no atomics.
#include <stdlib.h>

#include <type_traits>
#include <vector>

#include "bootstrap_reduce_core.cuh"
#include "common.cuh"
#include "launch_plan.cuh"
#include "quantile.cuh"
#include "sortnet.cuh"

namespace xc {
namespace {

// output of the exceedance kernels: per-period counts (tx90p & family) or per-(y, s) day masks
constexpr int kCount = 0, kMask = 1;

// MASK mode: mask [N (N - 1)][Wd][C] words, floor the threshold floor (-inf: none)
struct MaskOut {
  uint32_t* mask;
  int32_t Wd;
  double floor;
};
__device__ __forceinline__ bool has_floor(double floor) { return floor > (double)XC_NEG_INF; }
// max(P, floor), a NaN percentile taking the floor (`pr_per.where(pr_per > thresh, thresh)`); no floor: P
__device__ __forceinline__ double floored(double p, double floor) {
  return (has_floor(floor) && !(p > floor)) ? floor : p;
}
__device__ __forceinline__ void set_pair_bit(const MaskOut& mo, int64_t C, int64_t c, int N, int y, int s, int d) {
  const int64_t pair = (int64_t)y * (N - 1) + (s < y ? s : s - 1);
  uint32_t* w = mo.mask + (pair * mo.Wd + (d >> 5)) * C + c;
  *w |= 1u << (d & 31);
}
// x beats P^(y<-s) for every s: the mask bit is x op floor (x op max(P, f) == x op P && x op f for > / >=)
template <int OP>
__device__ __forceinline__ void set_year_bits(const MaskOut& mo, int64_t C, int64_t c, int N, int y, int d, double x) {
  if (has_floor(mo.floor) && !cmpd<OP>(x, mo.floor)) return;
  for (int s = 0; s < N; ++s)
    if (s != y) set_pair_bit(mo, C, c, N, y, s, d);
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

// The rank shortcuts of both kernels count "x beats the threshold" on the selection side, which is the
// operator's side only for >, >= with the top list and <, <= with the bottom one; any other pairing (a tx90p
// count against a low percentile) evaluates every year exactly.  They also assume that the threshold of every
// altered sample lies between its two neighbours.  An infinite neighbour, or two neighbours whose difference overflows float32, breaks that (the
// lerp can give +-inf, or NaN -> the sample maximum), so such a day sends every year through the exact
// per-(y, s) evaluation.  On interior days every neighbour is among the min(nbase, K) values at the top of tl
// (the selection side of S(d)); near the ends of the year block s can bring in a value from outside S(d), so
// there the whole raw window ([W][N] rows `stride` apart from `raw`) is checked.
template <int OP>
__device__ __forceinline__ bool rank_side(bool top) {
  return top == (OP == XC_OP_GT || OP == XC_OP_GE);
}
// interior days: hi = tl[0], lo = the last valid entry of tl
__device__ __forceinline__ bool span_overflows(float hi, float lo) { return !isfinite(__fsub_rn(hi, lo)); }
// days near the ends of the year ([count] values `stride` apart); out of line to keep the kernels' registers
__device__ __noinline__ bool raw_span_overflows(const float* raw, int stride, int count) {
  float hi = XC_NEG_INF, lo = -XC_NEG_INF;
  for (int i = 0; i < count; ++i) {
    const float v = raw[(size_t)i * stride];
    hi = fmaxf(hi, v);
    lo = fminf(lo, v);
  }
  return span_overflows(hi, lo);
}

// Largest value of the altered sample M(y, s, d): the window values of every block but y, plus block s's at
// the positions y contributes (vmask) -- the NaN-interpolation fallback (lerp_is_nan), rarely taken.  raw:
// this lane's [W][N] ring (rows `stride` apart, slot of day d-H = raw_first) holding sgn * x.
__device__ __noinline__ float altered_max(const float* raw, int stride, int raw_first, int W, int N, int L, int d,
                                          int y, int s, unsigned vmask, float sgn) {
  const int H = W / 2;
  float m = XC_NEG_INF;
  for (int k = 0; k < W; ++k) {
    const int e = d - H + k;
    const float* row = raw + (size_t)((raw_first + k) % W) * N * stride;
    for (int b = 0; b < N; ++b) {
      const bool valid = (e < 0) ? (b + 1 < N) : ((e >= L) ? (b >= 1) : true);
      if (valid && b != y) m = fmaxf(m, sgn * row[(size_t)b * stride]);
    }
    if ((vmask >> k) & 1u) m = fmaxf(m, sgn * row[(size_t)s * stride]);
  }
  return m;
}

// Shared-memory layout per lane (column `lane` of every row):
//   sring [W-1][KA]  sorted (selection-side, masked) extremes of the W-1 previous day lists
//   scnt  [W-1]      their valid counts
//   raw   [W][N]     raw block values x[base + b*L + dd] of the W days of the current window
template <int KA, int KB, int OP, int MODE>
__global__ void __launch_bounds__(kThreads)
bootstrap_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, int64_t base_start, int32_t N, int32_t L,
                 int32_t W, QuantSpec spec, const int32_t* __restrict__ step_period, int32_t doys_per_chunk,
                 int32_t* __restrict__ counts, MaskOut mo) {
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

  int raw_first = 0;  // raw-ring slot of day d-H
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
    const bool hostile = !rank_side<OP>(top) ||
                         ((d >= H) && (d + H < L) ? nbase > 0 && span_overflows(tl[0], pick<KA>(tl, min(nbase, KA) - 1))
                                                  : raw_span_overflows(raw + lane, kThreads, W * N));
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
      if (ok0 && ok1 && N <= kBootExactAbove && !hostile) {
        if (gtA >= k1max + 2) {
          decided = true;                       // never beats the threshold
        } else if (geT < KA && geA + W <= k1min) {
          decided = true;                       // beats it for every other year s
          if constexpr (MODE == kCount) atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, N - 1);
          else set_year_bits<OP>(mo, C, c, N, y, d, (double)xq);
        }
      }
      if (!decided) band |= (N <= kBootExactAbove) ? (1u << y) : 0u;
    }
    // exact evaluation of the in-band years (all years when N > kBootExactAbove)
    int y_all = 0;
    while (true) {
      int y = -1;
      if (N <= kBootExactAbove) {
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
        double p = finalize_quantile<KB>(bl, nm, spec);
        if (lerp_is_nan(p, nm)) p = altered_max(raw + lane, kThreads, raw_first, W, N, L, d, y, s, vmask, 1.f);
        if constexpr (MODE == kCount) cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
        else if (cmpd<OP>((double)xq, floored(p, mo.floor))) set_pair_bit(mo, C, c, N, y, s, d);
      }
      if (cnt) atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, cnt);
    }
    // rotate the rings (window 1 keeps no sorted ring: R == 0 slots)
    if (R > 0) {
#pragma unroll
      for (int k = 0; k < KA; ++k) sring[((size_t)oldest * KA + k) * kThreads + lane] = ynew[k];
      scnt[oldest * kThreads + lane] = nnew;
      oldest = (oldest + 1 == R) ? 0 : oldest + 1;
    }
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

template <int OP, int MODE>
__global__ void __launch_bounds__(kBT)
bootstrap5_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, int64_t base_start, int32_t N, int32_t L,
                  QuantSpec spec, const int32_t* __restrict__ step_period, int32_t doys_per_chunk,
                  int32_t* __restrict__ counts, MaskOut mo) {
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
    const bool hostile = !rank_side<OP>(top) ||
                         (interior ? nbase > 0 && span_overflows(tl[0], pick16(tl, min(nbase, KA) - 1))
                                   : raw_span_overflows(raw + lane, kBT, W * N));
    // ---- day constants: list ranks of the interpolated order statistics over every possible count
    // na in [nbase - W, nbase] of A_y (k1 is non-decreasing in n), cf. the per-year test below
    bool okA, okB, okC;
    const int k1lo = k1_of(nbase - W, okA);            // smallest k1min over the years
    const int k1hi = k1_of(nbase + W, okB);            // largest k1max
    const int k1reg = k1_of(nbase, okC);               // regular item: na + W = nbase
    const bool day_ok = okA && okB && (nbase - W >= 2) && !hostile;
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
          if constexpr (MODE == kCount) atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, N - 1);
          else set_year_bits<OP>(mo, C, c, N, y, d, (double)(sgn * xs));
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
      ok0 = ok0 && (na >= 2) && !hostile;
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
          if constexpr (MODE == kCount) atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, N - 1);
          else set_year_bits<OP>(mo, C, c, N, y, d, (double)(sgn * xs));
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
      const bool regular = interior && !hostile && okm && k1 >= 0 && (k1 + 1 <= KA - 1 - W);
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
        if constexpr (MODE == kCount) {
          cnt = t0 * __popc(others & ~owners);
        } else if (cmpd<OP>((double)xq, floored(p0, mo.floor))) {
          for (unsigned m = others & ~owners; m; m &= m - 1u) set_pair_bit(mo, C, c, N, y, __ffs(m) - 1, d);
        }
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
          if constexpr (MODE == kCount) cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
          else if (cmpd<OP>((double)xq, floored(p, mo.floor))) set_pair_bit(mo, C, c, N, y, s, d);
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
          if constexpr (MODE == kCount) cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
          else if (cmpd<OP>((double)xq, floored(p, mo.floor))) set_pair_bit(mo, C, c, N, y, s, d);
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
        double p = finalize_quantile<KB>(bl, nm, spec);
        if (lerp_is_nan(p, nm)) p = altered_max(raw + lane, kBT, raw_first, W, N, L, d, y, s, vmask, sgn);
        if constexpr (MODE == kCount) cnt += cmpd<OP>((double)xq, p) ? 1 : 0;
        else if (cmpd<OP>((double)xq, floored(p, mo.floor))) set_pair_bit(mo, C, c, N, y, s, d);
      }
      if (cnt) atomicAdd(counts + (int64_t)step_period[y * L + d] * C + c, cnt);
    }
    raw_first = (raw_first + 1 == W) ? 0 : raw_first + 1;
  }
}

__global__ void __launch_bounds__(256)
bootstrap_finish_kernel(const int32_t* __restrict__ counts, int64_t n, double denom, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (double)counts[i] / denom;
}

template <int KA, int KB, int MODE>
int32_t launch_bootstrap(const BootPlan& p, int32_t op, const float* x, int64_t C, int64_t ldx, int64_t base_start,
                         int32_t N, int32_t L, int32_t W, const int32_t* step_period, int32_t* counts,
                         const MaskOut& mo, cudaStream_t st) {
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    auto kern = bootstrap_kernel<KA, KB, decltype(OPC)::value, MODE>;
    if (int32_t e = allow_smem(kern, p.smem, "cudaFuncSetAttribute(bootstrap_kernel)")) return e;
    kern<<<dim3((unsigned)p.cblocks, (unsigned)p.split.chunks, 1), kThreads, p.smem, st>>>(
        x, C, ldx, base_start, N, L, W, p.spec, step_period, p.split.per, counts, mo);
    return launch_status("bootstrap_kernel");
  });
}

// The exceedance kernel of plan_bootstrap: the same choice in both modes
template <int MODE>
int32_t launch_exceedance(const float* x, int64_t C, int64_t ldx, int64_t base_start, int32_t N, int32_t L,
                          int32_t window, double percentile, double alpha, double beta, int32_t op,
                          const int32_t* step_period, int32_t* counts, const MaskOut& mo, cudaStream_t st) {
  BootPlan p;
  const int32_t ep = plan_bootstrap(N, L, window, percentile, alpha, beta, MODE == kMask,
                                    getenv("XCLIM_B200_BOOT_V1") != nullptr, C, sm_count(), &p);
  if (ep) return ep;
  if (p.kernel == kBoot5)
    return dispatch_op(op, [&](auto OPC) -> int32_t {
      auto kern = bootstrap5_kernel<decltype(OPC)::value, MODE>;
      if (int32_t e = allow_smem(kern, p.smem, "cudaFuncSetAttribute(bootstrap5_kernel)")) return e;
      kern<<<dim3((unsigned)p.cblocks, (unsigned)p.split.chunks, 1), kBT, p.smem, st>>>(
          x, C, ldx, base_start, N, L, p.spec, step_period, p.split.per, counts, mo);
      return launch_status("bootstrap5_kernel");
    });
#define XC_BOOT(E) launch_bootstrap<kBoot[E].ka, kBoot[E].kb, MODE>(p, op, x, C, ldx, base_start, N, L, window, \
                                                                  step_period, counts, mo, st)
  if (p.kernel == kBoot16x8) return XC_BOOT(kBoot16x8);
  if (p.kernel == kBoot32x16) return XC_BOOT(kBoot32x16);
  return XC_BOOT(kBoot32x32);
#undef XC_BOOT
}

// One lane per (cell, in-base year y = blockIdx.y): year y's index against each altered table, averaged
// (bootstrap_reduce_core.cuh).  mask: [N (N - 1)][Wd][C]; x, wet, out: the tile's first cell, rows ldx / ldo apart.
template <int RED>
__global__ void __launch_bounds__(kThreads)
bootstrap_reduce_kernel(const uint32_t* __restrict__ mask, int64_t C, int32_t Wd, int32_t N, int32_t L,
                        const int32_t* __restrict__ step_period, int32_t window, int32_t after,
                        const float* __restrict__ x, int64_t ldx, int64_t base_start,
                        const float* __restrict__ wet, int64_t ldo, void* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int y = blockIdx.y;
  const float* xy = x + (base_start + (int64_t)y * L) * ldx + c;
  auto word = [&](int pair, int w) { return __ldg(mask + ((int64_t)pair * Wd + w) * C + c); };
  auto xval = [&](int d) { return __ldg(xy + (int64_t)d * ldx); };
  auto wetp = [&](int p) { return __ldg(wet + (int64_t)p * ldo + c); };
  auto store_int = [&](int p, long long isum) {
    static_cast<double*>(out)[(int64_t)p * ldo + c] = boot_int_mean(isum, N);
  };
  auto store_frac = [&](int p, double fsum, int nf) {
    static_cast<float*>(out)[(int64_t)p * ldo + c] = boot_frac_mean(fsum, nf);
  };
  boot_reduce_year<RED>(N, L, y, step_period + (int64_t)y * L, window, after != 0, word, xval, wetp, store_int,
                        store_frac);
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
  XC_CHECK_CUDA(cudaMemsetAsync(count_scratch, 0, (size_t)P * C * 4, st));
  const int32_t e = launch_exceedance<kCount>(x, C, ldx, base_start, n_base_years, year_len, window, percentile, alpha,
                                              beta, op, step_period, count_scratch, MaskOut{nullptr, 0, 0.0}, st);
  if (e) return e;
  const int64_t n = (int64_t)P * C;
  bootstrap_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(count_scratch, n, (double)(n_base_years - 1),
                                                                      out);
  return launch_status("bootstrap_finish_kernel");
}

static int64_t mask_bytes_per_cell(int32_t N, int32_t L) { return (int64_t)N * (N - 1) * ((L + 31) / 32) * 4; }

extern "C" int64_t xc_bootstrap_doy_index_scratch_bytes(int32_t n_base_years, int32_t year_len, int64_t C) {
  if (n_base_years < 2 || year_len < 1 || C < 1) return 0;
  return mask_bytes_per_cell(n_base_years, year_len) * C;
}

extern "C" int32_t xc_bootstrap_doy_index_f32(const float* x, int64_t T, int64_t C, int64_t ldx, int64_t base_start,
                                              int32_t n_base_years, int32_t year_len, const int32_t* step_period,
                                              int32_t P, int32_t window, double percentile, double alpha,
                                              double beta, int32_t op, int32_t reducer, int32_t run_window,
                                              int32_t resample_before_rl, double floor, const float* wet_total,
                                              void* scratch, int64_t scratch_bytes, void* out, void* stream) {
  XC_REQUIRE(x && step_period && scratch && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0, "bad shape");
  XC_REQUIRE(n_base_years >= 2 && year_len >= 1, "bootstrap needs at least two base years");
  XC_REQUIRE(base_start >= 0 && base_start + (int64_t)n_base_years * year_len <= T, "base period outside the series");
  XC_REQUIRE(window >= 1 && window % 2 == 1 && window <= 31 && window <= year_len, "window must be odd and <= 31");
  XC_REQUIRE(op == XC_OP_GT || op == XC_OP_GE || op == XC_OP_LT || op == XC_OP_LE,
             "Operation `%d` not permitted for indice.", op);
  XC_REQUIRE(reducer == XC_BOOT_COUNT || reducer == XC_BOOT_SPELL || reducer == XC_BOOT_SUM,
             "unknown bootstrap index %d", reducer);
  XC_REQUIRE(reducer != XC_BOOT_SPELL || run_window >= 1, "run window must be >= 1");
  XC_REQUIRE(!(floor != floor), "floor must not be NaN");
  XC_REQUIRE(floor == (double)-INFINITY || op == XC_OP_GT || op == XC_OP_GE, "a threshold floor needs op > or >=");
  XC_REQUIRE((wet_total != nullptr) == (reducer == XC_BOOT_SUM), "wet_total is given exactly for XC_BOOT_SUM");
  XC_REQUIRE(((uintptr_t)scratch & 15) == 0, "scratch must be 16-byte aligned");
  const int32_t N = n_base_years, L = year_len, Wd = (L + 31) / 32;
  const int64_t per_cell = mask_bytes_per_cell(N, L);
  const int64_t fit = scratch_bytes > 0 ? scratch_bytes / per_cell : 0;
  const int64_t tile = fit >= C ? C : fit / kThreads * kThreads;
  XC_REQUIRE(tile > 0, "scratch of %lld bytes holds the masks of %lld cells; a tile needs %lld (%lld bytes per cell)",
             (long long)scratch_bytes, (long long)fit, (long long)(C < kThreads ? C : kThreads), (long long)per_cell);
  cudaStream_t st = (cudaStream_t)stream;
  uint32_t* mask = static_cast<uint32_t*>(scratch);
  const size_t osz = reducer == XC_BOOT_SUM ? 4 : 8;
  for (int64_t c0 = 0; c0 < C; c0 += tile) {
    const int64_t n = C - c0 < tile ? C - c0 : tile;
    XC_CHECK_CUDA(cudaMemsetAsync(mask, 0, (size_t)(per_cell * n), st));
    int32_t e = launch_exceedance<kMask>(x + c0, n, ldx, base_start, N, L, window, percentile, alpha, beta, op,
                                         step_period, nullptr, MaskOut{mask, Wd, floor}, st);
    if (e) return e;
    dim3 grid((unsigned)((n + kThreads - 1) / kThreads), (unsigned)N, 1);
    const float* wet = wet_total ? wet_total + c0 : nullptr;
    void* o = static_cast<char*>(out) + (size_t)c0 * osz;
    const int after = resample_before_rl ? 0 : 1;
    switch (reducer) {
      case XC_BOOT_COUNT:
        bootstrap_reduce_kernel<XC_BOOT_COUNT><<<grid, kThreads, 0, st>>>(mask, n, Wd, N, L, step_period, run_window,
                                                                          after, x + c0, ldx, base_start, wet, C, o);
        break;
      case XC_BOOT_SPELL:
        bootstrap_reduce_kernel<XC_BOOT_SPELL><<<grid, kThreads, 0, st>>>(mask, n, Wd, N, L, step_period, run_window,
                                                                          after, x + c0, ldx, base_start, wet, C, o);
        break;
      default:
        bootstrap_reduce_kernel<XC_BOOT_SUM><<<grid, kThreads, 0, st>>>(mask, n, Wd, N, L, step_period, run_window,
                                                                        after, x + c0, ldx, base_start, wet, C, o);
    }
    e = launch_status("bootstrap_reduce_kernel");
    if (e) return e;
  }
  return XC_OK;
}
