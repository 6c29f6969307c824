// Streaming per-period statistics: threshold counts, run-length statistics, reductions.
//
// Replaces (reference paths relative to /root/reference/src/xclim):
//   indices/generic.py:301-361      compare, threshold_count
//   indices/generic.py:543-585      _spell_length_statistics (window == 1)
//   indices/run_length.py:87-132    resample_and_rl
//   indices/run_length.py:143-335   _cumsum_reset_np, rle, rle_statistics
//   indices/run_length.py:381-488   windowed_run_events / windowed_run_count
//   indices/generic.py:83-125       select_resample_op ; 1514-1552 cumulative_difference
//   core/missing.py:296-322         MissingAny's valid-step count (fused as `valid_count`)
//
// Design: the (time, lat, lon) buffer is coalesced along cells, so a THREAD owns VEC=4
// adjacent cells (one 128-bit load per time step; a warp reads 512 contiguous bytes per step) and
// marches through the time steps of ONE period keeping the run-length state machine in
// registers -- no shuffles, no shared memory, no intermediate arrays.  The grid is
// (cell-vectors, periods): every (period, cell) unit is independent when runs are cut at period
// edges; with resample_before_rl == 0 a unit additionally looks one step back (to skip a run
// that started earlier) and reads past the period end until its open runs close.  UNROLL
// independent 16-byte loads are issued before any use so that each thread keeps >= 128 B in
// flight; data is read exactly once (ld.global.nc.L1::no_allocate).
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "launch_plan.cuh"
#include "runstat.cuh"

namespace xc {
namespace {

// ------------------------------------------------------------------------------------------------
// threshold count (+ valid count)
// ------------------------------------------------------------------------------------------------
template <int OP, int VEC, bool VALID>
__global__ void __launch_bounds__(kThreads)
period_count_kernel(const float* __restrict__ x, int64_t C, int64_t ldx,
                    const int32_t* __restrict__ poff, float thr,
                    int32_t* __restrict__ out, int32_t* __restrict__ valid) {
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  int32_t cnt[VEC], nv[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { cnt[i] = 0; nv[i] = 0; }
  stream_rows<VEC>(x + c0, ldx, t0, t1, [&](const Vec<VEC>& r) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      cnt[i] += cmp<OP>(r.v[i], thr) ? 1 : 0;
      if constexpr (VALID) nv[i] += (r.v[i] == r.v[i]) ? 1 : 0;
    }
  });
  store_vec<VEC>(out + (int64_t)p * C + c0, cnt);
  if constexpr (VALID) store_vec<VEC>(valid + (int64_t)p * C + c0, nv);
}

// ------------------------------------------------------------------------------------------------
// run-length statistics
// ------------------------------------------------------------------------------------------------
// FASTMAX: reducer == max and window == 1 takes run_step's running form, which needs no run-end detection
// (this is the maximum_consecutive_dry_days configuration).  THR: the threshold source (runstat.cuh), a scalar or a
// day-of-year table (warm / cold spell duration indices, indices/_multivariate.py:69-153, 1719-1795).
template <int OP, int RED, int VEC, bool VALID, bool AFTER, bool FASTMAX, typename THR = ScalarThr>
__global__ void __launch_bounds__(kThreads)
period_runstat_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                      const int32_t* __restrict__ poff, typename ThrParam<THR>::type thr_param, int32_t window,
                      float* __restrict__ out, int32_t* __restrict__ valid) {
  using Row = typename THR::template Row<VEC>;
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c0;
  const THR thr = ThrParam<THR>::get(thr_param);

  int32_t cur[VEC], nv[VEC];
  PeriodMask pm[VEC];
  RunAcc<RED> acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { cur[i] = 0; nv[i] = 0; pm[i].init(); acc[i].init(); }

  if constexpr (AFTER) {
    if (t0 > 0) {
      Vec<VEC> r;
      Row th;
      r.load(col + (int64_t)(t0 - 1) * ldx);
      thr.load(th, c0, t0 - 1);
#pragma unroll
      for (int i = 0; i < VEC; ++i) pm[i].look_back(cmp<OP>(r.v[i], thr.at(th, i)));
    }
  }

  stream_rows_thr<VEC>(col, ldx, t0, t1, thr, c0, [&](const Vec<VEC>& r, const Row& th) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const bool c = cmp<OP>(r.v[i], thr.at(th, i));
      if constexpr (VALID) nv[i] += (r.v[i] == r.v[i]) ? 1 : 0;
      run_step<FASTMAX>(cur[i], acc[i], pm[i].inside(AFTER, c), window);
    }
  });

  if constexpr (AFTER) {
    // read on until every open run has closed (VALID counts only the period's own steps)
    bool open = false;
#pragma unroll
    for (int i = 0; i < VEC; ++i) open = open || (cur[i] > 0);
    for (int t = t1; open && t < (int)T; ++t) {
      Vec<VEC> r;
      Row th;
      r.load(col + (int64_t)t * ldx);
      thr.load(th, c0, t);
      open = false;
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const bool c = PeriodMask::past_end(cmp<OP>(r.v[i], thr.at(th, i)), cur[i] > 0);
        run_step<FASTMAX>(cur[i], acc[i], c, window);
        open = open || c;
      }
    }
  }
  float res[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    run_close<FASTMAX>(cur[i], acc[i], window);
    res[i] = acc[i].result();
  }
  store_vec<VEC>(out + (int64_t)p * C + c0, res);
  if constexpr (VALID) store_vec<VEC>(valid + (int64_t)p * C + c0, nv);
}

// The same statistic for a scalar threshold with runs cut at the period edges (AFTER == false), fed by the bulk-copy
// row ring (BulkRows, runstat.cuh): a persistent grid walks the (period, tile of kBulkCells cells) work items
// period-major, so that the CTAs running together stream the same rows and the tail is one item, not a partial wave.
// Every element goes through the same cmp / valid increment / run_step, in time order, as in period_runstat_kernel:
// the results are identical.
constexpr int kBulkCells = 4096;
constexpr int kBulkGroups = 4;   // 4-cell groups per consumer thread: 16 cells, 256 consumers
using RunRing = BulkRows<kBulkCells, 4, 3, kBulkGroups>;
constexpr int kBulkThreads = RunRing::kConsumers + 32;   // + one producer warp

template <int OP, int RED, bool VALID, bool FASTMAX>
__global__ void __launch_bounds__(kBulkThreads, 1)
period_runstat_bulk_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                           int32_t P, float thr, int32_t window, float* __restrict__ out, int32_t* __restrict__ valid) {
  constexpr int N = 4 * kBulkGroups;
  extern __shared__ __align__(128) unsigned char smem[];
  RunRing ring;
  ring.init(smem);
  const int64_t ntiles = (C + kBulkCells - 1) / kBulkCells;
  const int64_t items = ntiles * P;
  if (threadIdx.x >= RunRing::kConsumers) {
    if (threadIdx.x == RunRing::kConsumers) {
      for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const int p = (int)(it / ntiles);
        const int64_t c0 = (it - (int64_t)p * ntiles) * kBulkCells;
        ring.produce(x + c0, ldx, (int)min((int64_t)kBulkCells, C - c0), __ldg(poff + p), __ldg(poff + p + 1));
      }
    }
    return;
  }
  const int j = threadIdx.x;
  for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
    const int p = (int)(it / ntiles);
    const int64_t c0 = (it - (int64_t)p * ntiles) * kBulkCells;
    int32_t cur[N], nv[N];
    RunAcc<RED> acc[N];
#pragma unroll
    for (int i = 0; i < N; ++i) { cur[i] = 0; nv[i] = 0; acc[i].init(); }
    ring.consume(j, __ldg(poff + p), __ldg(poff + p + 1), [&](int v, const Vec<4>& r) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * v + e;
        const bool m = cmp<OP>(r.v[e], thr);
        if constexpr (VALID) nv[i] += (r.v[e] == r.v[e]) ? 1 : 0;
        run_step<FASTMAX>(cur[i], acc[i], m, window);
      }
    });
#pragma unroll
    for (int v = 0; v < kBulkGroups; ++v) {
      const int64_t c = c0 + 4 * (j + v * RunRing::kConsumers);
      if (c < C) {
        float res[4];
        int32_t n[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          run_close<FASTMAX>(cur[4 * v + e], acc[4 * v + e], window);
          res[e] = acc[4 * v + e].result();
          n[e] = nv[4 * v + e];
        }
        store_vec<4>(out + (int64_t)p * C + c, res);
        if constexpr (VALID) store_vec<4>(valid + (int64_t)p * C + c, n);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// windowed_max_run_sum of the excess over a threshold (indices/run_length.py:491-540 applied to
// `(x - thr).clip(0)`, indices/_threshold.py:2064-2073 `hot_spell_max_magnitude`): per period the
// largest sum of (x - thr) over a run of x > thr (x < thr: thr - x) at least `window` long, 0 if none.
// The excess is formed in float32 like the reference's `tasmax - thresh`; run sums are float64.
// ------------------------------------------------------------------------------------------------
template <int OP, int VEC, bool AFTER>
__global__ void __launch_bounds__(kThreads)
period_run_maxsum_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                         const int32_t* __restrict__ poff, float thr, int32_t window, float* __restrict__ out) {
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c0;
  int32_t cur[VEC];
  double rs[VEC], best[VEC];
  PeriodMask pm[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { cur[i] = 0; rs[i] = 0.0; best[i] = 0.0; pm[i].init(); }
  auto excess = [&](float v) -> float {
    const float d = (OP == XC_OP_GT || OP == XC_OP_GE) ? (v - thr) : (thr - v);
    return (d > 0.f) ? d : 0.f;  // NaN -> 0: not part of a run (rle: da > 0)
  };
  if constexpr (AFTER) {
    if (t0 > 0) {
      Vec<VEC> r;
      r.load(col + (int64_t)(t0 - 1) * ldx);
#pragma unroll
      for (int i = 0; i < VEC; ++i) pm[i].look_back(excess(r.v[i]) > 0.f);
    }
  }
  auto step = [&](int i, float e, bool in) {
    if (in) {
      cur[i] += 1;
      rs[i] += (double)e;
    } else {
      if (cur[i] >= window) best[i] = fmax(best[i], rs[i]);
      cur[i] = 0;
      rs[i] = 0.0;
    }
  };
  stream_rows<VEC>(col, ldx, t0, t1, [&](const Vec<VEC>& r) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float e = excess(r.v[i]);
      step(i, e, pm[i].inside(AFTER, e > 0.f));
    }
  });
  if constexpr (AFTER) {
    bool open = false;
#pragma unroll
    for (int i = 0; i < VEC; ++i) open = open || (cur[i] > 0);
    for (int t = t1; open && t < (int)T; ++t) {
      Vec<VEC> r;
      r.load(col + (int64_t)t * ldx);
      open = false;
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float e = excess(r.v[i]);
        const bool in = PeriodMask::past_end(e > 0.f, cur[i] > 0);
        step(i, e, in);
        open = open || in;
      }
    }
  }
  float res[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    if (cur[i] >= window) best[i] = fmax(best[i], rs[i]);
    res[i] = (float)best[i];
  }
  store_vec<VEC>(out + (int64_t)p * C + c0, res);
}

// ------------------------------------------------------------------------------------------------
// per-period reductions with optional fused transform
// ------------------------------------------------------------------------------------------------
template <int STAT, int TF, int OP, int VEC, bool VALID>
__global__ void __launch_bounds__(kThreads)
period_reduce_kernel(const float* __restrict__ x, int64_t C, int64_t ldx,
                     const int32_t* __restrict__ poff, float thr,
                     float* __restrict__ out, int32_t* __restrict__ valid) {
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  double s[VEC], q[VEC];
  float m[VEC];
  int32_t n[VEC], nv[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    s[i] = 0.0; q[i] = 0.0; n[i] = 0; nv[i] = 0;
    m[i] = (STAT == XC_STAT_MIN) ? INFINITY : -INFINITY;
  }
  stream_rows<VEC>(x + c0, ldx, t0, t1, [&](const Vec<VEC>& r) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      float v = r.v[i];
      if constexpr (VALID) nv[i] += (v == v) ? 1 : 0;
      if constexpr (TF == XC_TF_EXCESS) {
        // (x - t).clip(0) / (t - x).clip(0) in float32 (indices/generic.py:1545-1549)
        float d = (OP == XC_OP_GT || OP == XC_OP_GE) ? (v - thr) : (thr - v);
        v = (d != d) ? d : fmaxf(d, 0.f);
      }
      if constexpr (TF == XC_TF_WHERE) v = cmp<OP>(v, thr) ? v : NAN;
      const bool ok = (v == v);
      n[i] += ok ? 1 : 0;
      if constexpr (STAT == XC_STAT_SUM || STAT == XC_STAT_MEAN || STAT == XC_STAT_STD ||
                    STAT == XC_STAT_VAR)
        s[i] += ok ? (double)v : 0.0;
      if constexpr (STAT == XC_STAT_STD || STAT == XC_STAT_VAR) q[i] += ok ? (double)v * (double)v : 0.0;
      if constexpr (STAT == XC_STAT_MIN) m[i] = fminf(m[i], v);  // fminf ignores NaN
      if constexpr (STAT == XC_STAT_MAX) m[i] = fmaxf(m[i], v);
    }
  });
  float res[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const double nn = (double)n[i];
    if constexpr (STAT == XC_STAT_SUM) res[i] = (float)s[i];
    if constexpr (STAT == XC_STAT_COUNT) res[i] = (float)n[i];
    if constexpr (STAT == XC_STAT_MEAN) res[i] = n[i] ? (float)(s[i] / nn) : NAN;
    if constexpr (STAT == XC_STAT_MIN || STAT == XC_STAT_MAX) res[i] = n[i] ? m[i] : NAN;
    if constexpr (STAT == XC_STAT_STD || STAT == XC_STAT_VAR) {
      // stat_result()'s formula, kept as a copy: calling it reorders the register allocation of this kernel.
      // Every operation rounded, as there: this file is built with -fmad.
      if (n[i] == 0) {
        res[i] = NAN;
      } else {
        const double mean = __ddiv_rn(s[i], nn);
        double var = __dsub_rn(__ddiv_rn(q[i], nn), __dmul_rn(mean, mean));
        var = var > 0.0 ? var : 0.0;
        res[i] = (STAT == XC_STAT_STD) ? (float)__dsqrt_rn(var) : (float)var;
      }
    }
  }
  store_vec<VEC>(out + (int64_t)p * C + c0, res);
  if constexpr (VALID) store_vec<VEC>(valid + (int64_t)p * C + c0, nv);
}

inline bool can_vec4(const void* x, int64_t C, int64_t ldx, const void* o1, const void* o2) {
  return (C % 4 == 0) && (ldx % 4 == 0) && aligned16(x) && aligned16(o1) && (o2 == nullptr || aligned16(o2));
}

inline dim3 grid_for(int64_t C, int vec, int32_t P) {
  int64_t nvec = (C + vec - 1) / vec;
  return dim3((unsigned)((nvec + kThreads - 1) / kThreads), (unsigned)P, 1);
}

int32_t check_common(const void* x, int64_t T, int64_t C, int64_t ldx, const void* poff, int32_t P,
                     const void* out) {
  XC_REQUIRE(x != nullptr && out != nullptr && poff != nullptr, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C, "bad shape: T=%lld C=%lld ldx=%lld", (long long)T, (long long)C,
             (long long)ldx);
  XC_REQUIRE(T < 2147483647LL, "time axis too long");
  XC_REQUIRE(P > 0 && P <= 65535, "number of periods must be in [1, 65535], got %d", P);
  return XC_OK;
}


// ------------------------------------------------------------------------------------------------
// threshold count against a float64 threshold that varies by cell (TableThr, runstat.cuh): a day-of-year table
// (indices/_multivariate.py:1583-1590, `tx90p` & family, with `resample_doy` as an index into the table) or an array
// (indices/generic.py:301-361 with a DataArray threshold).
//   out[p, c] = #{ t in p : x[t, c] op thr[row(t) * rstride + c] },  row(t) = doy[t] - 1, or t without doy
// (rstride = 0: one threshold per cell).  The grid is (period, cell block) with the period fastest, so that the
// blocks of one cell range run together and share the threshold rows through L2.  U steps of data and thresholds
// are in flight before any use.
// SUMS (fraction_over_precip_thresh, indices/_multivariate.py:1283-1295) sums instead of counting, from the same
// read of x:  out[p, c] = sum of the x[t, c] that pass the table test,  valid[p, c] = sum of the x[t, c] with
// x op wet (the float32 wet-day threshold).  Both add float32 values into a float64 sum in time order and round it
// to float32 once, as period_reduce_kernel's conditional sum (thresholded_statistics, reducer "sum") does.
// ------------------------------------------------------------------------------------------------
template <int OP, int VEC, bool VALID, bool DOY, bool SUMS = false>
__global__ void __launch_bounds__(kThreads)
period_count_thr_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                        const int16_t* __restrict__ doy, const double* __restrict__ thr, int64_t rstride,
                        std::conditional_t<SUMS, float, int32_t>* __restrict__ out,
                        std::conditional_t<SUMS, float, int32_t>* __restrict__ valid, float wet) {
  constexpr int U = 4;
  const int p = blockIdx.x;
  const int64_t c0 = ((int64_t)blockIdx.y * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int t0 = poff[p], t1 = poff[p + 1];
  int32_t cnt[VEC], nv[VEC];
  double s_thr[VEC], s_wet[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { cnt[i] = 0; nv[i] = 0; }
  if constexpr (SUMS) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) { s_thr[i] = 0.0; s_wet[i] = 0.0; }
  }
  const float* col = x + c0;
  const double* tcol = thr + c0;
  // TableThr's row of step t, read through this kernel's __restrict__ pointers
  auto load = [&](int t, Vec<VEC>& r, double (&th)[VEC]) {
    r.load(col + (int64_t)t * ldx);
    load_thr<VEC>(tcol + (DOY ? (int64_t)(doy[t] - 1) : (int64_t)t) * rstride, th);
  };
  auto tally = [&](const Vec<VEC>& r, const double (&th)[VEC]) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      if constexpr (SUMS) {
        const float v = r.v[i];
        s_thr[i] += cmp<OP>(v, fold_f64<OP>(th[i])) ? (double)v : 0.0;
        s_wet[i] += cmp<OP>(v, wet) ? (double)v : 0.0;
      } else {
        cnt[i] += cmp<OP>(r.v[i], fold_f64<OP>(th[i])) ? 1 : 0;
        if constexpr (VALID) nv[i] += (r.v[i] == r.v[i]) ? 1 : 0;
      }
    }
  };
  int t = t0;
  for (; t + U <= t1; t += U) {
    Vec<VEC> r[U];
    double th[U][VEC];
#pragma unroll
    for (int u = 0; u < U; ++u) load(t + u, r[u], th[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) tally(r[u], th[u]);
  }
  for (; t < t1; ++t) {
    Vec<VEC> r;
    double th[VEC];
    load(t, r, th);
    tally(r, th);
  }
  if constexpr (SUMS) {
    float a[VEC], b[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) { a[i] = (float)s_thr[i]; b[i] = (float)s_wet[i]; }
    store_vec<VEC>(out + (int64_t)p * C + c0, a);
    store_vec<VEC>(valid + (int64_t)p * C + c0, b);
  } else {
    store_vec<VEC>(out + (int64_t)p * C + c0, cnt);
    if constexpr (VALID) store_vec<VEC>(valid + (int64_t)p * C + c0, nv);
  }
}

// 4 cells per thread when the layout allows 128-bit accesses, 1 otherwise; valid counts with a doy index only
// (SUMS: both sums always)
template <bool DOY, bool SUMS = false>
int32_t launch_count_thr(const float* x, int64_t C, int64_t ldx, const int32_t* poff, int32_t P, const int16_t* doy,
                         const double* thr, int64_t rstride, int32_t op, std::conditional_t<SUMS, float, int32_t>* out,
                         std::conditional_t<SUMS, float, int32_t>* valid, cudaStream_t st, float wet = 0.f) {
  const bool v4 = can_vec4(x, C, ldx, out, valid) && aligned16(thr) && rstride % 4 == 0;
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    auto go = [&](auto VECC, auto VALC) -> int32_t {
      constexpr int VEC = decltype(VECC)::value;
      const int64_t cblocks = (C + VEC * kThreads - 1) / (VEC * kThreads);
      XC_REQUIRE(cblocks <= 65535, "too many cells for one launch: tile the grid by latitude");
      const dim3 grid((unsigned)P, (unsigned)cblocks, 1);
      period_count_thr_kernel<decltype(OPC)::value, VEC, decltype(VALC)::value, DOY, SUMS>
          <<<grid, kThreads, 0, st>>>(x, C, ldx, poff, doy, thr, rstride, out, valid, wet);
      return launch_status("period_count_thr_kernel");
    };
    auto go2 = [&](auto VECC) -> int32_t {
      if constexpr (SUMS) {
        return go(VECC, std::true_type{});
      } else {
        if constexpr (DOY) {
          if (valid) return go(VECC, std::true_type{});
        }
        return go(VECC, std::false_type{});
      }
    };
    return v4 ? go2(std::integral_constant<int, 4>{}) : go2(std::integral_constant<int, 1>{});
  });
}

// ------------------------------------------------------------------------------------------------
// fused multi-output pass: every count / run statistic / reduction that shares (x, periods)
// ------------------------------------------------------------------------------------------------
// One thread = 2 adjacent cells x one period (64-bit loads, UNROLL rows in flight); the state of NC
// conditions (run length, count, longest run), NR windowed run outputs, NM largest-run-sum outputs and NS
// conditional sums lives in registers next to the plain statistics -- about 25 registers per cell for the
// richest pass of the batch (tasmax), so that 4-5 CTAs stay resident per SM.  Per element and cell: 7
// instructions per condition, 3 per run output, ~10 per run sum, 6 per conditional sum, 8 for the plain
// statistics.  The template arguments are the (rounded-up) numbers of each kind: unused entries are
// computed and dropped (their slots are -1).
// a[j] for a warp-uniform runtime j without dynamic register indexing (which would go through local memory)
template <int N, typename T>
__device__ __forceinline__ T pick_uniform(const T (&a)[N], int j) {
  T r = a[0];
#pragma unroll
  for (int k = 1; k < N; ++k) r = (j == k) ? a[k] : r;
  return r;
}

// Pipe balance (an SM sub-partition issues one warp instruction per clock but the ALU pipe -- compares, selects, integer
// adds, min/max -- and the FMA pipe each take one every OTHER clock): run lengths and counters are kept as
// float32 (exact below 2^24 steps) so that their updates are FFMA / FADD on the FMA pipe,
//     cf = (sgn * v > thr) ? 1 : 0;   len' = cf * len + cf;   fin = len - cf * len;   n += cf
// leaving one FSET and one FMNMX per condition on the ALU pipe, and the run outputs sit at fixed places (two
// per leading condition) so that no select chain is needed to find their condition.  (Integer state with 4 cells
// per thread needed 255 registers; integer state spends 18 FSEL + 18 ISETP per element in the select chains.)
// VEC / UNROLL: light passes (no run outputs) take 4 cells per thread, the others 2 cells and more rows in flight.
template <int NC, int NCR, int NM, int NS, int VEC, int UNROLL>
__global__ void __launch_bounds__(kThreads)
period_multi_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                    const XcMultiPlan plan, float* __restrict__ out, int64_t slot_stride) {
  constexpr int NR = 2 * NCR;
  constexpr int NC1 = NC > 0 ? NC : 1, NR1 = NR > 0 ? NR : 1, NM1 = NM > 0 ? NM : 1, NS1 = NS > 0 ? NS : 1;
  static_assert(NCR <= NC && (NM == 0 || NC > 0), "run outputs need their condition");
  const int64_t c0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * VEC;
  if (c0 >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  double s[VEC];
  float mn[VEC], mx[VEC], nok[VEC];
  float c_len[NC1][VEC], c_n[NC1][VEC], c_mx[NC1][VEC];
  float r_acc[NR1][VEC];
  double m_rs[NM1][VEC], m_best[NM1][VEC];
  double q[NS1][VEC];
  // run outputs: value added when a run of length L >= window closes = ra * L + rb  (sum: L, count: 1)
  float r_w[NR1], r_a[NR1], r_b[NR1];
#pragma unroll
  for (int k = 0; k < NR; ++k) {
    r_w[k] = (float)plan.runs[k].window;
    r_a[k] = plan.runs[k].kind == 0 ? 1.f : 0.f;
    r_b[k] = 1.f - r_a[k];
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    s[i] = 0.0; mn[i] = INFINITY; mx[i] = -INFINITY; nok[i] = 0.f;
#pragma unroll
    for (int j = 0; j < NC; ++j) { c_len[j][i] = 0.f; c_n[j][i] = 0.f; c_mx[j][i] = 0.f; }
#pragma unroll
    for (int k = 0; k < NR; ++k) r_acc[k][i] = 0.f;
#pragma unroll
    for (int k = 0; k < NM; ++k) { m_rs[k][i] = 0.0; m_best[k][i] = 0.0; }
#pragma unroll
    for (int k = 0; k < NS; ++k) q[k][i] = 0.0;
  }
  stream_rows<VEC, UNROLL>(x + c0, ldx, t0, t1, [&](const Vec<VEC>& r) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float v = r.v[i];
      const bool ok = (v == v);
      nok[i] += ok ? 1.f : 0.f;
      s[i] += ok ? (double)v : 0.0;
      mn[i] = fminf(mn[i], v);
      mx[i] = fmaxf(mx[i], v);
      float cf[NC1], fin[NC1];   // cf: condition as 1 / 0; fin: length of the run that ends at this step (0: none)
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        cf[j] = (plan.cond[j].sgn * v > plan.cond[j].thr) ? 1.f : 0.f;
        const float L = c_len[j][i];
        fin[j] = __fmaf_rn(-cf[j], L, L);
        c_len[j][i] = __fmaf_rn(cf[j], L, cf[j]);
        c_n[j][i] += cf[j];
        c_mx[j][i] = fmaxf(c_mx[j][i], c_len[j][i]);
      }
#pragma unroll
      for (int k = 0; k < NR; ++k) {   // windows are >= 1: fin == 0 never qualifies
        const float L = fin[k >> 1];
        const float take = (L >= r_w[k]) ? 1.f : 0.f;
        r_acc[k][i] = __fmaf_rn(take, __fmaf_rn(r_a[k], L, r_b[k]), r_acc[k][i]);
      }
      if constexpr (NM > 0) {
        const float e = plan.msum[0].sgn * (v - plan.msum[0].thr0);   // float32 excess, like `tasmax - thresh`
        m_best[0][i] = (fin[0] >= (float)plan.msum[0].window) ? fmax(m_best[0][i], m_rs[0][i]) : m_best[0][i];
        m_rs[0][i] = (cf[0] != 0.f) ? m_rs[0][i] + (double)e : 0.0;
      }
#pragma unroll
      for (int k = 0; k < NS; ++k) {
        if (plan.sums[k].mode == 0) {
          const float d = plan.sums[k].off_sgn * (v - plan.sums[k].off);     // (x - t) / (t - x) in float32
          q[k][i] += ok ? (double)fmaxf(d, 0.f) : 0.0;
        } else {
          q[k][i] += (plan.sums[k].sgn * v > plan.sums[k].thr) ? (double)v : 0.0;
        }
      }
    }
  });
  auto put_f = [&](int slot, const float (&v)[VEC]) {
    if (slot >= 0) store_vec<VEC>(out + (int64_t)slot * slot_stride + (int64_t)p * C + c0, v);
  };
  auto put_i = [&](int slot, const int32_t (&v)[VEC]) {
    if (slot >= 0) store_vec<VEC>(reinterpret_cast<int32_t*>(out) + (int64_t)slot * slot_stride + (int64_t)p * C + c0, v);
  };
  float rf[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) rf[i] = (float)s[i];
  put_f(plan.slot_sum, rf);
#pragma unroll
  for (int i = 0; i < VEC; ++i) rf[i] = (nok[i] != 0.f) ? (float)(s[i] / (double)nok[i]) : NAN;
  put_f(plan.slot_mean, rf);
#pragma unroll
  for (int i = 0; i < VEC; ++i) rf[i] = (nok[i] != 0.f) ? mn[i] : NAN;
  put_f(plan.slot_min, rf);
#pragma unroll
  for (int i = 0; i < VEC; ++i) rf[i] = (nok[i] != 0.f) ? mx[i] : NAN;
  put_f(plan.slot_max, rf);
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    int32_t ri[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) ri[i] = (int32_t)c_n[j][i];
    put_i(plan.cond[j].slot_n, ri);
#pragma unroll
    for (int i = 0; i < VEC; ++i) rf[i] = (c_mx[j][i] >= (float)plan.cond[j].wmax) ? c_mx[j][i] : 0.f;
    put_f(plan.cond[j].slot_max, rf);
  }
#pragma unroll
  for (int k = 0; k < NR; ++k) {      // runs closed by the period end
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float L = c_len[k >> 1][i];
      rf[i] = r_acc[k][i] + ((L >= r_w[k]) ? __fmaf_rn(r_a[k], L, r_b[k]) : 0.f);
    }
    put_f(plan.runs[k].slot, rf);
  }
  if constexpr (NM > 0) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float L = c_len[0][i];
      rf[i] = (float)((L >= (float)plan.msum[0].window) ? fmax(m_best[0][i], m_rs[0][i]) : m_best[0][i]);
    }
    put_f(plan.msum[0].slot, rf);
  }
#pragma unroll
  for (int k = 0; k < NS; ++k) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) rf[i] = (float)q[k][i];
    put_f(plan.sums[k].slot, rf);
  }
}

template <int NC, int NCR, int NM, int NS>
int32_t launch_multi(const float* x, int64_t C, int64_t ldx, const int32_t* poff, int32_t P, const XcMultiPlan& plan,
                     float* out, cudaStream_t st) {
  constexpr MultiShape s = multi_shape(NC, 2 * NCR, NM, NS);
  period_multi_kernel<NC, NCR, NM, NS, s.vec, s.unroll><<<grid_for(C, s.vec, P), kThreads, 0, st>>>(
      x, C, ldx, poff, plan, out, (int64_t)P * C);
  return launch_status("period_multi_kernel");
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int32_t xc_period_count_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                       const int32_t* period_offsets, int32_t P, int32_t op, double thr,
                                       int32_t cmp_f64, int32_t* out_count, int32_t* valid_count,
                                       void* stream) {
  if (int32_t e = check_common(x, T, C, ldx, period_offsets, P, out_count)) return e;
  const float t32 = fold_threshold(op, thr, cmp_f64);
  const bool v4 = can_vec4(x, C, ldx, out_count, valid_count);
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_op_nan(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    auto go = [&](auto VECC, auto VALC) -> int32_t {
      constexpr int VEC = decltype(VECC)::value;
      constexpr bool VAL = decltype(VALC)::value;
      period_count_kernel<OP, VEC, VAL><<<grid_for(C, VEC, P), kThreads, 0, st>>>(
          x, C, ldx, period_offsets, t32, out_count, valid_count);
      return launch_status("period_count_kernel");
    };
    if (v4) return valid_count ? go(std::integral_constant<int, 4>{}, std::true_type{})
                               : go(std::integral_constant<int, 4>{}, std::false_type{});
    return valid_count ? go(std::integral_constant<int, 1>{}, std::true_type{})
                       : go(std::integral_constant<int, 1>{}, std::false_type{});
  });
}

namespace {
template <int OP, int RED, bool FASTMAX, bool VALID>
int32_t launch_runstat_bulk(const float* x, int64_t C, int64_t ldx, const int32_t* poff, int32_t P, float thr,
                            int32_t window, float* out, int32_t* valid, cudaStream_t st) {
  auto* kernel = period_runstat_bulk_kernel<OP, RED, VALID, FASTMAX>;
  constexpr size_t smem = RunRing::kSmemBytes;
  if (int32_t e = allow_smem(kernel, smem, "period_runstat_bulk_kernel")) return e;
  int per_sm = 0;
  XC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kBulkThreads, smem));
  const int64_t items = (C + kBulkCells - 1) / kBulkCells * P;
  const int grid = (int)std::min<int64_t>(items, (int64_t)sm_count() * std::max(per_sm, 1));
  kernel<<<grid, kBulkThreads, smem, st>>>(x, C, ldx, poff, P, thr, window, out, valid);
  return launch_status("period_runstat_bulk_kernel");
}

// v4: the layout of the threshold source allows 4 cells per thread as well.  A scalar threshold with runs cut at
// the period edges on at least one tile of cells goes to the bulk-copy kernel, unless XCLIM_B200_RUNSTAT_V1 is set
// (the per-lane kernel for every call: the two give identical results, and tests compare them).  The std reducer
// stays on the per-lane kernel.
template <int OP, int RED, bool FASTMAX, typename THR>
int32_t launch_runstat(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* poff, int32_t P,
                       THR thr, int32_t window, bool after, float* out, int32_t* valid, cudaStream_t st,
                       bool thr_v4 = true) {
  const bool v4 = can_vec4(x, C, ldx, out, valid) && thr_v4;
  // std keeps the per-lane kernel: its 64-bit sums of squares for 16 cells per thread spill in the bulk kernel
  if constexpr (std::is_same_v<THR, ScalarThr> && RED != XC_RL_STD) {
    if (v4 && !after && C >= kBulkCells && !getenv("XCLIM_B200_RUNSTAT_V1")) {
      return valid ? launch_runstat_bulk<OP, RED, FASTMAX, true>(x, C, ldx, poff, P, thr.t, window, out, valid, st)
                   : launch_runstat_bulk<OP, RED, FASTMAX, false>(x, C, ldx, poff, P, thr.t, window, out, valid, st);
    }
  }
  auto go = [&](auto VECC, auto VALC, auto AFTC) -> int32_t {
    constexpr int VEC = decltype(VECC)::value;
    constexpr bool VAL = decltype(VALC)::value;
    constexpr bool AFT = decltype(AFTC)::value;
    period_runstat_kernel<OP, RED, VEC, VAL, AFT, FASTMAX, THR><<<grid_for(C, VEC, P), kThreads, 0, st>>>(
        x, T, C, ldx, poff, ThrParam<THR>::put(thr), window, out, valid);
    return launch_status("period_runstat_kernel");
  };
  auto go2 = [&](auto VECC) -> int32_t {
    if (valid) return after ? go(VECC, std::true_type{}, std::true_type{}) : go(VECC, std::true_type{}, std::false_type{});
    return after ? go(VECC, std::false_type{}, std::true_type{}) : go(VECC, std::false_type{}, std::false_type{});
  };
  return v4 ? go2(std::integral_constant<int, 4>{}) : go2(std::integral_constant<int, 1>{});
}
}  // namespace

extern "C" int32_t xc_period_runstat_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                         const int32_t* period_offsets, int32_t P, int32_t op, double thr,
                                         int32_t cmp_f64, int32_t reducer, int32_t window,
                                         int32_t resample_before_rl, float* out, int32_t* valid_count,
                                         void* stream) {
  if (int32_t e = check_common(x, T, C, ldx, period_offsets, P, out)) return e;
  XC_REQUIRE(window >= 1, "window must be >= 1, got %d", window);
  XC_REQUIRE(reducer >= XC_RL_MAX && reducer <= XC_RL_STD, "unknown run-length reducer %d", reducer);
  const float t32 = fold_threshold(op, thr, cmp_f64);
  const bool after = resample_before_rl == 0;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_op_nan(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
#define XC_RS(RED, FAST) \
  return launch_runstat<OP, RED, FAST>(x, T, C, ldx, period_offsets, P, ScalarThr{t32}, window, after, out, valid_count, st)
    switch (reducer) {
      case XC_RL_MAX:
        if (window == 1) { XC_RS(XC_RL_MAX, true); }
        XC_RS(XC_RL_MAX, false);
      case XC_RL_MIN: XC_RS(XC_RL_MIN, false);
      case XC_RL_SUM: XC_RS(XC_RL_SUM, false);
      case XC_RL_COUNT: XC_RS(XC_RL_COUNT, false);
      case XC_RL_MEAN: XC_RS(XC_RL_MEAN, false);
      default: XC_RS(XC_RL_STD, false);
    }
#undef XC_RS
  });
}

namespace {
template <int STAT, int TF, int OP>
int32_t launch_reduce(const float* x, int64_t C, int64_t ldx, const int32_t* poff, int32_t P, float t32,
                      float* out, int32_t* valid, cudaStream_t st) {
  const bool v4 = can_vec4(x, C, ldx, out, valid);
  auto go = [&](auto VECC, auto VALC) -> int32_t {
    constexpr int VEC = decltype(VECC)::value;
    constexpr bool VAL = decltype(VALC)::value;
    period_reduce_kernel<STAT, TF, OP, VEC, VAL><<<grid_for(C, VEC, P), kThreads, 0, st>>>(x, C, ldx, poff, t32,
                                                                                         out, valid);
    return launch_status("period_reduce_kernel");
  };
  if (v4) return valid ? go(std::integral_constant<int, 4>{}, std::true_type{})
                       : go(std::integral_constant<int, 4>{}, std::false_type{});
  return valid ? go(std::integral_constant<int, 1>{}, std::true_type{})
               : go(std::integral_constant<int, 1>{}, std::false_type{});
}

template <int TF, int OP>
int32_t reduce_stat(int32_t stat, const float* x, int64_t C, int64_t ldx, const int32_t* poff, int32_t P, float t32,
                    float* out, int32_t* valid, cudaStream_t st) {
  switch (stat) {
    case XC_STAT_SUM: return launch_reduce<XC_STAT_SUM, TF, OP>(x, C, ldx, poff, P, t32, out, valid, st);
    case XC_STAT_MEAN: return launch_reduce<XC_STAT_MEAN, TF, OP>(x, C, ldx, poff, P, t32, out, valid, st);
    case XC_STAT_MIN: return launch_reduce<XC_STAT_MIN, TF, OP>(x, C, ldx, poff, P, t32, out, valid, st);
    case XC_STAT_MAX: return launch_reduce<XC_STAT_MAX, TF, OP>(x, C, ldx, poff, P, t32, out, valid, st);
    case XC_STAT_STD: return launch_reduce<XC_STAT_STD, TF, OP>(x, C, ldx, poff, P, t32, out, valid, st);
    case XC_STAT_VAR: return launch_reduce<XC_STAT_VAR, TF, OP>(x, C, ldx, poff, P, t32, out, valid, st);
    case XC_STAT_COUNT: return launch_reduce<XC_STAT_COUNT, TF, OP>(x, C, ldx, poff, P, t32, out, valid, st);
  }
  set_error("unknown reduction %d", stat);
  return XC_ERR_INVALID;
}
}  // namespace

extern "C" int32_t xc_period_reduce_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                        const int32_t* period_offsets, int32_t P, int32_t stat,
                                        int32_t transform, int32_t op, double thr, float* out,
                                        int32_t* valid_count, void* stream) {
  if (int32_t e = check_common(x, T, C, ldx, period_offsets, P, out)) return e;
  cudaStream_t st = (cudaStream_t)stream;
  if (transform == XC_TF_NONE)
    return reduce_stat<XC_TF_NONE, XC_OP_GT>(stat, x, C, ldx, period_offsets, P, 0.f, out, valid_count, st);
  // thresholds of the fused transforms are applied in float32 (float32 data op python float)
  const float t32 = (float)thr;
  if (transform == XC_TF_EXCESS) {
    XC_REQUIRE(op >= XC_OP_GT && op <= XC_OP_LE, "Operation `%d` not permitted for indice.", op);
    if (op == XC_OP_GT || op == XC_OP_GE)
      return reduce_stat<XC_TF_EXCESS, XC_OP_GT>(stat, x, C, ldx, period_offsets, P, t32, out, valid_count, st);
    return reduce_stat<XC_TF_EXCESS, XC_OP_LT>(stat, x, C, ldx, period_offsets, P, t32, out, valid_count, st);
  }
  if (transform == XC_TF_WHERE) {
    return dispatch_op(op, [&](auto OPC) -> int32_t {
      constexpr int OP = decltype(OPC)::value;
      return reduce_stat<XC_TF_WHERE, OP>(stat, x, C, ldx, period_offsets, P, t32, out, valid_count, st);
    });
  }
  set_error("unknown transform %d", transform);
  return XC_ERR_INVALID;
}

extern "C" int32_t xc_period_run_maxsum_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                            const int32_t* period_offsets, int32_t P, int32_t op, double thr,
                                            int32_t window, int32_t resample_before_rl, float* out, void* stream) {
  if (int32_t e = check_common(x, T, C, ldx, period_offsets, P, out)) return e;
  XC_REQUIRE(window >= 1, "window must be >= 1, got %d", window);
  XC_REQUIRE(op >= XC_OP_GT && op <= XC_OP_LE, "Operation `%d` not permitted for indice.", op);
  const float t32 = (float)thr;
  const bool after = resample_before_rl == 0;
  const bool v4 = can_vec4(x, C, ldx, out, nullptr);
  cudaStream_t st = (cudaStream_t)stream;
  auto go = [&](auto OPC, auto VECC, auto AFTC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    constexpr int VEC = decltype(VECC)::value;
    constexpr bool AFT = decltype(AFTC)::value;
    period_run_maxsum_kernel<OP, VEC, AFT><<<grid_for(C, VEC, P), kThreads, 0, st>>>(x, T, C, ldx, period_offsets,
                                                                                   t32, window, out);
    return launch_status("period_run_maxsum_kernel");
  };
  auto go2 = [&](auto OPC) -> int32_t {
    if (v4) return after ? go(OPC, std::integral_constant<int, 4>{}, std::true_type{})
                         : go(OPC, std::integral_constant<int, 4>{}, std::false_type{});
    return after ? go(OPC, std::integral_constant<int, 1>{}, std::true_type{})
                 : go(OPC, std::integral_constant<int, 1>{}, std::false_type{});
  };
  return (op == XC_OP_GT || op == XC_OP_GE) ? go2(std::integral_constant<int, XC_OP_GT>{})
                                            : go2(std::integral_constant<int, XC_OP_LT>{});
}

extern "C" int32_t xc_period_multi_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                       const int32_t* period_offsets, int32_t P, const XcMultiPlan* plan_host,
                                       void* out, int32_t n_slots, void* stream) {
  int32_t e = check_common(x, T, C, ldx, period_offsets, P, out);
  if (e) return e;
  XC_REQUIRE(plan_host != nullptr, "null pointer argument");
  // run lengths and counters are float32: exact integers only below 2^24 steps
  XC_REQUIRE(T < (1LL << 24), "xc_period_multi_f32 counts in float32: time axis must be shorter than 2^24 steps, got %lld",
             (long long)T);
  XcMultiPlan pl = *plan_host;
  XC_REQUIRE(can_vec4(x, C, ldx, out, nullptr), "xc_period_multi_f32 needs C, ldx multiples of 4 and 16-byte aligned buffers");
  if (int32_t ep = check_multi_plan(pl, n_slots)) return ep;
  cudaStream_t st = (cudaStream_t)stream;
  float* o = (float*)out;
  const MultiShape sh = multi_shape(pl.n_cond, pl.n_runs, pl.n_msum, pl.n_sums);
  const int nc = sh.nc, ncr = sh.ncr, nm = sh.nm, ns = sh.ns;
#define XC_MULTI(CN, R, M, S) \
  if (nc == CN && ncr == R && nm == M && ns == S) return launch_multi<CN, R, M, S>(x, C, ldx, period_offsets, P, pl, o, st)
#define XC_MULTI_C(CN)                                                                                   \
  XC_MULTI(CN, 0, 0, 0); XC_MULTI(CN, 0, 0, 3); XC_MULTI(CN, 1, 0, 0); XC_MULTI(CN, 1, 0, 3);            \
  XC_MULTI(CN, 2, 0, 0); XC_MULTI(CN, 2, 0, 3); XC_MULTI(CN, 0, 1, 0); XC_MULTI(CN, 0, 1, 3);            \
  XC_MULTI(CN, 1, 1, 0); XC_MULTI(CN, 1, 1, 3); XC_MULTI(CN, 2, 1, 0); XC_MULTI(CN, 2, 1, 3)
  XC_MULTI(0, 0, 0, 0); XC_MULTI(0, 0, 0, 3);
  XC_MULTI_C(2); XC_MULTI_C(4); XC_MULTI_C(6);
#undef XC_MULTI_C
#undef XC_MULTI
  set_error("plan shape not instantiated");
  return XC_ERR_UNSUPPORTED;
}

extern "C" int32_t xc_period_count_arr_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                           const int32_t* period_offsets, int32_t P, int32_t op,
                                           const double* thr, int64_t thr_tstride, int32_t* out_count, void* stream) {
  int32_t e = check_common(x, T, C, ldx, period_offsets, P, out_count);
  if (e) return e;
  XC_REQUIRE(thr != nullptr, "null pointer argument");
  XC_REQUIRE(thr_tstride == 0 || thr_tstride >= C, "threshold time stride must be 0 (per cell) or >= C");
  return launch_count_thr<false>(x, C, ldx, period_offsets, P, nullptr, thr, thr_tstride, op, out_count, nullptr,
                                 (cudaStream_t)stream);
}

extern "C" int32_t xc_doy_threshold_count_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                              const int32_t* period_offsets, int32_t P,
                                              const int16_t* doy_index, const double* table, int32_t n_doy,
                                              int32_t op, int32_t* out_count, int32_t* valid_count, void* stream) {
  XC_REQUIRE(x && period_offsets && doy_index && table && out_count, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && n_doy > 0, "bad shape");
  return launch_count_thr<true>(x, C, ldx, period_offsets, P, doy_index, table, C, op, out_count, valid_count,
                                (cudaStream_t)stream);
}

extern "C" int32_t xc_doy_runstat_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                      const int32_t* period_offsets, int32_t P, const int16_t* doy_index,
                                      const double* table, int32_t n_doy, int32_t op, int32_t reducer,
                                      int32_t window, int32_t resample_before_rl, float* out, int32_t* valid_count,
                                      void* stream) {
  if (int32_t e = check_common(x, T, C, ldx, period_offsets, P, out)) return e;
  XC_REQUIRE(doy_index != nullptr && table != nullptr, "null pointer argument");
  XC_REQUIRE(n_doy > 0, "n_doy must be > 0, got %d", n_doy);
  XC_REQUIRE(window >= 1, "window must be >= 1, got %d", window);
  XC_REQUIRE(reducer >= XC_RL_MAX && reducer <= XC_RL_STD, "unknown run-length reducer %d", reducer);
  XC_REQUIRE(op >= XC_OP_GT && op <= XC_OP_LE, "Operation `%d` not permitted for indice.", op);
  const bool after = resample_before_rl == 0;
  const bool thr_v4 = aligned16(table);
  cudaStream_t st = (cudaStream_t)stream;
  auto by_op = [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    const TableThr<OP, true> src{doy_index, table, C};
#define XC_RS(RED) \
  return launch_runstat<OP, RED, false>(x, T, C, ldx, period_offsets, P, src, window, after, out, valid_count, st, thr_v4)
    switch (reducer) {
      case XC_RL_MAX: XC_RS(XC_RL_MAX);
      case XC_RL_MIN: XC_RS(XC_RL_MIN);
      case XC_RL_SUM: XC_RS(XC_RL_SUM);
      case XC_RL_COUNT: XC_RS(XC_RL_COUNT);
      case XC_RL_MEAN: XC_RS(XC_RL_MEAN);
      default: XC_RS(XC_RL_STD);
    }
#undef XC_RS
  };
  switch (op) {
    case XC_OP_GT: return by_op(std::integral_constant<int, XC_OP_GT>{});
    case XC_OP_LT: return by_op(std::integral_constant<int, XC_OP_LT>{});
    case XC_OP_GE: return by_op(std::integral_constant<int, XC_OP_GE>{});
    default: return by_op(std::integral_constant<int, XC_OP_LE>{});
  }
}

extern "C" int32_t xc_period_sums_thr_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                          const int32_t* period_offsets, int32_t P, const int16_t* doy_index,
                                          const double* thr, int64_t thr_rstride, int32_t op, double wet,
                                          float* out_sum_thr, float* out_sum_wet, void* stream) {
  if (int32_t e = check_common(x, T, C, ldx, period_offsets, P, out_sum_thr)) return e;
  XC_REQUIRE(thr != nullptr && out_sum_wet != nullptr, "null pointer argument");
  XC_REQUIRE(thr_rstride == 0 || thr_rstride >= C, "threshold row stride must be 0 (per cell) or >= C");
  XC_REQUIRE(op == XC_OP_GT || op == XC_OP_GE, "Operation `%d` not permitted for indice.", op);
  // the wet-day threshold is a Python float in the reference: compared in float32
  const float w32 = (float)wet;
  cudaStream_t st = (cudaStream_t)stream;
  if (doy_index)
    return launch_count_thr<true, true>(x, C, ldx, period_offsets, P, doy_index, thr, thr_rstride, op, out_sum_thr,
                                        out_sum_wet, st, w32);
  return launch_count_thr<false, true>(x, C, ldx, period_offsets, P, nullptr, thr, thr_rstride, op, out_sum_thr,
                                       out_sum_wet, st, w32);
}
