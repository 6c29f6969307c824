// First / last run of at least `window` steps per period.
//
// Replaces indices/run_length.py:543-740 (`_boundary_run`, `first_run`, `last_run`), general
// (non-ufunc) branches with `freq` given:
//   window == 1 : per period, index of the first (last) True; NaN when argmax == argmin, i.e. when
//                 the period is all False -- or all True (:603-605, reproduced on purpose).
//   window  > 1 : d = (_cumsum_reset(da, index=position) >= window) on the WHOLE series (:632-633),
//                 then per period the first (last) position where d is set: "first" = first t of the
//                 period with da true on t..t+window-1 (the run may extend past the period end),
//                 "last" = last t of the period with da true on t-window+1..t.
// Output: float32 index relative to the period start, NaN when there is none.
#include "runstat.cuh"

namespace xc {
namespace {

constexpr int kThreads = 128;
constexpr int kChunk = 8;

// Rows [lo, hi) of one cell in time order (or reversed), kChunk independent loads in flight before
// the serial state machine consumes them; body(step, value) returns true to stop (early exit at
// chunk granularity: at most kChunk - 1 rows are fetched for nothing).
template <typename F>
__device__ __forceinline__ void scan_forward(const float* __restrict__ col, int64_t ldx, int lo, int hi, F&& body) {
  for (int s0 = lo; s0 < hi; s0 += kChunk) {
    float v[kChunk];
#pragma unroll
    for (int k = 0; k < kChunk; ++k)
      if (s0 + k < hi) v[k] = ld_stream(col + (int64_t)(s0 + k) * ldx);
#pragma unroll
    for (int k = 0; k < kChunk; ++k)
      if (s0 + k < hi) {
        if (body(s0 + k, v[k])) return;
      }
  }
}
template <typename F>
__device__ __forceinline__ void scan_backward(const float* __restrict__ col, int64_t ldx, int lo, int hi, F&& body) {
  for (int s0 = hi - 1; s0 >= lo; s0 -= kChunk) {
    float v[kChunk];
#pragma unroll
    for (int k = 0; k < kChunk; ++k)
      if (s0 - k >= lo) v[k] = ld_stream(col + (int64_t)(s0 - k) * ldx);
#pragma unroll
    for (int k = 0; k < kChunk; ++k)
      if (s0 - k >= lo) {
        if (body(s0 - k, v[k])) return;
      }
  }
}

template <int OP>
__global__ void __launch_bounds__(kThreads)
boundary_run_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                    const int32_t* __restrict__ poff, float thr, int32_t window, int32_t last,
                    float* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c;
  float res = NAN;
  if (window == 1) {
    int first = -1, lastt = -1, ntrue = 0;
    scan_forward(col, ldx, t0, t1, [&](int t, float v) {
      if (cmp<OP>(v, thr)) {
        if (first < 0) first = t;
        lastt = t;
        ++ntrue;
      }
      return false;
    });
    if (ntrue > 0 && ntrue < t1 - t0) res = (float)((last ? lastt : first) - t0);
  } else if (!last) {
    int cur = 0, first = -1;
    bool any_false = false;
    const int end = min((int)T, t1 + window - 1);
    scan_forward(col, ldx, t0, end, [&](int s, float v) {
      const bool m = cmp<OP>(v, thr);
      cur = m ? cur + 1 : 0;
      any_false = any_false || !m;
      if (first < 0 && cur >= window) {
        first = s - window + 1;        // < t1 because s < t1 + window - 1
        if (first > t0) return true;   // d[t0] == 0: the argmax == argmin rule cannot apply
      }
      return first >= 0 && any_false;
    });
    // every position of the period qualifies (d all ones) -> argmax == argmin == 0 -> NaN (:603-605)
    const bool all_set = (first == t0) && !any_false && (end == t1 + window - 1);
    if (first >= 0 && !all_set) res = (float)(first - t0);
  } else {
    int cur = 0, lastt = -1;
    bool any_false = false;
    const int begin = max(0, t0 - window + 1);
    scan_backward(col, ldx, begin, t1, [&](int s, float v) {
      const bool m = cmp<OP>(v, thr);
      cur = m ? cur + 1 : 0;
      any_false = any_false || !m;
      if (lastt < 0 && cur >= window) {
        lastt = s + window - 1;
        if (lastt < t1 - 1) return true;
      }
      return lastt >= 0 && any_false;
    });
    const bool all_set = (lastt == t1 - 1) && !any_false && (begin == t0 - window + 1);
    if (lastt >= 0 && !all_set) res = (float)(lastt - t0);
  }
  out[(int64_t)p * C + c] = res;
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int32_t xc_period_boundary_run_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                              const int32_t* period_offsets, int32_t P, int32_t op, double thr,
                                              int32_t cmp_f64, int32_t window, int32_t position_last, float* out,
                                              void* stream) {
  XC_REQUIRE(x && period_offsets && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1, "window must be >= 1");
  const float t32 = fold_threshold(op, thr, cmp_f64);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P, 1);
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    boundary_run_kernel<OP><<<grid, kThreads, 0, st>>>(x, T, C, ldx, period_offsets, t32, window,
                                                       position_last ? 1 : 0, out);
    return launch_status("boundary_run_kernel");
  });
}

// ------------------------------------------------------------------------------------------------
// Runs confined to a per-period sub-range (date-bounded runs and seasons)
// ------------------------------------------------------------------------------------------------
// Replaces the per-group calls of indices/run_length.py:1148-1331 (`run_end_after_date`,
// `first_run_after_date`, `last_run_before_date`, `first_run_before_date`) and the two steps of
// `season` (:998-1110): the reference masks the group outside a date range (`da.where(time >= date)`,
// NaN -> False) and calls first_run / last_run on the group, so runs are confined to the range and to
// the group.  Here the range of period p is [range_lo[p], range_hi[p]) (absolute steps, inside the
// period; range_lo[p] < 0 = "the date is not in this group" -> NaN), `negate` evaluates the run on
// NOT(condition) (season end: `~da`, NaN data count as condition broken) and `cell_lo` (optional,
// (P, C) float32, relative to the period start, NaN -> 0) raises the lower bound per cell
// (`index >= beg.fillna(0)`, :977).
namespace xc {
namespace {

template <int OP>
__global__ void __launch_bounds__(kThreads)
boundary_run_range_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                          const int32_t* __restrict__ rlo, const int32_t* __restrict__ rhi, float thr,
                          int32_t negate, int32_t window, int32_t last, const float* __restrict__ cell_lo,
                          float* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  int lo = rlo[p], hi = min(rhi[p], t1);
  float res = NAN;
  if (lo >= 0) {
    lo = max(lo, t0);
    bool full = (lo == t0) && (hi == t1);
    if (cell_lo != nullptr) {
      const float b = cell_lo[(int64_t)p * C + c];
      const int bl = (b == b) ? (int)b : 0;
      if (t0 + bl > lo) { lo = t0 + bl; full = false; }
    }
    const float* col = x + c;
    auto cond = [&](float v) -> bool {
      const bool m = cmp<OP>(v, thr);
      return negate ? !m : m;
    };
    if (window == 1 && full) {
      // argmax == argmin rule on the whole group (indices/run_length.py:603-605): all-True -> NaN
      int first = -1, lastt = -1, ntrue = 0;
      scan_forward(col, ldx, lo, hi, [&](int s, float v) {
        if (cond(v)) {
          if (first < 0) first = s;
          lastt = s;
          ++ntrue;
        }
        return false;
      });
      if (ntrue > 0 && ntrue < hi - lo) res = (float)((last ? lastt : first) - t0);
    } else if (!last) {
      int cur = 0;
      scan_forward(col, ldx, lo, hi, [&](int s, float v) {
        cur = cond(v) ? cur + 1 : 0;
        if (cur >= window) res = (float)(s - window + 1 - t0);
        return cur >= window;
      });
    } else {
      int cur = 0;
      scan_backward(col, ldx, lo, hi, [&](int s, float v) {
        cur = cond(v) ? cur + 1 : 0;
        if (cur >= window) res = (float)(s + window - 1 - t0);
        return cur >= window;
      });
    }
  }
  out[(int64_t)p * C + c] = res;
}

}  // namespace
}  // namespace xc

extern "C" int32_t xc_period_boundary_run_range_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                                    const int32_t* period_offsets, const int32_t* range_lo,
                                                    const int32_t* range_hi, int32_t P, int32_t op, double thr,
                                                    int32_t cmp_f64, int32_t negate, int32_t window,
                                                    int32_t position_last, const float* cell_lo, float* out,
                                                    void* stream) {
  XC_REQUIRE(x && period_offsets && range_lo && range_hi && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1, "window must be >= 1");
  const float t32 = fold_threshold(op, thr, cmp_f64);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P, 1);
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    boundary_run_range_kernel<OP><<<grid, kThreads, 0, st>>>(x, C, ldx, period_offsets, range_lo, range_hi, t32,
                                                             negate ? 1 : 0, window, position_last ? 1 : 0, cell_lo,
                                                             out);
    return launch_status("boundary_run_range_kernel");
  });
}

// ------------------------------------------------------------------------------------------------
// Quantile of the run lengths of a period (rle_statistics reducer "qNN")
// ------------------------------------------------------------------------------------------------
// Replaces indices/run_length.py:320-327 with reducer = "quantile": `d.where(d >= window).quantile(q)`
// (numpy's linear / type-7 quantile over the run lengths >= window attributed to the period; 0 when
// there is none).  A lane owns one (period, cell): the runs closed inside the period go to its
// shared-memory column (uint16, at most ceil(len/2) runs, each at most len steps), the run still open
// at the period end is held in a register (`tail`): with resample_before_rl=False it keeps its full
// length up to the end of the series, which may exceed 65535.  The two neighbouring order statistics
// are found by counting over both.
namespace xc {
namespace {

template <int OP>
__global__ void __launch_bounds__(kThreads)
run_quantile_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                    float thr, int32_t window, int32_t after, double q, int32_t cap, float* __restrict__ out) {
  extern __shared__ unsigned short runs[];  // [cap][kThreads]
  const int lane = threadIdx.x;
  const int64_t c = (int64_t)blockIdx.x * kThreads + lane;
  if (c >= C) return;
  const int p = blockIdx.y;
  const int t0 = poff[p], t1 = poff[p + 1];
  const float* col = x + c;
  int m = 0, cur = 0, longest = 0;
  PeriodMask pm;
  pm.init();
  if (after && t0 > 0) pm.look_back(cmp<OP>(ld_stream(col + (int64_t)(t0 - 1) * ldx), thr));
  auto close_run = [&]() {   // a run that ends inside the period: cur <= t1 - t0 < 65536
    if (cur >= window && m < cap) {
      runs[(size_t)m++ * kThreads + lane] = (unsigned short)cur;
      longest = max(longest, cur);
    }
    cur = 0;
  };
  // 8 rows in flight (one dependent load per step reached 0.055 of the HBM roofline)
  stream_rows<1, 8>(col, ldx, t0, t1, [&](const Vec<1>& r) {
    if (pm.inside(after, cmp<OP>(r.v[0], thr))) ++cur; else close_run();
  });
  if (after) {   // the run open at t1 belongs to this period with its full length
    for (int t = t1; cur > 0 && t < (int)T; ++t) {
      if (!PeriodMask::past_end(cmp<OP>(ld_stream(col + (int64_t)t * ldx), thr), cur > 0)) break;
      ++cur;
    }
  }
  const int tail = cur >= window ? cur : 0;    // 0: no run
  longest = max(longest, tail);
  const int n = m + (tail > 0 ? 1 : 0);
  float res = 0.f;
  if (n > 0) {
    // numpy linear quantile: pos = q (n - 1); lerp of the two neighbouring order statistics
    const double pos = q * (double)(n - 1);
    const int ilo = (int)floor(pos);
    const int ihi = min(ilo + 1, n - 1);
    const double g = pos - (double)ilo;
    // order statistics ilo, ihi of n integers: bisection on the VALUE (#{run <= v} is monotone in v), at most
    // ceil(log2(longest + 1)) counting passes instead of the n^2 rank count; the upper neighbour is vlo itself when
    // ties cover rank ihi, else the smallest length above vlo
    int lo_v = 0, hi_v = longest;              // smallest v with #{run <= v} >= ilo + 1
    while (lo_v < hi_v) {
      const int mid = lo_v + ((hi_v - lo_v) >> 1);
      int le = (tail > 0 && tail <= mid) ? 1 : 0;
      for (int k = 0; k < m; ++k) le += (runs[(size_t)k * kThreads + lane] <= mid) ? 1 : 0;
      if (le >= ilo + 1) hi_v = mid; else lo_v = mid + 1;
    }
    int le = (tail > 0 && tail <= lo_v) ? 1 : 0;
    int nxt = (tail > lo_v) ? tail : INT_MAX;
    for (int k = 0; k < m; ++k) {
      const int vk = runs[(size_t)k * kThreads + lane];
      le += (vk <= lo_v) ? 1 : 0;
      nxt = (vk > lo_v && vk < nxt) ? vk : nxt;
    }
    const double vlo = (double)lo_v;
    const double vhi = (le >= ihi + 1) ? vlo : (double)nxt;
    const double d = vhi - vlo;
    res = (float)((g >= 0.5) ? (vhi - d * (1.0 - g)) : (vlo + d * g));
  }
  out[(int64_t)p * C + c] = res;
}

}  // namespace
}  // namespace xc

extern "C" int32_t xc_period_run_quantile_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                              const int32_t* period_offsets, const int32_t* period_offsets_host,
                                              int32_t P, int32_t op, double thr, int32_t cmp_f64, double q,
                                              int32_t window, int32_t resample_before_rl, float* out, void* stream) {
  XC_REQUIRE(x && period_offsets && period_offsets_host && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && P <= 65535 && T < 2147483647LL, "bad shape");
  XC_REQUIRE(window >= 1 && q >= 0.0 && q <= 1.0, "window must be >= 1 and q in [0, 1]");
  int maxlen = 0;
  for (int p = 0; p < P; ++p) {
    const int len = period_offsets_host[p + 1] - period_offsets_host[p];
    if (len > maxlen) maxlen = len;
  }
  const int cap = maxlen / 2 + 2;
  const size_t smem = (size_t)cap * kThreads * sizeof(unsigned short);
  if (smem > 200 * 1024) {
    set_error("periods of %d steps hold too many runs for the shared-memory run list", maxlen);
    return XC_ERR_UNSUPPORTED;
  }
  const float t32 = fold_threshold(op, thr, cmp_f64);
  dim3 grid((unsigned)((C + kThreads - 1) / kThreads), (unsigned)P, 1);
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    if (smem > 48 * 1024) {
      cudaError_t e = cudaFuncSetAttribute(run_quantile_kernel<OP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem);
      if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(run_quantile_kernel)");
    }
    run_quantile_kernel<OP><<<grid, kThreads, smem, st>>>(x, T, C, ldx, period_offsets, t32, window,
                                                          resample_before_rl ? 0 : 1, q, cap, out);
    return launch_status("run_quantile_kernel");
  });
}
