// Run-length reducers, period edges of the runs and per-period statistics shared by the streaming kernels: one
// copy of the rules.  The run-length code is __host__ __device__ so that a host build can test it.
#pragma once
#include <type_traits>

#include "common.cuh"

#define XC_RS_HD __host__ __device__ __forceinline__

namespace xc {

// ---- row streaming: VEC adjacent cells per thread, UNROLL rows in flight ------------------------------------------
template <int VEC>
struct Vec;
template <>
struct Vec<1> {
  float v[1];
  __device__ __forceinline__ void load(const float* p) { v[0] = ld_stream(p); }
};
template <>
struct Vec<2> {
  float v[2];
  __device__ __forceinline__ void load(const float* p) {
    float2 q;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(q.x), "=f"(q.y) : "l"(p));
    v[0] = q.x; v[1] = q.y;
  }
};
template <>
struct Vec<4> {
  float v[4];
  __device__ __forceinline__ void load(const float* p) {
    float4 q = ld_stream4(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  }
};

template <int VEC, typename T>
__device__ __forceinline__ void store_vec(T* dst, const T (&v)[VEC]) {
  if constexpr (VEC == 4 && sizeof(T) == 4) {
    uint4 q;
    q.x = *reinterpret_cast<const uint32_t*>(&v[0]);
    q.y = *reinterpret_cast<const uint32_t*>(&v[1]);
    q.z = *reinterpret_cast<const uint32_t*>(&v[2]);
    q.w = *reinterpret_cast<const uint32_t*>(&v[3]);
    *reinterpret_cast<uint4*>(dst) = q;
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) dst[i] = v[i];
  }
}

// Iterate f(Vec) over the rows t in [t0, t1) with UNROLL loads in flight.
template <int VEC, int UNROLL = 8, typename F>
__device__ __forceinline__ void stream_rows(const float* __restrict__ col, int64_t ldx, int t0, int t1, F&& f) {
  int t = t0;
  const float* p = col + (int64_t)t0 * ldx;
  for (; t + UNROLL <= t1; t += UNROLL) {
    Vec<VEC> r[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) r[u].load(p + (int64_t)u * ldx);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) f(r[u]);
    p += (int64_t)UNROLL * ldx;
  }
  for (; t < t1; ++t) {
    Vec<VEC> r;
    r.load(p);
    f(r);
    p += ldx;
  }
}

// ---- row streaming through shared memory: bulk copies (sm_90a) ------------------------------------------------------
// stream_rows for a tile of W contiguous cells read by W / (4 V) consumer threads of 4 V cells each, with the rows
// delivered by the bulk-copy engine instead of per-lane loads: one elected producer lane copies each row's W * 4 bytes
// (one cp.async.bulk per row) into a ring of S stages of R rows, each stage guarded by a full mbarrier (the bytes
// have landed) and an empty one (every consumer warp has read the stage).  A row touch is W * 4 bytes instead of a
// warp's 512 (wider touches measured faster on H100, up to 16 KB), and the bytes in flight do not drop to zero
// between batches of loads.  The producer and the consumers walk the same sequence of (cells, rows) ranges, each
// with its own BulkRows copy of the ring position.  Consumer j owns the 4-cell groups j + v * kConsumers, v < V,
// so that every shared-memory read of a warp is 512 contiguous bytes.
//   Copies need 16-byte aligned addresses and sizes: the tile's first cell, ldx and the cell count n are multiples
// of 4, and the buffer is 16-byte aligned.  Consumers beyond n read stale shared memory and must not store.
template <int W, int R, int S, int V>
struct BulkRows {
  static constexpr int kConsumers = W / (4 * V);
  static constexpr size_t kSmemBytes = (size_t)S * R * W * sizeof(float) + 2 * S * sizeof(uint64_t);
  static_assert(W % (128 * V) == 0, "whole consumer warps");

  float* ring;       // [S][R][W]
  uint64_t* full;    // [S]
  uint64_t* empty;   // [S]
  int stage;
  uint32_t phase;

  // every thread of the CTA, before the roles split (thread 0 initialises the barriers)
  __device__ __forceinline__ void init(unsigned char* smem) {
    ring = reinterpret_cast<float*>(smem);
    full = reinterpret_cast<uint64_t*>(smem + (size_t)S * R * W * sizeof(float));
    empty = full + S;
    stage = 0;
    phase = 0;
    if (threadIdx.x == 0) {
      for (int s = 0; s < S; ++s) {
        mbar_init(&full[s], 1);
        mbar_init(&empty[s], kConsumers / 32);
      }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
  }
  __device__ __forceinline__ void advance() {
    if (++stage == S) {
      stage = 0;
      phase ^= 1u;
    }
  }
  // producer lane: rows [t0, t1) of the n cells from `tile` (row stride ldx)
  __device__ __forceinline__ void produce(const float* tile, int64_t ldx, int n, int t0, int t1) {
    const uint32_t row_bytes = (uint32_t)n * sizeof(float);
    for (int t = t0; t < t1; t += R) {
      const int nr = min(R, t1 - t);
      mbar_wait(&empty[stage], phase ^ 1u);   // a fresh barrier passes parity 1: the first S stages are free
      mbar_expect_tx(&full[stage], (uint32_t)nr * row_bytes);
      const float* src = tile + (int64_t)t * ldx;
      for (int r = 0; r < nr; ++r) {
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
            ::"r"(smem_u32(ring + ((size_t)stage * R + r) * W)), "l"(src + (int64_t)r * ldx), "r"(row_bytes),
            "r"(smem_u32(&full[stage]))
            : "memory");
      }
      advance();
    }
  }
  // consumer thread j (0 <= j < kConsumers): f(v, Vec<4>) on its cell groups v = 0 .. V - 1 (cells
  // 4 (j + v * kConsumers) .. + 3) of every row of [t0, t1), in time order
  template <typename F>
  __device__ __forceinline__ void consume(int j, int t0, int t1, F&& f) {
    for (int t = t0; t < t1; t += R) {
      mbar_wait(&full[stage], phase);
      const float* s = ring + (size_t)stage * R * W + 4 * j;
      auto row = [&](int r) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const float4 q = *reinterpret_cast<const float4*>(s + (size_t)r * W + 4 * v * kConsumers);
          Vec<4> g;
          g.v[0] = q.x; g.v[1] = q.y; g.v[2] = q.z; g.v[3] = q.w;
          f(v, g);
        }
      };
      if (t + R <= t1) {
#pragma unroll
        for (int r = 0; r < R; ++r) row(r);
      } else {
        for (int r = 0; r < t1 - t; ++r) row(r);
      }
      __syncwarp();
      if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[stage]);
      advance();
    }
  }
};

// ---- threshold sources ----------------------------------------------------------------------------------------------
// What the element tests of a streaming kernel compare a cell's value with at step t.  A kernel loads the Row of a
// step with load() next to its data and takes the float32 threshold of lane i with at().
//   ScalarThr: one float32 threshold for every step and cell (nothing to load).
//   TableThr<OP, DOY>: float64 thresholds thr[row(t) * rstride + c], row(t) = doy[t] - 1 (a day-of-year table,
//     indices/_multivariate.py:1583-1590 with `resample_doy` as an index) or t (an array; rstride 0: one threshold
//     per cell).  numpy compares float32 data with a float64 threshold in float64 (SURVEY.md A.1); each threshold
//     is folded to the float32 with the same truth table (fold_f64), so that the element test is one float32
//     compare.
template <int VEC>
__device__ __forceinline__ void load_thr(const double* p, double (&t)[VEC]) {
  if constexpr (VEC == 4) {
    const double2 a = *reinterpret_cast<const double2*>(p), b = *reinterpret_cast<const double2*>(p + 2);
    t[0] = a.x; t[1] = a.y; t[2] = b.x; t[3] = b.y;
  } else {
    t[0] = *p;
  }
}

struct ScalarThr {
  float t;
  template <int VEC>
  struct Row {};
  template <int VEC>
  __device__ __forceinline__ void load(Row<VEC>&, int64_t, int) const {}
  template <int VEC>
  __device__ __forceinline__ float at(const Row<VEC>&, int) const { return t; }
};

// How a threshold source travels as a kernel parameter: a ScalarThr as its float, so that a kernel's scalar
// instantiation keeps the parameter list (and code) it has without a source.
template <typename SRC>
struct ThrParam {
  using type = SRC;
  static __host__ __device__ __forceinline__ SRC put(const SRC& s) { return s; }
  static __host__ __device__ __forceinline__ SRC get(const SRC& s) { return s; }
};
template <>
struct ThrParam<ScalarThr> {
  using type = float;
  static __host__ __device__ __forceinline__ float put(const ScalarThr& s) { return s.t; }
  static __host__ __device__ __forceinline__ ScalarThr get(float t) { return ScalarThr{t}; }
};

template <int OP, bool DOY>
struct TableThr {
  const int16_t* doy;
  const double* thr;
  int64_t rstride;
  template <int VEC>
  struct Row {
    double v[VEC];
  };
  // cells c0 .. c0 + VEC - 1 of step t
  template <int VEC>
  __device__ __forceinline__ void load(Row<VEC>& r, int64_t c0, int t) const {
    load_thr<VEC>(thr + c0 + (DOY ? (int64_t)(__ldg(doy + t) - 1) : (int64_t)t) * rstride, r.v);
  }
  template <int VEC>
  __device__ __forceinline__ float at(const Row<VEC>& r, int i) const { return fold_f64<OP>(r.v[i]); }
};

// stream_rows with the threshold rows of `src` (for the cells from c0) loaded alongside: f(Vec, Row) for every t in
// [t0, t1).  A ScalarThr source loads nothing: the loop is stream_rows'.
template <int VEC, int UNROLL = 8, typename SRC, typename F>
__device__ __forceinline__ void stream_rows_thr(const float* __restrict__ col, int64_t ldx, int t0, int t1,
                                                const SRC& src, int64_t c0, F&& f) {
  using Row = typename SRC::template Row<VEC>;
  int t = t0;
  const float* p = col + (int64_t)t0 * ldx;
  for (; t + UNROLL <= t1; t += UNROLL) {
    Vec<VEC> r[UNROLL];
    Row th[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      r[u].load(p + (int64_t)u * ldx);
      src.load(th[u], c0, t + u);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) f(r[u], th[u]);
    p += (int64_t)UNROLL * ldx;
  }
  for (; t < t1; ++t) {
    Vec<VEC> r;
    Row th;
    r.load(p);
    src.load(th, c0, t);
    f(r, th);
    p += ldx;
  }
}

// ---- run lengths ----------------------------------------------------------------------------------------------------
// Reducer value of a RunAcc that keeps every quantity and picks the reducer at run time (result(int)).
constexpr int kRunAny = -1;

// mean and std of n run lengths with sum s and sum of squares q; 0 when there is no run.  The variance is
// stat_result()'s, every operation rounded on the device (no contraction into a fused multiply-add).
XC_RS_HD float run_mean(int32_t n, int32_t s) {
  return n == 0 ? 0.f : (float)((double)s / (double)n);
}
XC_RS_HD float run_std(int32_t n, int32_t s, unsigned long long q) {
  if (n == 0) return 0.f;
  const double nn = (double)n;
#ifdef __CUDA_ARCH__
  const double m = __ddiv_rn((double)s, nn);
  const double var = __dsub_rn(__ddiv_rn((double)q, nn), __dmul_rn(m, m));
  return (float)__dsqrt_rn(var > 0.0 ? var : 0.0);
#else
  const double m = (double)s / nn;
  const double var = (double)q / nn - m * m;
  return (float)sqrt(var > 0.0 ? var : 0.0);
#endif
}

// Per-cell accumulator over the run lengths L >= window attributed to the period.
template <int RED>
struct RunAcc {
  int32_t a;        // MAX: max L ; MIN: min L ; SUM: sum L ; COUNT/MEAN/STD/any: n runs
  int32_t s;        // MEAN/STD/any: sum L
  unsigned long long q;  // STD/any: sum L^2
  int32_t mx, mn;   // any: max L, min L
  XC_RS_HD void init() {
    a = (RED == XC_RL_MIN) ? 0x7fffffff : 0;
    s = 0;
    q = 0ull;
    if constexpr (RED == kRunAny) {
      mx = 0;
      mn = 0x7fffffff;
    }
  }
  XC_RS_HD void add(int32_t L, bool take) {
    if constexpr (RED == XC_RL_MAX) a = take ? max(a, L) : a;
    if constexpr (RED == XC_RL_MIN) a = take ? min(a, L) : a;
    if constexpr (RED == XC_RL_SUM) a += take ? L : 0;
    if constexpr (RED == XC_RL_COUNT) a += take ? 1 : 0;
    if constexpr (RED == XC_RL_MEAN || RED == XC_RL_STD) {
      a += take ? 1 : 0;
      s += take ? L : 0;
    }
    if constexpr (RED == XC_RL_STD) q += take ? (unsigned long long)L * (unsigned long long)L : 0ull;
    if constexpr (RED == kRunAny) {
      // a branch, not selects: five branch-free updates with a 64-bit square cost registers on every step
      if (take) {
        a += 1;
        s += L;
        q += (unsigned long long)L * (unsigned long long)L;
        mx = max(mx, L);
        mn = min(mn, L);
      }
    }
  }
  XC_RS_HD float result() const {
    if constexpr (RED == XC_RL_MAX || RED == XC_RL_SUM || RED == XC_RL_COUNT) return (float)a;
    if constexpr (RED == XC_RL_MIN) return a == 0x7fffffff ? 0.f : (float)a;
    if constexpr (RED == XC_RL_MEAN) return run_mean(a, s);
    if constexpr (RED == XC_RL_STD) return run_std(a, s, q);
    return 0.f;
  }
  // the reducer chosen at run time (any); a fixed RED ignores `reducer`
  XC_RS_HD float result(int reducer) const {
    if constexpr (RED != kRunAny) return result();
    switch (reducer) {
      case XC_RL_MAX: return (float)mx;
      case XC_RL_MIN: return a ? (float)mn : 0.f;
      case XC_RL_SUM: return (float)s;
      case XC_RL_COUNT: return (float)a;
      case XC_RL_MEAN: return run_mean(a, s);
      default: return run_std(a, s, q);
    }
  }
};

// Run lengths of the mask a period sees into a RunAcc.  `cur` is the length of the open run (0: none; with the
// running SUM and COUNT forms 1 while a run is open).  run_step() extends the open run with mask value m or closes it,
// taken when it is at least `window` steps long; run_close() takes the run open at the period or series end.
// RUNNING selects the window-1 running forms, which need no run end: MAX the largest running length, SUM the number of
// mask steps, COUNT the number of run starts.
template <bool RUNNING = false, int RED>
XC_RS_HD void run_step(int32_t& cur, RunAcc<RED>& acc, bool m, int32_t window) {
  static_assert(!RUNNING || RED == XC_RL_MAX || RED == XC_RL_SUM || RED == XC_RL_COUNT, "no running form");
  if constexpr (RUNNING && RED == XC_RL_MAX) {
    cur = m ? cur + 1 : 0;
    acc.a = max(acc.a, cur);
  } else if constexpr (RUNNING && RED == XC_RL_SUM) {
    cur = m ? 1 : 0;
    acc.a += cur;
  } else if constexpr (RUNNING && RED == XC_RL_COUNT) {
    const int32_t now = m ? 1 : 0;
    acc.a += now & (cur ^ 1);
    cur = now;
  } else {
    const int32_t L = cur;
    acc.add(L, !m && L >= window);
    cur = m ? L + 1 : 0;
  }
}
template <bool RUNNING = false, int RED>
XC_RS_HD void run_close(int32_t cur, RunAcc<RED>& acc, int32_t window) {
  if constexpr (!RUNNING) acc.add(cur, cur >= window);
}

// The steps of a condition mask that make the runs of the period [t0, t1) (indices/run_length.py:87-132,
// resample_and_rl).  Without `after` (resample_before_rl=True) they are the runs of m[t0:t1], cut at the period
// edges.  With `after` (resample_before_rl=False) a run belongs to the period holding its FIRST step
// (run_length.py:329-334): a run already open at t0 belongs to an earlier period and is skipped, and a run still
// open at t1 keeps its full length past t1, where no new run may start (it would belong to a later period).
// A kernel passes the mask at t0 - 1 to look_back() (with `after`, when t0 > 0), every step of [t0, t1) through
// inside(), and with `after` the steps from t1 on through past_end() until its runs have closed.
struct PeriodMask {
  bool skip;   // the run open at t0 - 1 goes on
  XC_RS_HD void init() { skip = false; }
  XC_RS_HD void look_back(bool m) { skip = m; }
  XC_RS_HD bool inside(bool after, bool m) {
    if (after) {
      skip = skip && m;
      m = m && !skip;
    }
    return m;
  }
  // `open`: a run of this cell is open at the step before
  XC_RS_HD static bool past_end(bool m, bool open) { return m && open; }
};

// Statistic of n non-NaN values with float64 sum s and sum of squares q and their min or max m.  Mean, min and
// max of no values are NaN; std and var are q/n - mean^2 clamped at 0, each operation rounded to float64 with the
// _rn intrinsics: a fused multiply-add (-fmad) would round mean^2 differently, and the difference cancels to
// exactly what low-variance cells (a constant cell's 0) are made of.  oracle/stat_rule.py restates the rule that
// tests/test_gpu_stat_rule.py holds every copy of it to, bit for bit.
__device__ __forceinline__ float stat_result(int stat, int32_t n, double s, double q, float m) {
  const double nn = (double)n;
  switch (stat) {
    case XC_STAT_SUM: return (float)s;
    case XC_STAT_COUNT: return (float)n;
    case XC_STAT_MEAN: return n ? (float)(s / nn) : NAN;
    case XC_STAT_MIN:
    case XC_STAT_MAX: return n ? m : NAN;
    default: {
      if (!n) return NAN;
      const double mean = __ddiv_rn(s, nn);
      double var = __dsub_rn(__ddiv_rn(q, nn), __dmul_rn(mean, mean));
      var = var > 0.0 ? var : 0.0;
      return (stat == XC_STAT_STD) ? (float)__dsqrt_rn(var) : (float)var;
    }
  }
}

// Per-period statistic `stat` of a stream of values, NaN skipped.
struct StatAcc {
  int32_t n;
  double s, q;
  float m;         // min for XC_STAT_MIN, else max
  bool is_min;
  __device__ __forceinline__ void init(int stat) {
    n = 0;
    s = 0.0;
    q = 0.0;
    is_min = (stat == XC_STAT_MIN);
    m = is_min ? INFINITY : -INFINITY;
  }
  __device__ __forceinline__ void take(float r) {
    if (r == r) {
      ++n;
      s += (double)r;
      q += (double)r * (double)r;
      m = is_min ? fminf(m, r) : fmaxf(m, r);
    }
  }
  __device__ __forceinline__ float result(int stat) const { return stat_result(stat, n, s, q, m); }
};

}  // namespace xc
